"""Depth evaluation without a GPU: the oracle (oracle/depth_eval.py) against the numbers frozen from the reference's own
generate_depth_map, generate_mask and compute_errors, then ccb_velo_depth, ccb_spline_zoom and ccb_eigen_depth_errors
compiled by g++ against the CPU execution-model simulator (tests/sim) against the fixture, the oracle and scipy's zoom.
The same cases run on the H100 in tests/test_gpu_depth_eval.py."""
import numpy as np
import pytest
import torch
from cc_b200 import evaluate as CE
from oracle import depth_eval as OD
from tests import depth_eval_cases as DC
from tests.util import sim_lib      # noqa: F401  (module fixture: the simulator library)

CPU = torch.device('cpu')


@pytest.mark.parametrize('case', DC.velo_cases(), ids=lambda c: c[0])
def test_oracle_depth_map_equals_reference(case, tmp_path):
    """The same pixels; values within one fp64 ulp (the projection is numpy's dgemm, whose summation order depends on the
    CPU's BLAS kernel; on the machine that froze the fixture they are identical)."""
    name, points, calib, shape, want = case
    DC.write_calib(str(tmp_path), calib)
    P = CE.kitti_velo_to_image(str(tmp_path), 2)
    assert np.array_equal(P, DC.OD_projection(calib))
    got = OD.generate_depth_map(points, P, shape)
    assert np.array_equal(got != 0, want != 0) and DC.ulp_diff(got, want) <= 1, name


def test_load_velodyne_points(tmp_path):
    pts = DC.kitti_sweep(np.random.RandomState(1), 50)
    pts.tofile(str(tmp_path / 'sweep.bin'))
    got = CE.load_velodyne_points(str(tmp_path / 'sweep.bin'))
    assert got.dtype == np.float32 and np.array_equal(got[:, :3], pts[:, :3]) and (got[:, 3] == 1).all()


@pytest.mark.parametrize('case', DC.error_cases(), ids=lambda c: c['name'])
def test_oracle_errors_equal_reference(case):
    c = case
    assert np.array_equal(OD.generate_mask(c['gt'], c['lo'], c['hi'], DC.crop_fractions(c['crop'])), c['mask'])
    got = OD.sample_errors(c['gt'], c['pred'], c['lo'], c['hi'], DC.crop_fractions(c['crop']), c['poses'], c['displacements'])
    assert np.array_equal(got, c['out'], equal_nan=True), (c['name'], got, c['out'])


def test_depth_summary():
    per = np.random.RandomState(2).rand(5, 2, 7)
    errors = np.zeros((2, 7, 5), np.float32)
    for j in range(5):
        errors[:, :, j] = per[j]
    got = CE.depth_summary(per)
    assert got.dtype == np.float32 and np.array_equal(got, errors.mean(2))


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('case', DC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(CPU)


@pytest.mark.usefixtures('sim_lib')
def test_velo_fixture(tmp_path):
    DC.case_velo_fixture(CPU, tmp_path)


@pytest.mark.usefixtures('sim_lib')
def test_velo_fixture_kitti_size(tmp_path):
    DC.case_velo_fixture(CPU, tmp_path, kitti=True)


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('sizes', DC.ZOOM_SIZES + [DC.KITTI], ids=lambda s: '%dx%d-%dx%d' % s)
def test_spline_zoom_vs_scipy(sizes):
    DC.case_zoom_vs_scipy(CPU, sizes, N=1 if sizes == DC.KITTI else 2)
