"""Depth evaluation on the H100: the kernel cases of tests/depth_eval_cases.py on the sm_90a library, the KITTI sizes at
B = 1 and B = 4 with bit-identical reruns, depth_eval_batch against the host depth_sample_errors and the oracle nets, and
the ground truth, zoom and errors chain inside a CUDA graph."""
import numpy as np
import pytest
import torch
from cc_b200 import evaluate as CE
from tests import depth_eval_cases as DC
from tests.util import assert_graph_replays, device_lib      # noqa: F401  (module fixture: the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]
DEV = torch.device('cuda:0')


@pytest.mark.parametrize('case', DC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(DEV)


@pytest.mark.parametrize('kitti', [False, True])
def test_velo_fixture(kitti, tmp_path):
    DC.case_velo_fixture(DEV, tmp_path, kitti=kitti)


@pytest.mark.parametrize('sizes', DC.ZOOM_SIZES + [DC.KITTI], ids=lambda s: '%dx%d-%dx%d' % s)
def test_spline_zoom_vs_scipy(sizes):
    DC.case_zoom_vs_scipy(DEV, sizes)


@pytest.mark.parametrize('B', [1, 4])
def test_kitti_size_exact_and_repeatable(B):
    """375x1242: ground truth and errors against the oracle per sample, and two more runs give the same bits."""
    DC.case_velo_vs_oracle(DEV, B=B, H=375, W=1242, n=60000, seed=60 + B, reruns=2)
    DC.case_errors_vs_oracle(DEV, B=B, H=375, W=1242, seed=70 + B, reruns=2)
    x = torch.from_numpy((1.0 / (np.random.RandomState(B).rand(B, 256, 832) * 0.3 + 0.01)).astype(np.float32)).to(DEV)
    z = CE.spline_zoom(x, 375, 1242, 1e-3, 80.0)
    for _ in range(2):
        assert torch.equal(CE.spline_zoom(x, 375, 1242, 1e-3, 80.0), z)


@pytest.mark.parametrize('with_pose', [False, True], ids=['DispResNet6', 'DispResNet6+PoseNetB6'])
def test_depth_eval_batch(with_pose):
    DC.case_eval_batch(DEV, with_pose)


def test_chain_in_cuda_graph():
    """Ground truth, zoom and errors make no host round-trip: captured once, replayed on new inputs in the same buffers."""
    B, H, W, h, w = 2, 60, 200, 40, 128
    rs = np.random.RandomState(90)
    P = DC.OD_projection(DC.kitti_calib(rs)) * np.array([[W / 1242.0], [H / 375.0], [1.0]])

    def inputs(seed):
        r = np.random.RandomState(seed)
        pts = np.concatenate([DC.kitti_sweep(r, 5000) for _ in range(B)])
        return [torch.from_numpy(pts).to(DEV), torch.from_numpy((r.rand(B, h, w) * 0.3 + 0.02).astype(np.float32)).to(DEV),
                torch.from_numpy(r.randn(B, 2, 6).astype(np.float32)).to(DEV), torch.from_numpy(r.uniform(0.1, 1, (B, 2))).to(DEV)]
    offs = torch.tensor([0, 5000, 10000], dtype=torch.int64, device=DEV)
    Pd = torch.from_numpy(np.stack([P] * B)).to(DEV)

    def chain(pts, disp, poses, displacements):
        gt = CE.velodyne_depth(pts, offs, Pd, H, W)
        pred = CE.spline_zoom(1 / disp, H, W, 1e-3, 80.0)
        return CE.depth_errors(gt, pred, 1e-3, 80.0, 'eigen', poses, displacements)
    eager = assert_graph_replays(chain, inputs(1), inputs(2))
    assert not torch.equal(eager[0], eager[1])
