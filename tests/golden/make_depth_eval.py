#!/usr/bin/env python
"""Generate tests/golden/depth_eval_small.npz from the UNMODIFIED reference: kitti_eval/depth_evaluation_utils.py
generate_depth_map (:148-191) and generate_mask (:194-206), stillbox_eval/depth_evaluation_utils.py generate_mask
(:68-80) and test_disp.py compute_errors (:171-187).  Run:  python tests/golden/make_depth_eval.py   (the reference
checkout is found as in make_golden.py; the other fixtures are not touched).

The modules import path, tqdm and scipy.misc (imread / imresize, gone from scipy), and test_disp also utils, models,
loss_functions and scipy.ndimage.interpolation; none of them is used by these functions, so each gets a stand-in for the
import (scipy.ndimage.interpolation an alias holding scipy's zoom).  generate_depth_map calls np.int, which numpy 2
removed: it is set to int around the calls.  Calibration files and .bin sweeps are written to a temporary directory by
tests/depth_eval_cases.py's writers.  The body of test_disp's sample loop (:124-141) lives inside main(): it is written
out here line by line around the reference's compute_errors and generate_mask.

Velodyne cases (<case>_points float32 [N,4], <case>_calib_<key> the calibration values, <case>_shape, the depth map
stored sparsely as <case>_idx / <case>_val):
  quirks        exact_calib() and quirk_sweep(9) in a 6x9 frame: every rule and quirk of the function
  random        a KITTI-like calibration and an 8000-point sweep, 40x130 (the intrinsics scaled to the frame)
  kitti         the same calibration unscaled, a 50000-point sweep, 375x1242
Error cases (<case>_gt_idx / _gt_val / _shape, <case>_pred fp32, _crop, _lo, _hi, <case>_mask packed bits from the
reference's generate_mask, optional _poses fp32 [R,6] and _displacements, <case>_out [2,7] the script's two rows in fp64):
  eigen_odd, eigen_even     Garg crop, odd / even mask counts, poses (one displacement 0), gt exactly at min and max depth
  stillbox                  the stillbox crop, poses
  zero_scale                no displacement > 0: scale 0, the script's inf / nan row
  nopose                    row 0 zeros"""
import os
import sys
import tempfile
import types
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG                      # noqa: E402  (reference import path, save helpers)
from make_mask_eval import _Absent            # noqa: E402
from tests import depth_eval_cases as DC     # noqa: E402


def import_reference():
    import pathlib
    import scipy.ndimage
    unused = ['path', 'tqdm', 'scipy.misc', 'utils', 'models', 'loss_functions']
    added = [m for m in unused if m not in sys.modules]
    for m in added:
        sys.modules[m] = _Absent(m)
    sys.modules['path'].Path = pathlib.Path
    if 'scipy.ndimage.interpolation' not in sys.modules:
        added.append('scipy.ndimage.interpolation')
        alias = types.ModuleType('scipy.ndimage.interpolation')
        alias.zoom = scipy.ndimage.zoom
        sys.modules['scipy.ndimage.interpolation'] = alias
    try:
        import test_disp
        from kitti_eval import depth_evaluation_utils as kitti
        from stillbox_eval import depth_evaluation_utils as stillbox
    finally:
        for m in added:
            del sys.modules[m]
    for mod in (test_disp, kitti, stillbox):
        assert os.path.abspath(mod.__file__).startswith(os.path.abspath(MG.REF)), mod.__file__
    return test_disp, kitti, stillbox


def gen():
    import pathlib
    test_disp, kitti, stillbox = import_reference()
    rs = np.random.RandomState(77)
    d, velo_cases, error_cases = {}, [], []
    tmp = tempfile.mkdtemp()

    def velo(name, calib, points, shape):
        cdir = os.path.join(tmp, name)
        DC.write_calib(cdir, calib)
        fn = os.path.join(tmp, name + '.bin')
        points.tofile(fn)
        np.int = int
        try:
            depth = kitti.generate_depth_map(pathlib.Path(cdir), fn, shape, 2)
        finally:
            del np.int
        d[name + '_points'] = points
        for k, v in calib.items():
            d[name + '_calib_' + k] = v
        d[name + '_shape'] = np.array(shape)
        d[name + '_idx'], d[name + '_val'] = DC.sparse(depth)
        velo_cases.append(name)
        return depth

    with np.errstate(divide='ignore', invalid='ignore'):
        q = velo('quirks', DC.exact_calib(), DC.quirk_sweep(9), (6, 9))
    assert q[1, 2] == 1.0 and q[2, 3] == 0.0 and q[0, 8] == 1.0 and q[1, 0] == 1.0 and q[3, 0] == 1.0 and q[2, 8] == 1.0, q
    calib = DC.kitti_calib(rs)
    small = dict(calib, P_rect_02=(calib['P_rect_02'].reshape(3, 4) * np.array([[130 / 1242.0], [40 / 375.0], [1.0]])).ravel())
    velo('random', small, DC.kitti_sweep(rs, 8000), (40, 130))
    full = velo('kitti', calib, DC.kitti_sweep(rs, 50000), (375, 1242))
    assert 0.02 < (full > 0).mean() < 0.2

    def poses(R):
        """fp32 poses whose torch norms are the correctly rounded ones (the oracle's and the kernel's), redrawn otherwise:
        the fixture pins the script's arithmetic, not an ulp of torch's CPU norm."""
        while True:
            p = rs.randn(R, 6).astype(np.float32)
            if np.array_equal(torch.from_numpy(p)[:, :3].norm(2, 1).numpy(), DC.OD.pose_norms(p)):
                return p

    def errors(name, gt, pred, crop, poses=None, displacements=None, lo=1e-3, hi=80.0):
        mask = (kitti if crop == 'eigen' else stillbox).generate_mask(gt, lo, hi)
        pred_m, gt_m = pred[mask], gt[mask]
        out = np.zeros((2, 7))
        with np.errstate(divide='ignore', invalid='ignore'):
            if poses is not None:                                          # test_disp.py:130-138
                disp = torch.from_numpy(poses)[:, :3].norm(2, 1).numpy()
                assert np.array_equal(disp, DC.OD.pose_norms(poses)), 'torch and the correctly rounded norm differ'
                displacements = np.array(displacements)                    # sample['displacements'], fp64
                scale_factors = [s1 / s2 for s1, s2 in zip(displacements, disp) if s1 > 0]
                scale_factor = np.mean(scale_factors) if len(scale_factors) > 0 else 0
                out[0] = test_disp.compute_errors(gt_m, pred_m * scale_factor)
            scale_factor = np.median(gt_m) / np.median(pred_m)             # :140-141
            out[1] = test_disp.compute_errors(gt_m, pred_m * scale_factor)
        d[name + '_gt_idx'], d[name + '_gt_val'] = DC.sparse(gt)
        d[name + '_shape'], d[name + '_pred'], d[name + '_crop'] = np.array(gt.shape), pred, np.array(crop)
        d[name + '_lo'], d[name + '_hi'] = np.array(lo), np.array(hi)
        d[name + '_mask'] = np.packbits(mask.ravel())
        if poses is not None:
            d[name + '_poses'], d[name + '_displacements'] = poses, np.asarray(displacements, np.float64)
        d[name + '_out'] = out
        error_cases.append(name)
        return mask, out

    for name, (H, W) in (('eigen_odd', (48, 150)), ('eigen_even', (48, 150))):
        while True:
            gt, pred = DC.error_inputs(rs, H, W)
            mask = kitti.generate_mask(gt, 1e-3, 80.0)
            if (mask.sum() % 2 == 1) == (name == 'eigen_odd'):
                break
        errors(name, gt, pred, 'eigen', poses(4), [0.7, 0.0, 1.3, 0.2])
    gt, pred = DC.error_inputs(rs, 40, 60)
    errors('stillbox', gt, pred, 'stillbox', poses(2), [0.4, 0.9])
    gt, pred = DC.error_inputs(rs, 30, 50)
    _, out = errors('zero_scale', gt, pred, 'eigen', poses(3), [0.0, -1.0, 0.0])
    assert out[0, 0] == 1.0 and np.isinf(out[0, 3]) and not out[0, 4:].any(), out
    gt, pred = DC.error_inputs(rs, 30, 50)
    errors('nopose', gt, pred, 'stillbox')
    d['velo_cases'], d['error_cases'] = np.array(velo_cases), np.array(error_cases)
    MG.save('depth_eval_small', d)


if __name__ == '__main__':
    gen()
