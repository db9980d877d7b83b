#!/usr/bin/env python
"""Generate tests/golden/make3d_eval_small.npz from the UNMODIFIED reference test_make3d.py: its test_framework (:37-74)
and compute_errors (:174-190).  Run:  python tests/golden/make_make3d_eval.py   (the reference checkout is found as in
make_golden.py; the other fixtures are not touched).

test_make3d imports cv2, path, tqdm, scipy.misc (imread / imresize, gone from scipy), utils, models and loss_functions,
and scipy.ndimage.interpolation; each gets a stand-in for the import (scipy.ndimage.interpolation an alias holding
scipy's zoom).  path.Path is a str subclass with '/', because test_framework hands root/'Test134/*.jpg' to glob.glob as
it is.  scipy.misc.imresize is scipy 1.1's, stated below from its documented behaviour (toimage -> bytescale, then
Pillow's resize); the main-loop body (:98-102 and :141-148) lives inside main() and is written out here line by line
around the reference's imresize stand-in and compute_errors.

Framework (a tree of 64 + 64 files from tests/make3d_eval_cases.write_make3d_tree): framework_length,
framework_img_files / _depth_files (base names of the paired lists), framework_<i>_tgt (uint8: the reference's float32
holds integers), _gt_depth, _mask for i in 0, 60, 61, 62.
Stretch cases (<case>_crop uint8, <case>_size (h, w), <case>_resize, <case>_stretched the bytescale of the float32 crop
where imresize runs, <case>_out the uint8 of the frame the net normalises):
  tie_0_202      range [0, 202] with 101 in it: (x - 0) * (255/202) = 127.49999 in float32 -> 127 (exact: 128)
  const          one value: cscale 0 -> 1, all zeros
  make3d_ratio   852x48 -> 256x16, the Make3D aspect ratio
  upscale        9x13 -> 20x30, range [5, 250]
  full_range     [0, 255]: the stretch is the identity
  narrow         range [100, 103]
  every_5_137    every value of [5, 137]: x * scale - cmin * scale fused into one rounding moves some of them
  same_size      already h x w: no stretch, no resize
  no_resize      --no-resize: no stretch, no resize
Error cases (<case>_gt fp64 [21,305], <case>_pred fp32 (zoomed, clipped), _lo, _hi, <case>_out [2,7] fp64, row 0 zeros):
  odd, even      odd / even mask counts; gt exactly at min_depth and max_depth (outside the mask)
  cap            the scaled prediction passes max_depth: the cap changes every entry but a1
  empty          no gt inside (min_depth, max_depth): a NaN row
summary: errors.mean(2)[1] of the script's float32 [2,7,N] array over the non-empty error cases."""
import os
import sys
import tempfile
import types
import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG                      # noqa: E402  (reference import path, save helpers)
from make_mask_eval import _Absent            # noqa: E402
from tests import make3d_eval_cases as MC     # noqa: E402


def imresize(arr, size, interp='bilinear', mode=None):
    """scipy 1.1's scipy.misc.imresize of a float array with an int-tuple size: toimage(arr) byte-scales the whole array
    (bytescale: cmin, cmax = arr.min(), arr.max(); cscale = cmax - cmin, 1 when 0; scale = 255 / cscale;
    (((arr - cmin) * scale).clip(0, 255) + 0.5).astype(uint8), numpy arithmetic in the array's float32), makes an RGB
    image of it, resizes it to (size[1], size[0]) with Pillow's filter and returns the uint8 array."""
    from PIL import Image
    assert interp == 'bilinear' and mode is None and arr.dtype == np.float32 and arr.ndim == 3 and arr.shape[2] == 3
    assert 3 not in arr.shape[:2], 'toimage would take the first axis of length 3 for the channels'
    cmin, cmax = arr.min(), arr.max()
    cscale = cmax - cmin
    if cscale == 0:
        cscale = 1
    scale = float(255 - 0) / cscale
    bytedata = (arr - cmin) * scale + 0
    bytedata = (bytedata.clip(0, 255) + 0.5).astype(np.uint8)
    assert bytedata.dtype == np.uint8
    imresize.last_bytescale = bytedata
    return np.array(Image.fromarray(bytedata, 'RGB').resize((size[1], size[0]), resample=Image.BILINEAR))


class Path(str):
    """path.Path as test_framework uses it: a str that joins with '/'."""

    def __truediv__(self, other):
        return Path(os.path.join(self, other))


def import_reference():
    import scipy.ndimage
    unused = ['cv2', 'path', 'tqdm', 'scipy.misc', 'utils', 'models', 'loss_functions']
    added = [m for m in unused if m not in sys.modules or m == 'scipy.misc']
    saved = {m: sys.modules[m] for m in added if m in sys.modules}
    for m in added:
        sys.modules[m] = _Absent(m)
    sys.modules['path'].Path = Path
    sys.modules['scipy.misc'].imresize = imresize
    if 'scipy.ndimage.interpolation' not in sys.modules:
        added.append('scipy.ndimage.interpolation')
        alias = types.ModuleType('scipy.ndimage.interpolation')
        alias.zoom = scipy.ndimage.zoom
        sys.modules['scipy.ndimage.interpolation'] = alias
    try:
        import test_make3d
    finally:
        for m in added:
            del sys.modules[m]
        sys.modules.update(saved)
    assert os.path.dirname(os.path.abspath(test_make3d.__file__)) == os.path.abspath(MG.REF), test_make3d.__file__
    assert test_make3d.imresize is imresize and test_make3d.zoom is scipy.ndimage.zoom
    return test_make3d


def gen():
    ref = import_reference()
    rs = np.random.RandomState(91)
    d = {}

    # ---- test_framework over a written tree
    root = tempfile.mkdtemp()
    MC.write_make3d_tree(root)
    fw = ref.test_framework(Path(root), 1e-3, 70.0)
    d['framework_length'] = np.array(len(fw))
    d['framework_img_files'] = np.array([os.path.basename(f) for f in fw.img_files])
    d['framework_depth_files'] = np.array([os.path.basename(f) for f in fw.depth_files])
    assert len(fw) == 63 and MC.FRAMEWORK_INDICES[-1] == len(fw) - 1
    for i in MC.FRAMEWORK_INDICES:
        s = fw[i]
        assert s['tgt'].dtype == np.float32 and np.array_equal(s['tgt'].astype(np.uint8), s['tgt'])
        d['framework_%d_tgt' % i] = s['tgt'].astype(np.uint8)
        d['framework_%d_gt_depth' % i] = s['gt_depth']
        d['framework_%d_mask' % i] = s['mask']

    # ---- stretch and resize: the main loop's :98-102 on float32 crops
    stretch = []

    def crop_case(name, crop, size, resize=True):
        tgt_img = crop.astype(np.float32)
        h, w, _ = tgt_img.shape
        imresize.last_bytescale = None
        if resize and (h != size[0] or w != size[1]):
            tgt_img = ref.imresize(tgt_img, size).astype(np.float32)
        d[name + '_crop'], d[name + '_size'], d[name + '_resize'] = crop, np.array(size), np.array(resize)
        if imresize.last_bytescale is not None:
            d[name + '_stretched'] = imresize.last_bytescale
        d[name + '_out'] = tgt_img.astype(np.uint8)
        stretch.append(name)
        return imresize.last_bytescale

    tie = rs.randint(0, 203, (20, 24, 3)).astype(np.uint8)
    tie[0, 0, 0], tie[1, 1, 1], tie[2, 2, 2], tie[5, 7, :] = 0, 202, 101, 101
    s = crop_case('tie_0_202', tie, (8, 10))
    assert s[2, 2, 2] == 127 and s[5, 7, 0] == 127
    assert int((np.float64(101) * 255 / 202) + 0.5) == 128                   # what exact arithmetic would give
    s = crop_case('const', np.full((12, 16, 3), 77, np.uint8), (6, 8))
    assert not s.any()
    crop_case('make3d_ratio', rs.randint(17, 232, (852, 48, 3)).astype(np.uint8), (256, 16))
    crop_case('upscale', rs.randint(5, 251, (9, 13, 3)).astype(np.uint8), (20, 30))
    full = rs.randint(0, 256, (16, 20, 3)).astype(np.uint8)
    full[0, 0, 0], full[0, 0, 1] = 0, 255
    s = crop_case('full_range', full, (7, 9))
    assert np.array_equal(s, full)
    crop_case('narrow', rs.randint(100, 104, (30, 40, 3)).astype(np.uint8), (16, 20))
    every = np.concatenate([np.arange(5, 138), rs.randint(5, 138, 19 * 21 * 3 - 133)]).astype(np.uint8)
    crop_case('every_5_137', rs.permutation(every).reshape(19, 21, 3), (11, 13))
    crop_case('same_size', rs.randint(30, 201, (10, 14, 3)).astype(np.uint8), (10, 14))
    crop_case('no_resize', tie, (8, 10), resize=False)
    d['stretch_cases'] = np.array(stretch)

    # ---- errors: the main loop's :141-148 around the reference's compute_errors
    errors_cases, rows = [], []

    def errors(name, gt_depth, pred_depth_zoomed, min_depth=1e-3, max_depth=70.0, cap=True):
        mask = np.logical_and(gt_depth > min_depth, gt_depth < max_depth)      # test_framework's sample['mask']
        pred_depth_zoomed = pred_depth_zoomed[mask]
        gt_depth = gt_depth[mask]
        with np.errstate(divide='ignore', invalid='ignore'):
            scale_factor = np.median(gt_depth) / np.median(pred_depth_zoomed)
            pred_depth_zoomed = scale_factor * pred_depth_zoomed
            if cap:
                pred_depth_zoomed[pred_depth_zoomed > max_depth] = max_depth
            out = np.zeros((2, 7))
            out[1] = ref.compute_errors(gt_depth, pred_depth_zoomed)
        return out, int(mask.sum())

    def freeze(name, gt, pred, lo=1e-3, hi=70.0):
        out, n = errors(name, gt, pred, lo, hi)
        d[name + '_gt'], d[name + '_pred'], d[name + '_lo'], d[name + '_hi'], d[name + '_out'] = gt, pred, np.array(lo), \
            np.array(hi), out
        errors_cases.append(name)
        return out, n

    for name in ('odd', 'even'):
        while True:
            gt, pred = MC.error_inputs(rs, k=0.6)
            n = int(((gt > 1e-3) & (gt < 70.0)).sum())
            if (n % 2 == 1) == (name == 'odd'):
                break
        out, _ = freeze(name, gt, pred)
        rows.append(out)
    gt, pred = MC.error_inputs(rs, k=0.3)
    out, _ = freeze('cap', gt, pred)
    rows.append(out)
    uncapped, _ = errors('cap', gt, pred, cap=False)
    assert (out[1, :4] != uncapped[1, :4]).all(), (out, uncapped)
    gt, pred = MC.error_inputs(rs)
    gt = np.where(gt > 0, 90.0, 0.0)
    gt[3, 4], gt[5, 6] = 1e-3, 70.0
    out, n = freeze('empty', gt, pred)
    assert n == 0 and np.isnan(out[1]).all() and not out[0].any()
    d['error_cases'] = np.array(errors_cases)
    script = np.zeros((2, 7, len(rows)), np.float32)                         # test_make3d.py:90,148,150
    for j, r in enumerate(rows):
        script[1, :, j] = r[1]
    d['summary'] = script.mean(2)[1]
    MG.save('make3d_eval_small', d)


if __name__ == '__main__':
    gen()
