#!/usr/bin/env python
"""Generate tests/golden/mask_eval_small.npz from the UNMODIFIED reference test_mask.py: its own `mask_error` (:224-262) on
synthetic masks and ground truth.  Run:  python tests/golden/make_mask_eval.py   (the reference checkout is found as in
make_golden.py; the other fixtures are not touched).

test_mask.py imports tqdm, path, tensorboardX, its dataset crawler, logger and drawing helpers at module level; none of
them is used by `mask_error`, so each is replaced by an empty stand-in module for the import.  `mask_error` itself runs on
numpy and the installed scipy.ndimage.zoom.  The body of the script's sample loop (:119-156) lives inside main() and cannot
be called: like the other evaluation loops it is pinned only as a restatement (oracle/evaluate_mask.py).

Cases (<case>_pred is the mask as passed, <case>_gt names the ground truth <gt>_obj / <gt>_sem it is scored against,
<case>_out holds the six numbers returned):
  small_float, small_bool, small_const   64x128 -> 96x200: a float32 0/1 mask (what `combined` is), a bool mask (what `census`
                and `bare` are) and an all-ones mask, scored one after the other against ONE ground-truth array, as the script
                does: the reference relabels that array in place, so the second and third call see labels 0 / 1 / 255
  full_float, full_bool   256x832 -> 375x1242, the KITTI sizes of the script, each on a fresh copy of the ground truth
  nocar_bool    a semantic map without label 26: every pixel is ignored, all counts are zero
  odd_float     32x96 -> 47x150
Object maps carry instance ids 0..5 (0 on about 60 % of the pixels); semantic maps carry 26 on about a third of the pixels,
in rectangular patches."""
import os
import sys
import types
import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG                      # noqa: E402  (reference import path, save helpers)


class _Absent(types.ModuleType):
    """Stand-in for a module test_mask.py imports and mask_error does not use: any attribute is another stand-in."""

    def __getattr__(self, name):
        if name.startswith('__'):
            raise AttributeError(name)
        return _Absent(self.__name__ + '.' + name)


def import_test_mask():
    import scipy.ndimage
    unused = ['tqdm', 'path', 'tensorboardX', 'custom_transforms', 'datasets', 'datasets.validation_flow', 'logger',
              'torchvision', 'torchvision.transforms', 'flowutils', 'flowutils.flowlib', 'utils']
    added = [m for m in unused if m not in sys.modules]
    for m in added:
        sys.modules[m] = _Absent(m)
    if 'scipy.ndimage.interpolation' not in sys.modules:      # the old name of the namespace zoom lives in
        added.append('scipy.ndimage.interpolation')
        alias = types.ModuleType('scipy.ndimage.interpolation')
        alias.zoom = scipy.ndimage.zoom
        sys.modules['scipy.ndimage.interpolation'] = alias
    try:
        import test_mask
    finally:
        for m in added:
            del sys.modules[m]
    assert os.path.dirname(os.path.abspath(test_mask.__file__)) == os.path.abspath(MG.REF), test_mask.__file__
    assert test_mask.zoom is scipy.ndimage.zoom
    return test_mask


def ground_truth(rs, Hg, Wg, car=True):
    obj = (rs.randint(1, 6, size=(Hg, Wg)) * (rs.rand(Hg, Wg) > 0.6)).astype(np.uint8)
    labels = np.array([26, 7, 11] if car else [24, 7, 11], np.uint8)
    patches = labels[rs.randint(0, 3, size=((Hg + 4) // 5, (Wg + 6) // 7))]
    sem = np.kron(patches, np.ones((5, 7), np.uint8))[:Hg, :Wg]
    return obj, np.ascontiguousarray(sem)


def gen():
    RM = import_test_mask()
    rs = np.random.RandomState(41)
    d, cases = {}, []

    def truth(gt, Hg, Wg, car=True):
        d[gt + '_obj'], d[gt + '_sem'] = ground_truth(rs, Hg, Wg, car)
        if car:
            assert 0.25 < (d[gt + '_sem'] == 26).mean() < 0.42 and len(np.unique(d[gt + '_obj'])) == 6
        return gt

    def score(name, pred, gt, shared=None):
        """shared: the array the reference relabels in place (the script's gt_mask_np); a fresh copy otherwise."""
        obj = d[gt + '_obj'].copy() if shared is None else shared
        d[name + '_pred'], d[name + '_gt'] = pred.copy(), np.array(gt)
        d[name + '_out'] = np.array(RM.mask_error(obj, d[gt + '_sem'], pred), np.float64)
        cases.append(name)

    gt = truth('gt_small', 96, 200)
    shared = d[gt + '_obj'].copy()
    score('small_float', (rs.rand(64, 128) > 0.5).astype(np.float32), gt, shared)
    assert set(np.unique(shared)) == {0, 1, 255}, 'the first call must have relabelled the shared array'
    score('small_bool', rs.rand(64, 128) > 0.4, gt, shared)
    score('small_const', np.ones((64, 128), np.float32), gt, shared)
    gt = truth('gt_full', 375, 1242)
    score('full_float', (rs.rand(256, 832) > 0.5).astype(np.float32), gt)
    score('full_bool', rs.rand(256, 832) > 0.6, gt)
    score('nocar_bool', rs.rand(64, 128) > 0.5, truth('gt_nocar', 96, 200, car=False))
    assert not d['nocar_bool_out'].any()
    score('odd_float', (rs.rand(32, 96) > 0.5).astype(np.float32), truth('gt_odd', 47, 150))
    d['cases'] = np.array(cases)
    MG.save('mask_eval_small', d)


if __name__ == '__main__':
    gen()
