#!/usr/bin/env python
"""Generate tests/golden/flow_eval_small.npz from the UNMODIFIED reference datasets/validation_flow.py (ValidationFlow),
flowutils/flow_io.py (flow_read_png), loss_functions.py (compute_all_epes) and logger.py (AverageMeter).  Run:
python tests/golden/make_flow_eval.py   (the reference checkout is found as in make_golden.py; the other fixtures are not
touched).

Stand-ins for modules the reference imports: scipy.misc (imread, gone from scipy: Pillow's decoder, which scipy's used),
skimage (not used by ValidationFlow), path (path.Path as ValidationFlow uses it: a str with joinpath), png (pypng is not
installed: its Reader yields the uint16 rows recorded when tests/flow_eval_cases.py wrote the tree, as pypng yields them),
blessings and progressbar (logger's terminal output, not used by AverageMeter).

test_flow.py's sample body lives inside main(); :127-140 are written out below line by line around seeded emask, flow_cam
and flow_fwd in place of the nets.  compute_all_epes is called as the script calls it (its THRESH left at 0.5), except in
the 'thresholds' case, which passes THRESH=0.3 with a census threshold of 0.05 so that the two cannot be confused.

Contents (all names prefixed by the case):
  mixed, rigid, census, thresholds  inputs emask [1,3,h,w], cam, fwd [1,2,h,w], gt [1,3,Hg,Wg], obj [1,Hg,Wg]; outputs
                 out (the 8 numbers), mask (the combined mask [1,1,h,w]) and b2f (test_back2future.py's 4 numbers)
  kitti          256x832 -> 375x1242, inputs regenerated from their seed (flow_eval_cases.case_inputs): out, b2f and the
                 mask as packed bits (kitti_mask_bits)
  tree_*         ValidationFlow over a tree of TREE_N samples in two frame sizes (sample 2 without obj_map, ids 0..3):
                 per sample the frames as uint8 (the float32 arrays hold integers), gt, obj (with its dtype), K, Kinv;
                 the flow_noc gt of sample 0; the sample body's out and mask around tree_net_outputs(i); the
                 AverageMeter averages of out (tree_avg) and of the flow-only numbers (tree_b2f_avg)"""
import array
import os
import sys
import tempfile
import types
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG                      # noqa: E402  (reference import path, save helpers)
from tests import flow_eval_cases as FC      # noqa: E402

ROWS = {}


class _Absent(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith('__'):
            raise AttributeError(name)
        return _Absent(self.__name__ + '.' + name)


class _Reader:
    def __init__(self, fpath):
        self.img = ROWS[str(fpath)]

    def asDirect(self):
        h, w, _ = self.img.shape
        return w, h, (array.array('H', row.reshape(-1).tolist()) for row in self.img), {}


class _Path(str):
    def joinpath(self, *parts):
        return _Path(os.path.join(self, *parts))


def _imread(path):
    from PIL import Image
    return np.asarray(Image.open(path))


def import_reference():
    png = types.ModuleType('png')
    png.Reader = _Reader
    misc = types.ModuleType('scipy.misc')
    misc.imread = _imread
    path = types.ModuleType('path')
    path.Path = _Path
    stand_ins = {'png': png, 'scipy.misc': misc, 'path': path, 'skimage': _Absent('skimage'),
                 'skimage.transform': _Absent('skimage.transform'), 'blessings': _Absent('blessings'),
                 'progressbar': _Absent('progressbar'), 'torchvision': _Absent('torchvision'),
                 'torchvision.transforms': _Absent('torchvision.transforms')}
    import scipy
    saved = {m: sys.modules[m] for m in stand_ins if m in sys.modules}
    had_misc = hasattr(scipy, 'misc')
    sys.modules.update(stand_ins)
    try:
        from datasets import validation_flow
        from flowutils import flow_io
        import logger
        import loss_functions
    finally:
        for m in stand_ins:
            del sys.modules[m]
        sys.modules.update(saved)
        if not had_misc and hasattr(scipy, 'misc'):
            del scipy.misc
    for mod in (validation_flow, flow_io, logger, loss_functions):
        assert os.path.abspath(mod.__file__).startswith(os.path.abspath(MG.REF)), mod.__file__
    return validation_flow, logger, loss_functions


def script_body(compute_all_epes, explainability_mask, flow_cam, flow_fwd, flow_gt_var, obj_map_gt_var, THRESH,
                epe_THRESH=None):
    """test_flow.py:127-140, line by line (the visualisation lines dropped), at batch 1."""
    kw = {} if epe_THRESH is None else {'THRESH': epe_THRESH}
    rigidity_mask = 1 - (1-explainability_mask[:,1])*(1-explainability_mask[:,2]).unsqueeze(1) > 0.5
    rigidity_mask_census_soft = (flow_cam - flow_fwd).abs()
    rigidity_mask_census_u = rigidity_mask_census_soft[:,0] < THRESH
    rigidity_mask_census_v = rigidity_mask_census_soft[:,1] < THRESH
    rigidity_mask_census = (rigidity_mask_census_u).type_as(flow_fwd) * (rigidity_mask_census_v).type_as(flow_fwd)
    rigidity_mask_combined = 1 - (1-rigidity_mask.type_as(explainability_mask))*(1-rigidity_mask_census.type_as(explainability_mask))
    obj_map_gt_var_expanded = obj_map_gt_var.unsqueeze(1).type_as(flow_fwd)
    _epe_errors = compute_all_epes(flow_gt_var, flow_cam, flow_fwd, rigidity_mask_combined, **kw) + \
        compute_all_epes(flow_gt_var, flow_cam, flow_fwd, (1-obj_map_gt_var_expanded), **kw)
    # test_back2future.py :74-77 on the same forward flow
    b2f = compute_all_epes(flow_gt_var, flow_fwd, flow_fwd, (1-obj_map_gt_var_expanded), **kw)
    return np.array(_epe_errors, np.float64), rigidity_mask_combined.numpy(), np.array(b2f, np.float64)


def gen():
    import warnings
    warnings.filterwarnings('ignore')
    validation_flow, logger, RL = import_reference()
    d = {}
    t = lambda a: torch.from_numpy(np.asarray(a))       # noqa: E731
    for name in FC.CASES:
        T, ET = FC.CASES[name][4:6]
        ins = FC.case_inputs(name)
        out, mask, b2f = script_body(RL.compute_all_epes, *(t(a) for a in ins), T, None if ET == 0.5 else ET)
        if name == 'kitti':
            assert mask.shape == (1, 1, 256, 832) and set(np.unique(mask)) <= {0.0, 1.0}
            d['kitti_mask_bits'] = np.packbits(mask.reshape(-1).astype(np.uint8))
        else:
            for k, a in zip(('emask', 'cam', 'fwd', 'gt', 'obj'), ins):
                d[name + '_' + k] = a
            d[name + '_mask'] = mask
        d[name + '_out'], d[name + '_b2f'] = out, b2f
        frac = mask.mean()
        assert {'rigid': frac == 1, 'census': frac == 1}.get(name, 0.2 < frac < 0.9), (name, frac)

    root = tempfile.mkdtemp()
    ROWS.update(FC.write_flow_tree(root))
    for occ in ('flow_occ', 'flow_noc'):
        ds = validation_flow.ValidationFlow(root, sequence_length=5, N=FC.TREE_N, occ=occ)
        for i in range(FC.TREE_N if occ == 'flow_occ' else 1):
            tgt, refs, K, Kinv, gt, obj = ds[i]
            if occ == 'flow_noc':
                d['tree_noc_gt0'] = gt.numpy()
                continue
            frames = np.stack([tgt] + refs)
            assert frames.dtype == np.float32 and np.array_equal(frames, np.round(frames))
            d['tree_%d_frames' % i] = frames.astype(np.uint8)
            d['tree_%d_gt' % i], d['tree_%d_obj' % i], d['tree_%d_K' % i], d['tree_%d_Kinv' % i] = gt.numpy(), obj, K, Kinv
    errors, errors_b2f = logger.AverageMeter(i=8), logger.AverageMeter(i=4)
    for i in range(FC.TREE_N):
        emask, cam, fwd = FC.tree_net_outputs(i)
        out, mask, b2f = script_body(RL.compute_all_epes, t(emask), t(cam), t(fwd), t(d['tree_%d_gt' % i])[None],
                                     t(d['tree_%d_obj' % i])[None], 0.01)
        d['tree_%d_out' % i], d['tree_%d_mask' % i] = out, mask
        errors.update(list(out))
        errors_b2f.update(list(b2f))
    d['tree_avg'], d['tree_b2f_avg'] = np.array(errors.avg, np.float64), np.array(errors_b2f.avg, np.float64)
    assert d['tree_2_obj'].dtype == np.float64 and d['tree_0_obj'].dtype == np.float32
    MG.save('flow_eval_small', d)


if __name__ == '__main__':
    gen()
