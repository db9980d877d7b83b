#!/usr/bin/env python
"""Generate tests/golden/train_data_small.npz from the UNMODIFIED reference datasets/sequence_folders.py,
datasets/stacked_sequence_folders.py, datasets/validation_folders.py and logger.py (AverageMeter).  Run:
python tests/golden/make_train_data.py   (the reference checkout is found as in make_golden.py; the other fixtures are
not touched; a rerun rebuilds the file byte for byte).

Stand-ins for modules the reference imports: scipy.misc (imread, gone from scipy: Pillow's decoder, which scipy's used),
path (path.Path as the loaders use it: a str with `/`, files(pattern), dirs(), dirname(), name, isfile()), blessings and
progressbar (logger's terminal output, not used by AverageMeter).

Contents:
  tree_names, tree_<i>       the data tree (tests/train_cases.tree_files): relative paths and their bytes
  seq<seed>_frames, _K       SequenceFolder(seq, seed, train=True, sequence_length=5).samples for seeds 0 and 3: per sample
                             [tgt, refs...] relative to the root, and the intrinsics
  seqval_frames, _K          the same with train=False, seed 0
  stacked_files, _K          the stacked SequenceFolder's samples (stacked/), in order
  stacked0_frames            its sample 0 decoded and split: uint8 [5,H,W,3] in [tgt, refs...] order (the float32 frames of
                             load_as_float hold integers)
  val_imgs, val_depth        ValidationSet(seq).imgs / .depth relative to the root
  val0_img, val0_depth       ValidationSet(seq)[0] without a transform (uint8 / float32)
  seq0_<i>_frames, _K, _Kinv SequenceFolder(seq, 0)[i] without a transform for i = 0, 1: uint8 [5,H,W,3], K, its inverse
  meter_in, meter_avg        AverageMeter(i=6) over 5 updates of six 0-dim float32 tensors: inputs [5,6], averages [6]
  meter_str                  str() of the meter's first average (what the summary csv holds for it)
  csv_full, csv_summary      bytes the reference's csv.writer calls (train.py:321-323,574-576 and :317-319,415-417) write
                             for the rows in csv_full_rows (the third column the int 0 in its second row) and for
                             [train_loss, meter avg[0]]"""
import csv
import io
import os
import sys
import tempfile
import types
import fnmatch
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG                      # noqa: E402  (reference import path, save helpers)
from tests import train_cases as TC           # noqa: E402


class _Absent(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith('__'):
            raise AttributeError(name)
        return _Absent(self.__name__ + '.' + name)


class _Path(str):
    def __truediv__(self, other):
        return _Path(os.path.join(self, other))

    def files(self, pattern='*'):
        return [_Path(os.path.join(self, f)) for f in os.listdir(self)
                if os.path.isfile(os.path.join(self, f)) and fnmatch.fnmatch(f, pattern)]

    def dirs(self):
        return [_Path(os.path.join(self, f)) for f in os.listdir(self) if os.path.isdir(os.path.join(self, f))]

    def dirname(self):
        return _Path(os.path.dirname(self))

    @property
    def name(self):
        return os.path.basename(self)

    def isfile(self):
        return os.path.isfile(self)


def _imread(path):
    from PIL import Image
    return np.asarray(Image.open(path))


def import_reference():
    misc = types.ModuleType('scipy.misc')
    misc.imread = _imread
    path = types.ModuleType('path')
    path.Path = _Path
    stand_ins = {'scipy.misc': misc, 'path': path, 'blessings': _Absent('blessings'), 'progressbar': _Absent('progressbar')}
    import scipy
    saved = {m: sys.modules[m] for m in stand_ins if m in sys.modules}
    had_misc = hasattr(scipy, 'misc')
    sys.modules.update(stand_ins)
    try:
        from datasets import sequence_folders, stacked_sequence_folders, validation_folders
        import logger
    finally:
        for m in stand_ins:
            del sys.modules[m]
        sys.modules.update(saved)
        if not had_misc and hasattr(scipy, 'misc'):
            del scipy.misc
    for mod in (sequence_folders, stacked_sequence_folders, validation_folders, logger):
        assert os.path.abspath(mod.__file__).startswith(os.path.abspath(MG.REF)), mod.__file__
    return sequence_folders, stacked_sequence_folders, validation_folders, logger


def u8(a):
    a = np.asarray(a)
    assert a.dtype == np.float32 and np.array_equal(a, np.round(a)), a.dtype
    return a.astype(np.uint8)


def gen():
    import warnings
    warnings.filterwarnings('ignore')
    SF, SSF, VF, logger = import_reference()
    d = {}
    files = TC.tree_files()
    names = sorted(files)
    d['tree_names'] = np.array(names)
    for i, n in enumerate(names):
        d['tree_%d' % i] = np.frombuffer(files[n], np.uint8)
    root = TC.write_tree(tempfile.mkdtemp(), files)
    seq, stacked = os.path.join(root, 'seq'), os.path.join(root, 'stacked')
    r = lambda p: os.path.relpath(p, seq)          # noqa: E731

    for tag, seed, train in (('seq0', 0, True), ('seq3', 3, True), ('seqval', 0, False)):
        ds = SF.SequenceFolder(seq, seed=seed, train=train, sequence_length=5)
        d[tag + '_frames'] = np.array([[r(s['tgt'])] + [r(p) for p in s['ref_imgs']] for s in ds.samples])
        d[tag + '_K'] = np.stack([s['intrinsics'] for s in ds.samples])
        if tag == 'seq0':
            for i in range(2):
                tgt, refs, K, Kinv = ds[i]
                d['seq0_%d_frames' % i] = np.stack([u8(tgt)] + [u8(x) for x in refs])
                d['seq0_%d_K' % i], d['seq0_%d_Kinv' % i] = K, Kinv
    assert len(d['seq0_frames']) == 3 + 2 and not any('scene_c' in p for p in d['seq0_frames'].reshape(-1))

    ds = SSF.SequenceFolder(stacked, seed=0, train=True, sequence_length=5)
    d['stacked_files'] = np.array([os.path.relpath(s['img_stack'], stacked) for s in ds.samples])
    d['stacked_K'] = np.stack([s['intrinsics'] for s in ds.samples])
    tgt, refs, K, Kinv = ds[0]
    d['stacked0_frames'] = np.stack([u8(tgt)] + [u8(x) for x in refs])

    vs = VF.ValidationSet(seq)
    d['val_imgs'] = np.array([r(p) for p in vs.imgs])
    d['val_depth'] = np.array([r(p) for p in vs.depth])
    img, depth = vs[0]
    d['val0_img'], d['val0_depth'] = u8(img), depth

    rng = np.random.RandomState(7)
    meter_in = (rng.rand(5, 6) * 3).astype(np.float32)
    m = logger.AverageMeter(i=6)
    for row in meter_in:
        m.update([torch.tensor(v) for v in row])
    d['meter_in'] = meter_in
    d['meter_avg'] = np.array([float(a) for a in m.avg], np.float32)
    assert all(torch.is_tensor(a) and a.dim() == 0 and a.dtype == torch.float32 for a in m.avg)
    d['meter_str'] = np.array(str(m.avg[0]))

    rows = (rng.rand(3, 5) * 2).astype(np.float32)
    d['csv_full_rows'] = rows
    f = io.StringIO()
    writer = csv.writer(f, delimiter='\t')
    writer.writerow(['train_loss', 'photo_cam_loss', 'photo_flow_loss', 'explainability_loss', 'smooth_loss'])
    for k, row in enumerate(rows):
        loss, loss_1, loss_2, loss_3, loss_4 = (torch.tensor(v) for v in row)
        w2 = 0 if k == 1 else 0.1
        writer = csv.writer(f, delimiter='\t')
        writer.writerow([loss.item(), loss_1.item(), loss_2.item() if w2 > 0 else 0, loss_3.item(), loss_4.item()])
    d['csv_full'] = np.frombuffer(f.getvalue().encode(), np.uint8)
    f = io.StringIO()
    writer = csv.writer(f, delimiter='\t')
    writer.writerow(['train_loss', 'validation_loss'])
    train_loss = float(rows[0, 0]) * 4 / 4
    writer = csv.writer(f, delimiter='\t')
    writer.writerow([train_loss, m.avg[0]])
    d['csv_summary'] = np.frombuffer(f.getvalue().encode(), np.uint8)
    MG.save('train_data_small', d)


if __name__ == '__main__':
    gen()
