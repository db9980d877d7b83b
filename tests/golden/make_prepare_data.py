#!/usr/bin/env python
"""Generate tests/golden/prepare_small.npz by running the UNMODIFIED reference data/prepare_train_data.py main() (with its
data/kitti_raw_loader.py, data/cityscapes_loader.py and data/test_scenes.txt) on the trees of tests/prepare_cases.py.
Run:  python tests/golden/make_prepare_data.py   (the reference checkout is found as in make_golden.py; the other
fixtures are not touched; a rerun rebuilds the file byte for byte).

Stand-ins for what the reference imports and a current stack lacks: scipy.misc as scipy 1.1 behaves on uint8 RGB frames
(imread: np.asarray(Image.open(p)); imresize: toimage passes uint8 through, then Pillow's BILINEAR resize; imsave:
Image.fromarray(a).save(p), recording a), path.Path (a str with '/', '+', files() and dirs() in listdir order,
makedirs_p, rmtree ...), joblib.Parallel / delayed run one call after another, tqdm (the iterable itself), and np.int
(removed from numpy: int).  np.save is wrapped to record each depth map it writes.  Each run is made from a working
directory holding the tree as raw/ (relative paths, see tests/prepare_cases.py) with sys.argv set to its arguments.

Contents:
  <tree>_tree_names, <tree>_tree_<i>   the raw trees' files (kitti, cityscapes) and their bytes ('/'-ended: empty folder)
per run (tests/prepare_cases.RUNS):
  <run>_files                          the dump's files after the run, sorted
  <run>_cam_names, <run>_cam_text      each cam.txt and its text
  <run>_jpg_names, <run>_jpg_<i>       each jpg and the uint8 frame imsave was given for it
  <run>_npy_names, <run>_npy_<i>       each depth map np.save wrote in a folder that was kept (train folders' included,
                                       whose files the split deletes), float32
  <run>_order                          the folders as the split's dirs() listed them
  <run>_train, <run>_val               train.txt and val.txt"""
import fnmatch
import os
import shutil
import sys
import tempfile
import types
import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG                      # noqa: E402  (reference import path, save helpers)
from tests import prepare_cases as PC        # noqa: E402

REC = dict(jpg={}, npy={}, dirs={})


class _Path(str):
    def __truediv__(self, other):
        return _Path(os.path.join(self, other))

    def __add__(self, other):
        return _Path(str.__add__(self, other))

    def files(self, pattern='*'):
        return [_Path(os.path.join(self, f)) for f in os.listdir(self)
                if os.path.isfile(os.path.join(self, f)) and fnmatch.fnmatch(f, pattern)]

    def dirs(self):
        out = [_Path(os.path.join(self, f)) for f in os.listdir(self) if os.path.isdir(os.path.join(self, f))]
        REC['dirs'][str(self)] = [os.path.basename(p) for p in out]
        return out

    def realpath(self):
        return _Path(os.path.realpath(self))

    def dirname(self):
        return _Path(os.path.dirname(self))

    @property
    def parent(self):
        return self.dirname()

    @property
    def name(self):
        return os.path.basename(self)

    def basename(self):
        return os.path.basename(self)

    def isfile(self):
        return os.path.isfile(self)

    def mkdir_p(self):
        os.makedirs(self, exist_ok=True)

    makedirs_p = mkdir_p

    def rmtree(self):
        shutil.rmtree(self)

    def remove_p(self):
        if os.path.exists(self):
            os.remove(self)


def _imread(path):
    from PIL import Image
    return np.asarray(Image.open(path))


def _imresize(arr, size):
    from PIL import Image
    assert arr.dtype == np.uint8 and arr.ndim == 3 and arr.shape[2] == 3 and len(size) == 2, (arr.dtype, arr.shape, size)
    return np.array(Image.fromarray(arr).resize((size[1], size[0]), resample=Image.BILINEAR))


def _imsave(path, arr):
    from PIL import Image
    assert arr.dtype == np.uint8 and arr.ndim == 3 and arr.shape[2] == 3, (arr.dtype, arr.shape)
    REC['jpg'][os.path.normpath(path)] = np.array(arr)
    Image.fromarray(arr).save(path)


def _np_save(path, arr):
    REC['npy'][os.path.normpath(path)] = np.array(arr)
    _save(path, arr)


_save = np.save


class _Parallel:
    def __init__(self, n_jobs=1):
        pass

    def __call__(self, jobs):
        return [f(*a, **k) for f, a, k in jobs]


def _delayed(f):
    return lambda *a, **k: (f, a, k)


def stand_ins():
    import scipy
    misc = types.ModuleType('scipy.misc')
    misc.imread, misc.imresize, misc.imsave = _imread, _imresize, _imsave
    path = types.ModuleType('path')
    path.Path = _Path
    joblib = types.ModuleType('joblib')
    joblib.Parallel, joblib.delayed = _Parallel, _delayed
    tqdm = types.ModuleType('tqdm')
    tqdm.tqdm = lambda it, *a, **k: it
    return scipy, {'scipy.misc': misc, 'path': path, 'joblib': joblib, 'tqdm': tqdm}


def run_reference(argv):
    """prepare_train_data.main() with sys.argv = ['prepare_train_data.py'] + argv, in the current directory."""
    scipy, mods = stand_ins()
    saved = {m: sys.modules[m] for m in list(mods) + ['prepare_train_data', 'kitti_raw_loader', 'cityscapes_loader']
             if m in sys.modules}
    had_misc, had_int = hasattr(scipy, 'misc'), hasattr(np, 'int')
    data = os.path.join(MG.REF, 'data')
    sys.path.insert(0, data)
    sys.modules.update(mods)
    scipy.misc = mods['scipy.misc']
    np.int = int
    np.save = _np_save
    argv0 = sys.argv
    sys.argv = ['prepare_train_data.py'] + list(argv)
    try:
        for m in ('prepare_train_data', 'kitti_raw_loader', 'cityscapes_loader'):
            sys.modules.pop(m, None)
        import prepare_train_data
        assert os.path.dirname(os.path.abspath(prepare_train_data.__file__)) == os.path.abspath(data)
        prepare_train_data.main()
    finally:
        sys.argv = argv0
        np.save = _save
        if not had_int:
            del np.int
        if not had_misc:
            del scipy.misc
        for m in list(mods) + ['prepare_train_data', 'kitti_raw_loader', 'cityscapes_loader']:
            sys.modules.pop(m, None)
        sys.modules.update(saved)
        sys.path.remove(data)


def reference_test_scenes():
    with open(os.path.join(MG.REF, 'data', 'test_scenes.txt')) as f:
        return [t[:-1] for t in f.readlines()]


def gen():
    import warnings
    warnings.filterwarnings('ignore')
    d = {}
    trees = {'kitti': PC.kitti_tree_files(), 'cityscapes': PC.cityscapes_tree_files()}
    listed = reference_test_scenes()
    drives = {n.split('/')[2] for n in trees['kitti'] if n.count('/') > 3}
    assert PC.EXCLUDED in listed and [dr for dr in drives if dr[:-5] in listed] == [PC.EXCLUDED + '_sync'], drives
    for kind, files in trees.items():
        names = sorted(files)
        d[kind + '_tree_names'] = np.array(names)
        for i, n in enumerate(names):
            if files[n] is not None:
                d['%s_tree_%d' % (kind, i)] = np.frombuffer(files[n], np.uint8)
    cwd = os.getcwd()
    for run, argv in PC.RUNS.items():
        work = tempfile.mkdtemp()
        PC.write_run_dir(work, trees[PC.RUN_TREE[run]])
        for k in REC:
            REC[k].clear()
        os.chdir(work)
        try:
            k = argv.index('--test-scenes') if '--test-scenes' in argv else len(argv)
            run_reference(argv[:k] + argv[k + 2:])          # the reference reads its own data/test_scenes.txt
        finally:
            os.chdir(cwd)
        dump = os.path.join(work, 'dump')
        files = PC.dump_files(dump)
        d[run + '_files'] = np.array(files)
        cams = [f for f in files if f.endswith('cam.txt')]
        d[run + '_cam_names'] = np.array(cams)
        d[run + '_cam_text'] = np.array([open(os.path.join(dump, f)).read() for f in cams])
        jpgs = [f for f in files if f.endswith('.jpg')]
        assert sorted(os.path.relpath(p, 'dump') for p in REC['jpg'] if os.path.isfile(os.path.join(work, p))) == jpgs
        d[run + '_jpg_names'] = np.array(jpgs)
        for i, f in enumerate(jpgs):
            d['%s_jpg_%d' % (run, i)] = REC['jpg'][os.path.join('dump', f)]
        order = REC['dirs']['dump']
        kept = set(order)
        npys = sorted(os.path.relpath(p, 'dump') for p in REC['npy'] if os.path.relpath(p, 'dump').split('/')[0] in kept)
        d[run + '_npy_names'] = np.array(npys)
        for i, f in enumerate(npys):
            a = REC['npy'][os.path.join('dump', f)]
            assert a.dtype == np.float32, a.dtype
            d['%s_npy_%d' % (run, i)] = a
        d[run + '_order'] = np.array(order)
        for split in ('train', 'val'):
            with open(os.path.join(dump, split + '.txt')) as f:
                d['%s_%s' % (run, split)] = np.array(f.read().splitlines())
        print(run, len(order), 'folders', len(jpgs), 'jpgs', len(npys), 'depth maps; val', list(d[run + '_val']))
        assert len(order) >= 3 and len(d[run + '_val']) >= 1
        shutil.rmtree(work)
    MG.save('prepare_small', d)


if __name__ == '__main__':
    gen()
