#!/usr/bin/env python
"""Generate tests/golden/run_inference_small.npz by running the UNMODIFIED reference run_inference.py main() (with its
utils.py and models/DispNetS.py) on the folder of tests/run_inference_cases.py.
Run:  python tests/golden/make_run_inference.py   (the reference checkout is found as in make_golden.py; the other
fixtures are not touched).

Stand-ins for what the reference imports and a current stack lacks:
  scipy.misc   imread: np.asarray(Image.open(p)); imresize: scipy 1.1's bytescale of the float32 image, then Pillow's
               BILINEAR resize (oracle.make3d_eval.imresize); imsave records the array it is given and writes nothing
               (scipy 1.1's imsave raises on the script's [3,H,W] arrays, see cc_b200/run_inference.py)
  path.Path    a str with '/', files(pattern) in os.listdir order, makedirs_p, namebase and ext
  tqdm         the iterable itself;  .cuda()  a no-op (make_golden.py)
  matplotlib   matplotlib.cm and matplotlib.colors with LinearSegmentedColormap, ListedColormap and get_cmap for 'bone'
               and 'magma': the restatement in oracle/run_inference.py, NOT matplotlib itself (matplotlib is not
               installed, and cm.get_cmap was removed in 3.9).  utils.py builds magma at import; the script never uses it.
The net's forward is wrapped to record each disparity map it returns.

Contents, per run of tests/run_inference_cases.RUNS:
  <run>_stdout                 what main() printed
  <run>_disp_<k>               the k-th disparity map the net returned, [1,1,h,w] float32
  <run>_saved_names            the file of each imsave call, in call order, relative to the output folder
  <run>_saved_<k>              the uint8 [3,H,W] array of the k-th imsave call
and the stand-in colormaps' uint8 tables, table_bone [10000,3] and table_rainbow [1000,3]."""
import contextlib
import fnmatch
import io
import os
import shutil
import sys
import tempfile
import types
import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG                      # noqa: E402  (reference import path, .cuda stand-in, save helpers)
from oracle import make3d_eval as OM, run_inference as ORI   # noqa: E402
from tests import run_inference_cases as RC  # noqa: E402

REC = dict(saved=[], disp=[])


class _Path(str):
    def __truediv__(self, other):
        return _Path(os.path.join(self, other))

    def files(self, pattern='*'):
        return [_Path(os.path.join(self, f)) for f in os.listdir(self)
                if os.path.isfile(os.path.join(self, f)) and fnmatch.fnmatch(f, pattern)]

    def makedirs_p(self):
        os.makedirs(self, exist_ok=True)

    @property
    def namebase(self):
        return os.path.splitext(os.path.basename(self))[0]

    @property
    def ext(self):
        return os.path.splitext(self)[1]


def _imread(path):
    from PIL import Image
    return np.asarray(Image.open(path))


def _imresize(arr, size):
    assert arr.ndim == 3 and arr.shape[2] == 3 and len(size) == 2, (arr.dtype, arr.shape, size)
    return OM.imresize(arr, size)


def _imsave(path, arr):
    REC['saved'].append((str(path), np.array(arr)))


def stand_ins():
    import scipy
    misc = types.ModuleType('scipy.misc')
    misc.imread, misc.imresize, misc.imsave = _imread, _imresize, _imsave
    path = types.ModuleType('path')
    path.Path = _Path
    tqdm = types.ModuleType('tqdm')
    tqdm.tqdm = lambda it, *a, **k: it
    mpl = types.ModuleType('matplotlib')
    cm = types.ModuleType('matplotlib.cm')
    cm.get_cmap = ORI.get_cmap
    colors = types.ModuleType('matplotlib.colors')
    colors.LinearSegmentedColormap, colors.ListedColormap = ORI.LinearSegmentedColormap, ORI.ListedColormap
    mpl.cm, mpl.colors = cm, colors
    return scipy, {'scipy.misc': misc, 'path': path, 'tqdm': tqdm, 'matplotlib': mpl, 'matplotlib.cm': cm,
                   'matplotlib.colors': colors}


def run_reference(argv):
    """run_inference.main() with sys.argv = ['run_inference.py'] + argv, in the current directory -> its stdout."""
    scipy, mods = stand_ins()
    own = ['run_inference', 'utils']
    saved = {m: sys.modules[m] for m in list(mods) + own if m in sys.modules}
    had_misc = hasattr(scipy, 'misc')
    sys.modules.update(mods)
    scipy.misc = mods['scipy.misc']
    forward = MG.RM.DispNetS.forward

    def recording(self, x):
        out = forward(self, x)
        REC['disp'].append(out.detach().numpy().copy())
        return out
    MG.RM.DispNetS.forward = recording
    argv0 = sys.argv
    sys.argv = ['run_inference.py'] + list(argv)
    buf = io.StringIO()
    try:
        for m in own:
            sys.modules.pop(m, None)
        import run_inference
        assert os.path.dirname(os.path.abspath(run_inference.__file__)) == os.path.abspath(MG.REF)
        with contextlib.redirect_stdout(buf):
            run_inference.main()
    finally:
        sys.argv = argv0
        MG.RM.DispNetS.forward = forward
        if not had_misc:
            del scipy.misc
        for m in list(mods) + own:
            sys.modules.pop(m, None)
        sys.modules.update(saved)
    return buf.getvalue()


def gen():
    import torch
    d = {}
    cwd = os.getcwd()
    for run, argv in RC.RUNS.items():
        work = tempfile.mkdtemp()
        RC.write_work_dir(work)
        REC['saved'].clear()
        REC['disp'].clear()
        os.chdir(work)
        try:
            with torch.no_grad():
                d[run + '_stdout'] = np.array(run_reference(argv))
        finally:
            os.chdir(cwd)
        out = argv[argv.index('--output-dir') + 1]
        d[run + '_saved_names'] = np.array([os.path.relpath(p, out) for p, _ in REC['saved']])
        for k, (_, a) in enumerate(REC['saved']):
            assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[0] == 3, (a.dtype, a.shape)
            d['%s_saved_%d' % (run, k)] = a
        for k, a in enumerate(REC['disp']):
            d['%s_disp_%d' % (run, k)] = a.astype(np.float32)
        print(run, repr(str(d[run + '_stdout'])), len(REC['disp']), 'net calls', len(REC['saved']), 'imsave calls')
        shutil.rmtree(work)
    for name in ('bone', 'rainbow'):
        d['table_' + name] = ORI.uint8_table(name)
    MG.save(RC.FIXTURE, d)


if __name__ == '__main__':
    gen()
