#!/usr/bin/env python
"""Generate tests/golden/test_disp_small.npz by running the UNMODIFIED reference test_disp.py main() (with
kitti_eval/ and stillbox_eval/depth_evaluation_utils.py, utils.py, loss_functions.py and models/) on the KITTI raw and
Stillbox trees of tests/depth_command_cases.py.
Run:  python tests/golden/make_test_disp.py   (the reference checkout is found as in make_golden.py; the other fixtures
are not touched).

Stand-ins for what the reference imports and a current stack lacks (make_run_inference.py's, and):
  scipy.misc   imread: np.asarray(Image.open(p)); imresize: scipy 1.1's bytescale then Pillow's BILINEAR resize
  path.Path    a str with '/', dirname(), isfile(), dirs(), name and makedirs_p
  tqdm         the iterable itself;  .cuda()  a no-op (make_golden.py);  np.int  int, for generate_depth_map's
               astype(np.int) (removed from numpy)
  matplotlib   the colormap restatement of oracle/run_inference.py (NOT matplotlib itself)
The one stand-in that adds behaviour, a documented deviation (cc_b200/test_disp.py): --output-dir raises KeyError: 'hot'
in the reference, because utils.COLORMAPS has no 'hot', and would then hand Pillow [3,H,W] arrays.  Here
utils.COLORMAPS['hot'] is matplotlib's 'hot' (N = 256, oracle/eval_disp.py's segment data) and test_disp's Image is a
stand-in whose fromarray(a).save(p) records a.transpose(1, 2, 0), the H x W x 3 image the script means, and writes
nothing.  compute_errors is wrapped to record each row it returns.

Contents, per run of tests/depth_command_cases.RUNS:
  <run>_stdout          what main() printed
  <run>_errors          the script's float32 errors [2,7,len(test_files)], rebuilt from the compute_errors rows in
                        call order (row 0 then row 1 per sample with a pose net, row 1 alone without)
  <run>_predictions     predictions.npy (runs with --output-dir)
  <run>_image_names     the viz files saved, in call order, relative to viz/;  <run>_image_<k>  the k-th, uint8 HWC
and table_hot, the stand-in's 'hot' as a uint8 [256,3] table."""
import contextlib
import io
import os
import shutil
import sys
import tempfile
import types
import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG                      # noqa: E402  (reference import path, .cuda stand-in, save helpers)
import make_run_inference as MRI              # noqa: E402  (scipy.misc, path, tqdm and matplotlib stand-ins)
from oracle import eval_disp as OT            # noqa: E402
from tests import depth_command_cases as DC   # noqa: E402

REC = dict(rows=[], images=[])


class _Path(MRI._Path):
    def __truediv__(self, other):
        return _Path(os.path.join(self, other))

    def dirname(self):
        return _Path(os.path.dirname(self))

    def isfile(self):
        return os.path.isfile(self)

    def dirs(self):
        return [_Path(os.path.join(self, d)) for d in os.listdir(self) if os.path.isdir(os.path.join(self, d))]

    @property
    def name(self):
        return os.path.basename(self)


class _Saved:
    def __init__(self, arr):
        self.arr = np.asarray(arr)

    def save(self, path):
        assert self.arr.ndim == 3 and self.arr.shape[0] == 3 and self.arr.dtype == np.uint8, (self.arr.shape, self.arr.dtype)
        REC['images'].append((str(path), np.ascontiguousarray(self.arr.transpose(1, 2, 0))))


def run_reference(argv):
    """test_disp.main() with sys.argv = ['test_disp.py'] + argv, in the current directory -> its stdout."""
    scipy, mods = MRI.stand_ins()
    mods['path'].Path = _Path
    own = ['test_disp', 'utils', 'kitti_eval', 'kitti_eval.depth_evaluation_utils', 'stillbox_eval',
           'stillbox_eval.depth_evaluation_utils']
    saved = {m: sys.modules[m] for m in list(mods) + own if m in sys.modules}
    had_misc, had_int = hasattr(scipy, 'misc'), hasattr(np, 'int')
    sys.modules.update(mods)
    scipy.misc = mods['scipy.misc']
    np.int = int
    argv0 = sys.argv
    sys.argv = ['test_disp.py'] + list(argv)
    buf = io.StringIO()
    try:
        for m in own:
            sys.modules.pop(m, None)
        import test_disp
        import utils
        assert os.path.dirname(os.path.abspath(test_disp.__file__)) == os.path.abspath(MG.REF)
        utils.COLORMAPS['hot'] = OT.HOT
        test_disp.Image = types.SimpleNamespace(fromarray=_Saved)
        compute_errors = test_disp.compute_errors

        def recording(gt, pred):
            out = compute_errors(gt, pred)
            REC['rows'].append(np.array(out, np.float64))
            return out
        test_disp.compute_errors = recording
        with contextlib.redirect_stdout(buf), np.errstate(all='ignore'):
            test_disp.main()
    finally:
        sys.argv = argv0
        if not had_misc:
            del scipy.misc
        if not had_int:
            del np.int
        for m in list(mods) + own:
            sys.modules.pop(m, None)
        sys.modules.update(saved)
    return buf.getvalue()


def gen():
    import torch
    d = {}
    cwd = os.getcwd()
    for run, argv in DC.RUNS.items():
        work = tempfile.mkdtemp()
        DC.write_work_dir(work)
        REC['rows'].clear()
        REC['images'].clear()
        os.chdir(work)
        try:
            with torch.no_grad():
                d[run + '_stdout'] = np.array(run_reference(argv))
            with open(DC.opt(argv, '--dataset-list')) as f:
                n = len(f.read().splitlines())
            out = DC.opt(argv, '--output-dir')
            if out is not None:
                d[run + '_predictions'] = np.load(os.path.join(out, 'predictions.npy'))
        finally:
            os.chdir(cwd)
        per = 2 if '--pretrained-posenet' in argv else 1
        errors = np.zeros((2, 7, n), np.float32)
        for k, row in enumerate(REC['rows']):
            errors[2 - per + k % per, :, k // per] = row
        d[run + '_errors'] = errors
        if REC['images']:
            d[run + '_image_names'] = np.array([os.path.basename(p) for p, _ in REC['images']])
            for k, (_, a) in enumerate(REC['images']):
                d['%s_image_%d' % (run, k)] = a
        print(run, repr(str(d[run + '_stdout'])), len(REC['rows']), 'error rows', len(REC['images']), 'images')
        shutil.rmtree(work)
    d['table_hot'] = OT.hot_table()
    MG.save(DC.FIXTURE, d)


if __name__ == '__main__':
    gen()
