#!/usr/bin/env python
"""Generate tests/golden/pose_eval_small.npz from the UNMODIFIED reference test_pose.py and test_sintel_pose.py (their
compute_pose_errors), kitti_eval/pose_evaluation_utils.py and sintel_eval/pose_evaluation_utils.py (both frameworks),
sintel_eval/sintel_io.py (cam_read) and inverse_warp.py (pose_vec2mat).  Run:  python tests/golden/make_pose_eval.py
(the reference checkout is found as in make_golden.py; the other fixtures are not touched).

Stand-ins for what the modules import and this fixture does not exercise or that modern packages lack:
  scipy.misc   imread: Pillow's decode as an array (the tree holds 8-bit RGB PNGs); imresize: make_make3d_eval's
               restatement of scipy 1.1 (no frame is resized here: the nets are not run)
  path         Path, a str with '/', dirs(pattern) / files(pattern) (fnmatch on the entry names, in os.listdir order),
               name, and replace returning a Path
  tqdm, models stand-ins (tqdm(x) is x)
  numpy        on the KITTI utils module only, a proxy whose stack accepts the generator that module passes (numpy 2.3
               raises TypeError on it); every other name is numpy's.
The scripts' main-loop bodies (test_pose.py:50-92, test_sintel_pose.py:55-97) live inside main(); they are written out
below line by line around the reference's pose_vec2mat and compute_pose_error, with seeded six-vectors in place of the
pose net's output.

Frameworks (a tree from tests/pose_eval_cases.write_pose_tree; KITTI patterns '0*', '01' at seq_length 5, Sintel
'alley_1' at 3): <kind>_n_rows (len(framework)), <kind>_order (the reference's sequence order: the hash order of a set,
the same on every run because the generator runs under PYTHONHASHSEED=0 on a tree at a fixed path), <kind>_names
(sorted), per sequence <kind>_<name>_files (base names), _snippets, _gt (compensated poses as the generator
yields them: fp64 for KITTI, float32 for Sintel), _poses6 (the six-vectors fed), _final, _errors ((ATE, RE) for KITTI, RE
for Sintel); <kind>_imgs0 (the first sample's frames), <kind>_summary (the printed mean and std rows) and
<kind>_predictions (the --output-dir array), both in the reference's order.
Algebra cases <mode>_L<L> (euler, quat at L = 3 and 5) and zero_t (no translation: ATE is 0/0, NaN): _mode, _poses6
[S,L-1,6] fp32, _gt [S,L,3,4] fp64, _final, _out [S,2]."""
import os
import shutil
import sys
import tempfile
import types
import warnings
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG                      # noqa: E402  (reference import path, save helpers)
from make_mask_eval import _Absent            # noqa: E402
from make_make3d_eval import imresize         # noqa: E402
from tests import pose_eval_cases as PC       # noqa: E402


def imread(path):
    from PIL import Image
    return np.array(Image.open(path))


class Path(str):
    """path.Path as the frameworks use it."""

    def __truediv__(self, other):
        return Path(os.path.join(self, other))

    def _entries(self, pattern, keep):
        import fnmatch
        return [Path(os.path.join(self, n)) for n in os.listdir(self) if keep(os.path.join(self, n)) and fnmatch.fnmatch(n, pattern)]

    def dirs(self, pattern='*'):
        return self._entries(pattern, os.path.isdir)

    def files(self, pattern='*'):
        return self._entries(pattern, os.path.isfile)

    @property
    def name(self):
        return os.path.basename(self)

    def replace(self, old, new):
        return Path(str.replace(self, old, new))


class _NumpyAcceptingGenerators(types.ModuleType):
    """numpy, with stack taking any iterable as numpy < 1.24 did."""

    def __init__(self):
        super().__init__('numpy')

    def __getattr__(self, name):
        return getattr(np, name)

    @staticmethod
    def stack(arrays, *args, **kw):
        return np.stack(list(arrays), *args, **kw)


def import_reference():
    misc = types.ModuleType('scipy.misc')
    misc.imread, misc.imresize = imread, imresize
    path = types.ModuleType('path')
    path.Path = Path
    tqdm = types.ModuleType('tqdm')
    tqdm.tqdm = lambda x, *a, **k: x
    stand_ins = {'scipy.misc': misc, 'path': path, 'tqdm': tqdm, 'models': _Absent('models')}
    saved = {m: sys.modules[m] for m in stand_ins if m in sys.modules}
    sys.modules.update(stand_ins)
    try:
        import test_pose
        import test_sintel_pose
        from kitti_eval import pose_evaluation_utils as kitti_utils
        from sintel_eval import pose_evaluation_utils as sintel_utils
        from sintel_eval import sintel_io
    finally:
        for m in stand_ins:
            del sys.modules[m]
        sys.modules.update(saved)
    for mod in (test_pose, test_sintel_pose, kitti_utils, sintel_utils, sintel_io):
        assert os.path.abspath(mod.__file__).startswith(os.path.abspath(MG.REF) + os.sep), mod.__file__
    assert test_pose.pose_vec2mat is test_sintel_pose.pose_vec2mat and sintel_utils.cam_read is sintel_io.cam_read
    kitti_utils.np = _NumpyAcceptingGenerators()
    return test_pose, test_sintel_pose, kitti_utils, sintel_utils


def main_loop_body(ref, poses, rotation_mode):
    """test_pose.py:74-86 (test_sintel_pose.py:79-91 is the same), with `poses` the net's [1,L-1,6] output."""
    from torch.autograd import Variable
    imgs = [None] * (poses.shape[1] + 1)
    poses = poses.cpu().data[0]
    poses = torch.cat([poses[:len(imgs)//2], torch.zeros(1,6).float(), poses[len(imgs)//2:]])

    inv_transform_matrices = ref.pose_vec2mat(Variable(poses), rotation_mode=rotation_mode).data.numpy().astype(np.float64)

    rot_matrices = np.linalg.inv(inv_transform_matrices[:,:,:3])
    tr_vectors = -rot_matrices @ inv_transform_matrices[:,:,-1:]

    transform_matrices = np.concatenate([rot_matrices, tr_vectors], axis=-1)

    first_inv_transform = inv_transform_matrices[0]
    final_poses = first_inv_transform[:,:3] @ transform_matrices
    final_poses[:,:,-1:] += first_inv_transform[:,-1:]
    return final_poses


def gen():
    TP, TS, KU, SU = import_reference()
    rs = np.random.RandomState(17)
    d = {}
    warnings.filterwarnings('ignore', category=RuntimeWarning)

    # ---- both frameworks over a written tree, and the scripts' loops with seeded six-vectors in place of the net
    tree = os.path.join(tempfile.gettempdir(), 'ccb_pose_eval_tree')         # a fixed path: its hash orders the set
    shutil.rmtree(tree, ignore_errors=True)
    kitti_root, sintel_root = PC.write_pose_tree(tree)
    for kind, fw, seq_length, script in (
            ('kitti', KU.test_framework_KITTI(Path(kitti_root), PC.KITTI_PATTERNS, PC.KITTI_LENGTH), PC.KITTI_LENGTH, TP),
            ('sintel', SU.test_framework_Sintel(Path(sintel_root), PC.SINTEL_PATTERNS, PC.SINTEL_LENGTH), PC.SINTEL_LENGTH, TS)):
        up = 2 if kind == 'kitti' else 1                  # <seq>/image_2/*.png or <seq>/*.png
        order = [os.path.basename(os.path.abspath(os.path.join(f[0], *['..'] * up))) for f in fw.img_files]
        per_seq = {n: dict(files=np.array([os.path.basename(f) for f in files]), snippets=np.array(idx), gt=[], poses6=[],
                           final=[], errors=[]) for n, files, idx in zip(order, fw.img_files, fw.sample_indices)}
        owner = [n for n, idx in zip(order, fw.sample_indices) for _ in idx]
        # test_pose.py:44-48,50-92 / test_sintel_pose.py:49-53,55-97
        if kind == 'kitti':
            errors = np.zeros((len(fw), 2), np.float32)
        else:
            RE = np.zeros((len(fw)), np.float32)
        predictions_array = np.zeros((len(fw), seq_length, 3, 4))
        for j, sample in enumerate(fw):
            imgs = sample['imgs']
            if j == 0:
                d[kind + '_imgs0'] = np.array(imgs).astype(np.uint8)
                assert np.array_equal(d[kind + '_imgs0'], np.array(imgs))
            poses = torch.from_numpy(PC.pose_vectors(rs, 1, seq_length, 'euler'))
            final_poses = main_loop_body(script, poses, 'euler')
            predictions_array[j] = final_poses
            if kind == 'kitti':
                ATE, RE_j = script.compute_pose_error(sample['poses'], final_poses)
                errors[j] = ATE, RE_j
                err = (ATE, RE_j)
            else:
                RE_j = script.compute_pose_error(sample['poses'], final_poses)
                RE[j] = RE_j
                err = (RE_j,)
            s = per_seq[owner[j]]
            s['gt'].append(sample['poses'])
            s['poses6'].append(poses.numpy()[0])
            s['final'].append(final_poses)
            s['errors'].append(err)
        if kind == 'kitti':
            d[kind + '_summary'] = np.stack([errors.mean(0), errors.std(0)])
        else:
            d[kind + '_summary'] = np.stack([RE.mean(), RE.std()])[:, None]
        d[kind + '_predictions'] = predictions_array
        d[kind + '_n_rows'] = np.array(len(fw))
        d[kind + '_order'] = np.array(order)
        d[kind + '_names'] = np.array(sorted(order))
        for n, s in per_seq.items():
            for k in ('files', 'snippets'):
                d['%s_%s_%s' % (kind, n, k)] = s[k]
            for k in ('gt', 'poses6', 'final', 'errors'):
                d['%s_%s_%s' % (kind, n, k)] = np.array(s[k])
        assert len(fw) > sum(len(s['snippets']) for s in per_seq.values())            # the zero rows
    assert sorted(d['kitti_order']) == ['00', '01'] and d['sintel_alley_1_gt'].dtype == np.float32

    # ---- the algebra: the main-loop body and compute_pose_error on seeded snippets
    cases = []
    for name, mode, L, zero_t in [('%s_L%d' % (m, L), m, L, False) for m, L in PC.ALGEBRA] + [('zero_t', 'euler', 5, True)]:
        S = 4
        poses6 = PC.pose_vectors(rs, S, L, mode, zero_t=zero_t)
        gt = np.stack([PC.trajectory(rs, L) for _ in range(S)])
        gt = np.stack([np.linalg.inv(g[0, :, :3]) @ np.concatenate([g[:, :, :3], g[:, :, 3:] - g[0, :, 3:]], 2) for g in gt])
        final = np.stack([main_loop_body(TP, torch.from_numpy(p[None]), mode) for p in poses6])
        out = np.array([TP.compute_pose_error(g, f) for g, f in zip(gt, final)])
        d[name + '_mode'], d[name + '_poses6'], d[name + '_gt'], d[name + '_final'], d[name + '_out'] = \
            np.array(mode), poses6, gt, final, out
        cases.append(name)
        assert np.isnan(out[:, 0]).all() == zero_t and np.isfinite(out[:, 1]).all()
    d['algebra_cases'] = np.array(cases)
    MG.save('pose_eval_small', d)


if __name__ == '__main__':
    if os.environ.get('PYTHONHASHSEED') != '0':            # the reference's sequence order is a set's: fix str hashing
        os.execve(sys.executable, [sys.executable] + sys.argv, dict(os.environ, PYTHONHASHSEED='0'))
    gen()
