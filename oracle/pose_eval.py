"""test_pose.py / test_sintel_pose.py's evaluation restated on numpy and torch's CPU ops: both frameworks
(kitti_eval/pose_evaluation_utils.py, sintel_eval/pose_evaluation_utils.py with sintel_io.cam_read), the snippet's pose
algebra (test_pose.py:74-86), both compute_pose_errors (test_pose.py:107-122, test_sintel_pose.py:108-121) and the printed
summary.  Snippet by snippet, as the scripts loop; tests/golden/pose_eval_small.npz holds what the reference's own code
returns for the same inputs."""
import fnmatch
import os
import warnings
import numpy as np
import torch
from oracle.geometry import pose_vec2mat


def _entries(parent, pattern, isdir):
    keep = os.path.isdir if isdir else os.path.isfile
    return [os.path.join(parent, n) for n in os.listdir(parent) if keep(os.path.join(parent, n)) and fnmatch.fnmatch(n, pattern)]


def _snippets(n, seq_length):
    demi = (seq_length - 1) // 2
    return [list(range(t - demi, t + demi + 1)) for t in range(demi, n - demi)]


def _compensated(poses):
    """One snippet's stacked poses [L,3,4]: every row minus the original first translation, then inv(R_0) @ each row."""
    poses = np.array(poses)
    t0 = poses[0, :, -1].copy()
    R0 = poses[0, :, :3].copy()
    for row in poses:
        row[:, -1] -= t0
    return np.linalg.inv(R0) @ poses


def framework(root, sequences, seq_length, sintel=False):
    """-> ([dict(name, files, snippets, gt)] in sorted sequence order, len(framework) = the image count)."""
    sub = 'clean' if sintel else 'sequences'
    dirs = sorted({d for p in sequences for d in _entries(os.path.join(root, sub), p, True)})
    seqs = []
    for d in dirs:
        name = os.path.basename(d)
        if sintel:
            files = sorted(_entries(d, '*.png', False))
            pose_list = [cam_read(c).astype(np.float32) for c in sorted(_entries(d.replace('/clean/', '/camdata_left/'), '*.cam', False))]
        else:
            files = sorted(_entries(os.path.join(d, 'image_2'), '*.png', False))
            pose_list = list(np.genfromtxt(os.path.join(root, 'poses', name + '.txt')).astype(np.float64).reshape(-1, 3, 4))
        snippets = _snippets(len(files), seq_length)
        gt = [_compensated([pose_list[i] for i in s]) for s in snippets]
        seqs.append(dict(name=name, files=files, snippets=np.array(snippets, np.int64).reshape(-1, seq_length),
                         gt=np.array(gt, np.float32 if sintel else np.float64).reshape(-1, seq_length, 3, 4)))
    return seqs, sum(len(s['files']) for s in seqs)


def cam_read(path):
    """A Sintel .cam file: the float32 tag 202021.25, the intrinsics (9 fp64), the extrinsics N (12 fp64) -> N [3,4]."""
    raw = open(path, 'rb').read()
    assert np.frombuffer(raw[:4], np.float32)[0] == 202021.25, path
    return np.frombuffer(raw[4 + 72:4 + 72 + 96], np.float64).reshape(3, 4)


def snippet_final(poses6, rotation_mode='euler'):
    """test_pose.py:74-86 of one snippet: the net's [L-1,6] fp32 six-vectors -> final poses fp64 [L,3,4].  pose_vec2mat
    runs in fp32 on torch's CPU ops; everything after the cast is fp64."""
    p = torch.as_tensor(np.asarray(poses6, np.float32))
    mid = (p.shape[0] + 1) // 2
    p = torch.cat([p[:mid], torch.zeros(1, 6), p[mid:]])
    inv_t = pose_vec2mat(p, rotation_mode).numpy().astype(np.float64)
    rot = np.linalg.inv(inv_t[:, :, :3])
    tm = np.concatenate([rot, -rot @ inv_t[:, :, -1:]], axis=-1)
    final = inv_t[0, :, :3] @ tm
    final[:, :, -1:] += inv_t[0, :, -1:]
    return final


def _re_terms(gt, pred):
    for g, p in zip(gt, pred):
        R = g[:, :3] @ np.linalg.inv(p[:, :3])
        yield np.arctan2(np.linalg.norm([R[0, 1] - R[1, 0], R[1, 2] - R[2, 1], R[0, 2] - R[2, 0]]), np.trace(R) - 1)


def pose_error(gt, pred):
    """test_pose.py compute_pose_error: (ATE, RE) of gt and pred [L,3,4].  No translation predicted: ATE is 0/0, NaN."""
    L = gt.shape[0]
    with np.errstate(divide='ignore', invalid='ignore'), warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)
        k = np.sum(gt[:, :, -1] * pred[:, :, -1]) / np.sum(pred[:, :, -1] ** 2)
        ate = np.linalg.norm((gt[:, :, -1] - k * pred[:, :, -1]).reshape(-1))
    return ate / L, sum(_re_terms(gt, pred)) / L


def sintel_pose_error(gt, pred):
    """test_sintel_pose.py compute_pose_error: RE alone (float32 gt promoted against the fp64 prediction)."""
    return sum(_re_terms(gt, pred)) / gt.shape[0]


def summary(per_snippet, n_rows, sintel=False):
    """The printed mean and std rows: [2,2] (ATE, RE), or [2,1] (RE) for Sintel, float32 over n_rows rows, the rest zero."""
    per_snippet = np.asarray(per_snippet, np.float64).reshape(-1, 2)
    errors = np.zeros((n_rows, 1 if sintel else 2), np.float32)
    for j, row in enumerate(per_snippet):
        errors[j] = row[1:] if sintel else row
    return np.stack([errors.mean(0), errors.std(0)])
