#!/usr/bin/env python
"""Generate tests/golden/augment_small.npz from the UNMODIFIED reference custom_transforms.py on uint8 frames.
Run:  python tests/golden/make_augment.py   (the reference checkout is found as in make_golden.py; the other fixtures are
not touched).

scipy.misc (removed from scipy) is stubbed with its historical implementations (scipy 1.1 misc/pilutil.py):
imrotate(arr, angle) = Image.rotate(angle, resample=BILINEAR), imresize(arr, size) = Image.resize((size[1], size[0]),
BILINEAR), both on the uint8 frames.  Every call is recorded, so the raw rotated / resized uint8 images are frozen as well.

Contents (random uint8 frames: every neighbour differs, the hardest case for a resampler):
  rot_*    (a) Compose([RandomRotate, RandomHorizontalFlip, ArrayToTensor, Normalize(.5, .5)]), B=4 x F=3 x 20x32;
           the seeds make some samples rotate and some not; rot_angle is the angle each sample was rotated by (nan: not
           rotated) and rot_u8 the imrotate outputs (the input frames for samples not rotated)
  full_*   (b) the flow-training transform Compose([RandomRotate, RandomHorizontalFlip, RandomScaleCrop, ArrayToTensor,
           Normalize]) (train.py:178-185) on the same frames
  loc_*    (c) (a) with NormalizeLocally; loc_stats [B,3,2] is the reference's per-sample mean / std (custom_transforms.py:37-39)
  down_* / up_*  (d) Scale(h, w) + ArrayToTensor + Normalize (train.py:189-190) at a KITTI-like x0.68 downscale
           (47x155 -> 32x104) and at an upscale (20x32 -> 27x45), B=2 x F=3; *_u8 are the imresize outputs
  angles_u8 imrotate of one 17x29 frame at fixed angles (angles_deg), including small ones whose border rows and columns
           are clamped and large ones with a wide fill region."""
import os
import random
import sys
import types
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG                      # noqa: E402  (reference import path, save helpers)
from PIL import Image                         # noqa: E402

CALLS = {'rotate': [], 'resize': []}


def _imrotate(arr, angle):
    out = np.array(Image.fromarray(arr).rotate(angle, resample=Image.BILINEAR))
    CALLS['rotate'].append((float(angle), out))
    return out


def _imresize(arr, size):
    out = np.array(Image.fromarray(arr).resize((size[1], size[0]), resample=Image.BILINEAR))
    CALLS['resize'].append(out)
    return out


misc = types.ModuleType('scipy.misc')
misc.imrotate, misc.imresize = _imrotate, _imresize
sys.modules['scipy.misc'] = misc
import scipy                                  # noqa: E402
scipy.misc = misc
import custom_transforms as CT                # noqa: E402

B, F, HS, WS = 4, 3, 20, 32
SEEDS = dict(rot=(11, 21), full=(13, 33), loc=(11, 21))     # (random.seed, np.random.seed) per case; (c) reuses (a)'s
K = np.array([[30.5, 0, 16.2], [0, 31.5, 10.1], [0, 0, 1]], np.float32)
NORM = CT.Normalize(mean=[0.5, 0.5, 0.5], std=[0.5, 0.5, 0.5])
ANGLES = [0.05, 0.7, 3.3, 7.3, 9.95]


def run(tf, frames, seeds):
    """tf per sample, as the dataset calls it: -> (outputs [B,F,3,H,W], K [B,3,3], rotation angle per sample, rotated u8)."""
    random.seed(seeds[0])
    np.random.seed(seeds[1])
    outs, Ks, angles, rot = [], [], [], np.array(frames)
    for b in range(frames.shape[0]):
        n0 = len(CALLS['rotate'])
        imgs, Kb = tf([frames[b, f] for f in range(frames.shape[1])], np.copy(K))
        calls = CALLS['rotate'][n0:]
        assert len(calls) in (0, frames.shape[1])
        angles.append(calls[0][0] if calls else np.nan)
        for f, (_, im) in enumerate(calls):
            rot[b, f] = im
        outs.append(torch.stack(imgs))
        Ks.append(torch.from_numpy(np.asarray(Kb, np.float32)))
    return torch.stack(outs), torch.stack(Ks), np.array(angles), rot


def gen():
    rs = np.random.RandomState(31)
    frames = rs.randint(0, 256, size=(B, F, HS, WS, 3)).astype(np.uint8)
    d = dict(frames=frames, K=K)
    tf_a = CT.Compose([CT.RandomRotate(), CT.RandomHorizontalFlip(), CT.ArrayToTensor(), NORM])
    out, Ko, ang, rot = run(tf_a, frames, SEEDS['rot'])
    assert 0 < np.isfinite(ang).sum() < B, 'the seeds must rotate some samples and leave others'
    d.update(rot_out=out, rot_K=Ko, rot_angle=ang, rot_u8=rot, rot_seeds=np.array(SEEDS['rot']))
    tf_b = CT.Compose([CT.RandomRotate(), CT.RandomHorizontalFlip(), CT.RandomScaleCrop(), CT.ArrayToTensor(), NORM])
    out, Ko, ang, _ = run(tf_b, frames, SEEDS['full'])
    assert 0 < np.isfinite(ang).sum() < B
    d.update(full_out=out, full_K=Ko, full_angle=ang, full_seeds=np.array(SEEDS['full']))
    tf_c = CT.Compose([CT.RandomRotate(), CT.RandomHorizontalFlip(), CT.ArrayToTensor(), CT.NormalizeLocally()])
    out, Ko, ang, _ = run(tf_c, frames, SEEDS['loc'])
    tf_c0 = CT.Compose([CT.RandomRotate(), CT.RandomHorizontalFlip(), CT.ArrayToTensor()])
    unit, _, _, _ = run(tf_c0, frames, SEEDS['loc'])
    stats = []
    for b in range(B):                        # custom_transforms.py:37-39 on the same frames
        v = unit[b].transpose(0, 1).contiguous().view(3, -1)
        stats.append(torch.stack([v.mean(1), v.std(1)], 1))
    d.update(loc_out=out, loc_K=Ko, loc_angle=ang, loc_stats=torch.stack(stats), loc_seeds=np.array(SEEDS['loc']))
    for name, (hs, ws, h, w) in (('down', (47, 155, 32, 104)), ('up', (20, 32, 27, 45))):
        fr = rs.randint(0, 256, size=(2, F, hs, ws, 3)).astype(np.uint8)
        tf_d = CT.Compose([CT.Scale(h=h, w=w), CT.ArrayToTensor(), NORM])
        CALLS['resize'].clear()
        out, Ko, _, _ = run(tf_d, fr, (0, 0))
        d.update({name + '_frames': fr, name + '_out': out, name + '_K': Ko,
                  name + '_u8': np.stack(CALLS['resize']).reshape(2, F, h, w, 3)})
    one = rs.randint(0, 256, size=(17, 29, 3)).astype(np.uint8)
    d.update(angles_frame=one, angles_deg=np.array(ANGLES), angles_u8=np.stack([misc.imrotate(one, a) for a in ANGLES]))
    MG.save('augment_small', d)


if __name__ == '__main__':
    gen()
