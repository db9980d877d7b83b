#!/usr/bin/env python
"""Developer micro-benchmark of the on-device input transforms (not bench.py): CUDA-event time per call after warm-up of
  * the train transform (cc_b200.input_pipeline.DeviceAugment: flip + scale-crop + normalise) at b4 x 5 frames x 256x832,
    rotation off / on (every sample rotated) x normalisation global / local;
  * the validation Scale (DeviceScale: imresize's contrast stretch, Pillow's BILINEAR resize, normalise) of one
    KITTI-2015-sized sample, 5 x 375x1242 -> 256x832.
The uint8 frames are on the device before the timed window (the H2D copy is not timed).  Each row reports the
algorithmic bytes (uint8 frames in + fp32 frames out) and that over the time, against the H100 SXM data sheet's
3.35 TB/s, and the time the same batch takes on the host through Pillow (or, where Pillow is not installed, through the
numpy restatement of Pillow in tests/augment_oracle.py), labelled as such.  The card's name and power limit are printed
with the numbers.  Prints one JSON document."""
import argparse
import json
import os
import random
import sys
import time
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cc_b200 import input_pipeline as CI   # noqa: E402
from oracle.make3d_eval import bytescale   # noqa: E402
from tools.card import card                # noqa: E402

PEAK_BW = 3.35e12      # H100 SXM HBM3, data sheet


def time_call(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        ts.append((a, b))
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in ts)
    return ms[len(ms) // 2], ms[0]


def host_path():
    """(rotate(im, angle), resize(im, h, w), label) on the host."""
    try:
        from PIL import Image, __version__ as v
        return (lambda im, a: np.array(Image.fromarray(im).rotate(a, resample=Image.BILINEAR)),
                lambda im, h, w: np.array(Image.fromarray(im).resize((w, h), Image.BILINEAR)),
                'host Pillow %s (single thread)' % v)
    except ImportError:
        from tests import augment_oracle as AO
        return (lambda im, a: AO.rotate_u8(im, CI.pil_rotate_affine(a, im.shape[1], im.shape[0])), AO.resize_u8,
                'host numpy restatement of Pillow (tests/augment_oracle.py), not Pillow itself')


def host_train(frames, p, rot, normalization, H, W, rotate_fn, resize_fn):
    """The reference's train transform on the host for the batch, with the host resampler (fp32 tensors out)."""
    outs = []
    for b in range(frames.shape[0]):
        imgs = [frames[b, f] for f in range(frames.shape[1])]
        if rot and p['rotate'][b]:
            imgs = [rotate_fn(im, p['angle'][b]) for im in imgs]
        if p['flip'][b]:
            imgs = [np.copy(np.fliplr(im)) for im in imgs]
        sh, sw, oy, ox = int(p['scaled_h'][b]), int(p['scaled_w'][b]), int(p['offset_y'][b]), int(p['offset_x'][b])
        imgs = [resize_fn(im, sh, sw)[oy:oy + H, ox:ox + W] for im in imgs]
        t = torch.stack([torch.from_numpy(np.transpose(im, (2, 0, 1)).copy()).float() / 255 for im in imgs])
        if normalization == 'global':
            t = (t - 0.5) / 0.5
        else:
            v = t.transpose(0, 1).contiguous().view(3, -1)
            t = (t - v.mean(1)[None, :, None, None]) / v.std(1)[None, :, None, None]
        outs.append(t)
    return outs


def host_time(fn, reps=1):
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t0) / reps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--host', type=int, default=1, help='1: also time the host path (one call per row)')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_input.py measures on a GPU; there is no CPU fallback'
    dev = torch.device('cuda:0')
    rotate_fn, resize_fn, host_label = host_path()
    res = dict(card=card(), host_path=host_label, peak_bw_TBps=PEAK_BW / 1e12, rows={})

    B, F, H, W = 4, 5, 256, 832
    rs = np.random.RandomState(0)
    frames = rs.randint(0, 256, size=(B, F, H, W, 3)).astype(np.uint8)
    dframes = torch.from_numpy(frames).to(dev)
    K = np.broadcast_to(np.array([[483.3, 0, 408.3], [0, 492.6, 118.0], [0, 0, 1]], np.float32), (B, 3, 3)).copy()
    random.seed(1)
    np.random.seed(2)
    p = CI.draw_params(B, H, W, rotate=True)
    p['rotate'][:] = True
    p['angle'][:] = rs.uniform(0, 10, B)
    alg = B * F * H * W * 3 + B * F * 3 * H * W * 4
    for rot in (False, True):
        for norm in ('global', 'local'):
            aug = CI.DeviceAugment(dev, rotate=rot, normalization=norm)
            ms, ms_min = time_call(lambda: aug(dframes, K, params=p), args.iters, args.warmup)
            row = dict(shape='%dx%dx%dx%d' % (B, F, H, W), ms=ms, min_ms=ms_min, alg_bytes=alg, GBps=alg / (ms * 1e-3) / 1e9,
                       share_of_3p35TBps=alg / (ms * 1e-3) / PEAK_BW)
            if args.host:
                row['host_ms'] = host_time(lambda: host_train(frames, p, rot, norm, H, W, rotate_fn, resize_fn))
            res['rows']['train_rotate_%s_%s' % ('on' if rot else 'off', norm)] = row

    Fv, Hs, Ws, h, w = 5, 375, 1242, 256, 832
    vframes = rs.randint(0, 256, size=(1, Fv, Hs, Ws, 3)).astype(np.uint8)
    dv = torch.from_numpy(vframes).to(dev)
    Kv = np.array([[[721.5, 0, 609.6], [0, 721.5, 172.9], [0, 0, 1]]], np.float32)
    sc = CI.DeviceScale(dev, h, w)
    ms, ms_min = time_call(lambda: sc(dv, Kv), args.iters, args.warmup)
    alg = Fv * Hs * Ws * 3 + Fv * 3 * h * w * 4
    row = dict(shape='1x%dx%dx%d->%dx%d' % (Fv, Hs, Ws, h, w), ms=ms, min_ms=ms_min, alg_bytes=alg,
               GBps=alg / (ms * 1e-3) / 1e9, share_of_3p35TBps=alg / (ms * 1e-3) / PEAK_BW)
    if args.host:
        def host_scale():
            return [(torch.from_numpy(np.transpose(resize_fn(bytescale(vframes[0, f]), h, w), (2, 0, 1)).copy()).float() / 255
                     - 0.5) / 0.5 for f in range(Fv)]
        row['host_ms'] = host_time(host_scale)
    res['rows']['valid_scale_global'] = row
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
