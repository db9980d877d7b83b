#!/usr/bin/env python
"""Developer benchmark of the pose evaluation (not bench.py): pose_eval_batch over a synthetic sequence the size of KITTI
odometry 09 (1591 uint8 frames of 370x1226, so 1587 snippets of L = 5; PoseNetB6 with seeded weights, 256x832 input as
test_pose.py's defaults), in chunks of snippets (each chunk's frames stretched and resized once; neighbouring chunks share
L - 1 frames), against the reference-style host loop on a subset (per snippet: scipy 1.1's imresize restated for every
frame of the snippet, the net at batch 1, the six-vectors copied back and the numpy algebra: pose_snippet_errors).  Both
timed with a host clock around work that ends in a device synchronise, after a warm-up of every shape.  Also reports the
largest difference of the printed rows (pose_summary) over the subset.  Prints one JSON object with the card's name and
power limit, read in the same run."""
import argparse
import json
import os
import sys
import time
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cc_b200 import evaluate as CE, models as CM, synth    # noqa: E402
from oracle import make3d_eval as OM                      # noqa: E402
from tests import pose_eval_cases as PC                   # noqa: E402
from tools.card import card                               # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=1591)
    ap.add_argument('--chunk', type=int, default=128, help='snippets per pose_eval_batch call')
    ap.add_argument('--host-snippets', type=int, default=48)
    ap.add_argument('--seq-length', type=int, default=5)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    N, L, H, W, h, w = args.frames, args.seq_length, 370, 1226, 256, 832
    rs = np.random.RandomState(0)
    base = (rs.randint(0, 200, (H, W + 64, 3)) // 2 + 40).astype(np.uint8)      # a range short of 0..255: the stretch matters
    frames = np.stack([base[:, (3 * i) % 64:(3 * i) % 64 + W] + np.uint8(i % 9) for i in range(N)])
    snippets = CE._snippet_indices(N, L)
    S = len(snippets)
    gt = CE._compensate(PC.trajectory(rs, N)[snippets])
    net = synth.seeded_fill(CM.PoseNetB6(nb_ref_imgs=L - 1), 5).to(dev).eval()
    frames_h = torch.from_numpy(frames).pin_memory()
    gt_h = torch.from_numpy(gt).pin_memory()

    def device_pass(first=0, last=S):
        outs, finals = [], []
        for s in range(first, last, args.chunk):
            e = min(s + args.chunk, last)
            f0 = int(snippets[s, 0])
            fr = frames_h[f0:int(snippets[e - 1, -1]) + 1].to(dev, non_blocking=True)
            out, final = CE.pose_eval_batch(net, fr, snippets[s:e] - f0, gt_h[s:e].to(dev, non_blocking=True), 'euler', h, w)
            outs.append(out)
            finals.append(final)
        out = torch.cat(outs)
        torch.cuda.synchronize()
        return out, torch.cat(finals)

    def host_pass(n):
        out = []
        for k in range(n):
            imgs = [OM.imresize(frames[i].astype(np.float32), (h, w)) for i in snippets[k]]
            ate, re, _ = CE.pose_snippet_errors(net, imgs, gt[k], 'euler', device=dev)
            out.append((ate, re))
        torch.cuda.synchronize()
        return np.array(out)

    device_pass(0, args.chunk)
    device_pass(S - (S % args.chunk or args.chunk), S)
    host_pass(2)
    times = []
    for _ in range(3):
        t = time.perf_counter()
        got, _ = device_pass()
        times.append(time.perf_counter() - t)
    dev_s = sorted(times)[1]
    n_host = min(args.host_snippets, S)
    t = time.perf_counter()
    host = host_pass(n_host)
    host_s = time.perf_counter() - t
    got = got.cpu().numpy()
    a = CE.pose_summary(got[:n_host], n_host + L - 1).astype(np.float64)
    b = CE.pose_summary(host, n_host + L - 1).astype(np.float64)
    print(json.dumps(dict(card=card(), frames=N, snippets=S, seq_length=L, chunk=args.chunk,
                          input='%dx%d -> %dx%d, PoseNetB6' % (H, W, h, w), device_s=dev_s,
                          device_ms_per_snippet=1e3 * dev_s / S, host_snippets=n_host, host_ms_per_snippet=1e3 * host_s / n_host,
                          speedup=(host_s / n_host) / (dev_s / S), summary_device=a.tolist(), summary_host=b.tolist(),
                          summary_max_rel_diff=float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-30))))))


if __name__ == '__main__':
    main()
