#!/usr/bin/env python
"""Developer benchmark of the Make3D evaluation (not bench.py): make3d_eval_batch over 133 synthetic samples (the size of
the reference's Make3D test list: 134 files less the popped one; 852x1704 uint8 crops, 21x305 ground truth, DispResNet6
with seeded weights, 256x256 input) in batches, against the reference's host loop on the same net (scipy 1.1's imresize
restated, the net at batch 1, the prediction copied back, scipy's zoom and the numpy errors per sample).  Both timed with
a host clock around work that ends in a device synchronise, after a warm-up of every shape.  Also reports the largest
difference of the averaged rows.  Prints one JSON object with the card's name and power limit, read in the same run."""
import argparse
import json
import os
import sys
import time
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cc_b200 import evaluate as CE, models as CM, synth    # noqa: E402
from tests import make3d_eval_cases as MC                 # noqa: E402
from tools.card import card                               # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--samples', type=int, default=133)
    ap.add_argument('--batch', type=int, default=19)
    ap.add_argument('--host-samples', type=int, default=133)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    rs = np.random.RandomState(0)
    N = args.samples
    crops = np.stack([np.clip(rs.randint(0, 40, (852, 1704, 3)) + (np.arange(1704) // 8)[None, :, None] % 190 + i % 7, 0, 255)
                      for i in range(N)]).astype(np.uint8)
    gt = np.stack([MC.error_inputs(rs)[0] for _ in range(N)])
    net = synth.seeded_fill(CM.DispResNet6(), 5).to(dev).eval()
    crops_d, gt_d = torch.from_numpy(crops).pin_memory(), torch.from_numpy(gt).pin_memory()

    def device_pass():
        outs = []
        for s in range(0, N, args.batch):
            c = crops_d[s:s + args.batch].to(dev, non_blocking=True)
            g = gt_d[s:s + args.batch].to(dev, non_blocking=True)
            outs.append(CE.make3d_eval_batch(net, c, g))
        out = torch.cat(outs)
        torch.cuda.synchronize()
        return out

    def host_pass(n):
        return np.stack([MC.host_sample_errors(net, crops[i], gt[i], 256, 256, dev) for i in range(n)])

    device_pass()
    host_pass(2)
    times = []
    for _ in range(3):
        t = time.perf_counter()
        got = device_pass()
        times.append(time.perf_counter() - t)
    dev_s = sorted(times)[1]
    n_host = min(args.host_samples, N)
    t = time.perf_counter()
    host = host_pass(n_host)
    host_s = time.perf_counter() - t
    got = got.cpu().numpy()
    a, b = CE.depth_summary(got[:n_host])[1].astype(np.float64), CE.depth_summary(host)[1].astype(np.float64)
    print(json.dumps(dict(card=card(), samples=N, batch=args.batch, input='852x1704 -> 256x256, gt 21x305, DispResNet6',
                          device_ms_per_sample=1e3 * dev_s / N, host_ms_per_sample=1e3 * host_s / n_host,
                          speedup=(host_s / n_host) / (dev_s / N), summary_device=a.tolist(), summary_host=b.tolist(),
                          summary_max_rel_diff=float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-30))))))


if __name__ == '__main__':
    main()
