#!/usr/bin/env python
"""Developer benchmark of the KITTI-2015 flow evaluation (not bench.py): flow_eval_batch over 200 synthetic samples of
KITTI's most common size (5 uint8 frames of 375x1242 each, ground truth and object maps of that size; DispResNet6,
PoseNetB6, MaskNet6 and Back2Future with seeded weights, 256x832 input as test_flow.py's defaults), in batches, against the
reference-style host loop on a subset (per sample: scipy 1.1's imresize restated for each of the 5 frames, the nets at
batch 1, the masks in torch ops and two compute_all_epes with their .item() round-trips: flow_sample_errors).  Both timed
with a host clock around work that ends in a device synchronise, after a warm-up of every shape.  Also reports the largest
difference of the averaged row (flow_summary) over the subset.  Prints one JSON object with the card's name and power
limit, read in the same run."""
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
from tests import flow_eval_cases as FC                   # noqa: E402
from tools.card import card                               # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--samples', type=int, default=200)
    ap.add_argument('--batch', type=int, default=8, help='samples per flow_eval_batch call')
    ap.add_argument('--host-samples', type=int, default=12)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    N, Hs, Ws, h, w, B = args.samples, 375, 1242, 256, 832, args.batch
    rs = np.random.RandomState(0)
    base = (rs.randint(0, 200, (Hs, Ws + 64, 3)) // 2 + 40).astype(np.uint8)     # a range short of 0..255: the stretch matters
    frames = np.stack([np.stack([base[:, (3 * i + f) % 64:(3 * i + f) % 64 + Ws] + np.uint8((i + f) % 9) for f in range(5)])
                       for i in range(N)])
    n_gt = min(N, 16)                                   # 16 distinct ground truths and object maps, repeated
    gt = np.stack([FC.gt_flow(rs, Hs, Ws) for _ in range(n_gt)])[np.arange(N) % n_gt]
    obj = np.stack([FC.obj_ids(rs, Hs, Ws) for _ in range(n_gt)]).astype(np.float32)[np.arange(N) % n_gt]
    K = np.tile(np.array([[721.5377, 0, 609.5593], [0, 721.5377, 172.854], [0, 0, 1]], np.float32), (N, 1, 1))
    nets = [synth.seeded_fill(CM.DispResNet6(), 1), synth.seeded_fill(CM.PoseNetB6(nb_ref_imgs=4), 2),
            synth.seeded_fill(CM.MaskNet6(nb_ref_imgs=4), 3), synth.seeded_fill(CM.Back2Future(nlevels=6), 4)]
    nets = [n.to(dev).eval() for n in nets]
    frames_h, gt_h, obj_h = (torch.from_numpy(np.ascontiguousarray(a)).pin_memory() for a in (frames, gt, obj))

    def device_pass(first=0, last=N):
        outs = []
        for s in range(first, last, B):
            e = min(s + B, last)
            outs.append(CE.flow_eval_batch(*nets, frames_h[s:e].to(dev, non_blocking=True), K[s:e],
                                           gt_h[s:e].to(dev, non_blocking=True), obj_h[s:e].to(dev, non_blocking=True)))
        out = torch.cat(outs)
        torch.cuda.synchronize()
        return out

    def host_pass(n):
        out = []
        Ks, Kinv = CE.flow_intrinsics(K[:n], Hs, Ws, h, w, dev)
        for k in range(n):
            x = [torch.from_numpy(OM.imresize(f.astype(np.float32), (h, w))) for f in frames[k]]
            x = [((t.permute(2, 0, 1)[None].float() / 255 - 0.5) / 0.5).to(dev) for t in x]
            errs, _ = CE.flow_sample_errors(*nets, x[0], x[1:], Ks[k:k + 1], Kinv[k:k + 1], torch.from_numpy(gt[k:k + 1]).to(dev),
                                            torch.from_numpy(obj[k:k + 1]).to(dev))
            out.append(errs)
        torch.cuda.synchronize()
        return np.array(out)

    with torch.no_grad():
        device_pass(0, B)
        device_pass(N - (N % B or B), N)
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
    a, _ = CE.flow_summary(got[:n_host])
    b, _ = CE.flow_summary(host)
    a, b = np.array(a), np.array(b)
    print(json.dumps(dict(card=card(), samples=N, batch=B, input='5 x %dx%d -> %dx%d, Back2Future' % (Hs, Ws, h, w),
                          device_s=dev_s, device_ms_per_sample=1e3 * dev_s / N, host_samples=n_host,
                          host_ms_per_sample=1e3 * host_s / n_host, speedup=(host_s / n_host) / (dev_s / N),
                          summary_device=a.tolist(), summary_host=b.tolist(),
                          summary_max_abs_diff=float(np.max(np.abs(a - b))))))


if __name__ == '__main__':
    main()
