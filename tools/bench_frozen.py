#!/usr/bin/env python
"""Developer benchmark of training with fixed networks (not the driver's bench.py): the README's canonical step
(cfg3 with MaskNet6 and Back2Future fixed, Trainer('cfg3', fixed=('mask', 'flow'))) against the all-four-nets cfg3 step,
at b4 256x832, both captured as CUDA graphs in one process and replayed alternately.

Reports per arm the median ms/step over the rounds with the min..max spread, triplets/s, the peak memory allocated above
what was resident before the arm was built; the Adam launch of each arm and the flow photometric forward (value-only
against full) timed with device events over many launches; and the card's name and power limit, read in the same run."""
import argparse
import json
import os
import statistics
import sys
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cc_b200 import synth, pyramid, loss_functions as CL   # noqa: E402
from cc_b200.train_step import Trainer                   # noqa: E402
from tools.card import card                              # noqa: E402

ARMS = (('cfg3', ()), ('canonical', ('mask', 'flow')))


def events_ms(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--B', type=int, default=4)
    ap.add_argument('--H', type=int, default=256)
    ap.add_argument('--W', type=int, default=832)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=20, help='timed replays per arm per round')
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--iters', type=int, default=200, help='launches per Adam / photometric timing')
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    B, H, W = args.B, args.H, args.W
    tgt, refs = synth.frames(B, H, W, seed=7)
    K, Kinv = synth.intrinsics(B, H, W)
    res = {'card': card(), 'B': B, 'H': H, 'W': W, 'rounds': args.rounds, 'steps_per_round': args.steps, 'arms': {}}

    trainers = {}
    for name, fixed in ARMS:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        tr = Trainer('cfg3', dev, seed=0, fixed=fixed)
        static = (tgt.to(dev), [r.to(dev) for r in refs], K.to(dev), Kinv.to(dev))
        tr.capture(*static)
        for _ in range(args.warmup):
            tr.replay()
        torch.cuda.synchronize()
        trainers[name] = tr
        res['arms'][name] = {'fixed': list(fixed),
                             'peak_alloc_GB': (torch.cuda.max_memory_allocated(dev) - base) / 1e9}

    times = {n: [] for n, _ in ARMS}
    for _ in range(args.rounds):
        for name, _ in ARMS:
            times[name].append(events_ms(trainers[name].replay, args.steps))
    for name, _ in ARMS:
        t = times[name]
        med = statistics.median(t)
        res['arms'][name].update(ms_per_step_median=med, ms_per_step_min=min(t), ms_per_step_max=max(t),
                                 ms_per_step_rounds=t, triplets_per_s=B / (med * 1e-3))

    # the Adam launch of each arm (one launch over all elements, or the ranges of the trained nets); the optimiser state is
    # restored afterwards
    for name, _ in ARMS:
        o = trainers[name].opt
        snap = o.snapshot()
        for _ in range(10):
            o.step()
        res['arms'][name]['adam_ms'] = events_ms(o.step, args.iters)
        res['arms'][name]['adam_ranges'] = len(o.ranges())
        o.restore(snap)
        trainers[name].refresh_weights()
    del trainers
    torch.cuda.empty_cache()

    # flow photometric forward (loss_4 of the step): full (saves the maps backward reads) against value-only
    s = synth.sample(B, H, W, seed=0, nlevels=6)
    s = {k: ([t.to(dev) for t in v] if isinstance(v, list) else v.to(dev)) for k, v in s.items()}
    ff = [f.clone().requires_grad_(True) for f in s['flow_fwd']]
    fb = [f.clone().requires_grad_(True) for f in s['flow_bwd']]
    em = [(1 - m[:, 1:3]).clone().requires_grad_(True) for m in s['emask']]
    photo = {}
    for tag, grad in (('full', True), ('value_only', False)):
        def fwd():
            with torch.set_grad_enabled(grad):
                CL.photometric_flow_loss(s['tgt'], s['refs'][1:3], [fb, ff], em, wssim=0.997)
        for _ in range(5):
            fwd()
        photo[tag + '_ms'] = events_ms(fwd, args.iters)
    pyramid.clear()
    res['flow_photometric_forward'] = photo
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
