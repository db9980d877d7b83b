#!/usr/bin/env python
"""Developer benchmark of FlowNetC6 (not bench.py):
  * the dilated 21x21 cost volume alone at [4,256,32,104] (conv3 of a b4 256x832 frame): forward and backward (both input
    gradients) with CUDA events over many launches, FLOP/s from shapes (2 B 441 h w C per forward, twice that backward);
  * the captured cfg3 training step at b4 256x832 with --flownet FlowNetC6 and with Back2Future, replays of the two
    graphs alternated in rounds within this one process.
Prints one JSON object with the card's name and power limit, read in the same run."""
import argparse
import json
import os
import sys
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cc_b200 import nn as cnn, synth, pyramid   # noqa: E402
from cc_b200.train_step import Trainer           # noqa: E402
from tools.card import card                      # noqa: E402


def time_loop(fn, launches):
    """Median over 5 windows of `launches` back-to-back calls, ms per call."""
    ts = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / launches)
    return sorted(ts)[2]


def bench_corr(dev, launches):
    B, C, h, w = 4, 256, 32, 104
    g = torch.Generator(device=dev).manual_seed(0)
    f1 = torch.randn(B, C, h, w, device=dev, generator=g).requires_grad_(True)
    f2 = torch.randn(B, C, h, w, device=dev, generator=g).requires_grad_(True)
    go = torch.randn(B, 441, h, w, device=dev, generator=g)
    out = cnn.corr441d(f1, f2)
    for _ in range(3):
        torch.autograd.grad(cnn.corr441d(f1, f2), [f1, f2], go)
    with torch.no_grad():
        t_f = time_loop(lambda: cnn.corr441d(f1, f2), launches)
    t_b = time_loop(lambda: torch.autograd.grad(out, [f1, f2], go, retain_graph=True), launches)
    flop = 2.0 * B * 441 * h * w * C
    return dict(shape=[B, C, h, w], fwd_ms=t_f, bwd_ms=t_b, fwd_TFLOPs=flop / (t_f * 1e-3) / 1e12,
                bwd_TFLOPs=2 * flop / (t_b * 1e-3) / 1e12)


def bench_steps(dev, rounds, replays):
    B, H, W = 4, 256, 832
    tgt, refs = synth.frames(B, H, W, seed=0)
    K, Kinv = synth.intrinsics(B, H, W)
    trainers = {}
    for name in ('FlowNetC6', 'Back2Future'):
        tr = Trainer('cfg3', dev, flownet=name)
        static = [t.to(dev) for t in [tgt] + refs + [K, Kinv]]
        tr.capture(static[0], static[1:5], static[5], static[6])
        trainers[name] = tr
    times = {n: [] for n in trainers}
    for _ in range(rounds):
        for n, tr in trainers.items():
            tr.replay()                                     # settle after switching graphs
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(replays):
                tr.replay()
            b.record()
            torch.cuda.synchronize()
            times[n].append(a.elapsed_time(b) / replays)
    pyramid.clear()
    return {n: dict(step_ms_median=sorted(t)[len(t) // 2], step_ms_min=min(t), rounds=[round(x, 3) for x in t])
            for n, t in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--launches', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--replays', type=int, default=5)
    ap.add_argument('--out', default=None, help='also write the JSON here')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_flownetc6 measures on the GPU'
    dev = torch.device('cuda:0')
    res = dict(card=card(), corr441d=bench_corr(dev, args.launches),
               cfg3_b4_256x832=bench_steps(dev, args.rounds, args.replays))
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(s + '\n')


if __name__ == '__main__':
    main()
