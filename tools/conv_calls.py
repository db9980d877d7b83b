#!/usr/bin/env python
"""Where the convolution time of one training step at the benchmark's size goes.

python tools/conv_calls.py [cfg] [top]
    every convolution call of one eager training step with the kernel it dispatched to and its CUDA-event time (helpers
    of the call and the host gaps between its launches included), per kernel and per layer.
python tools/conv_calls.py --isolated [cfg] [top] [--reps R]
    every distinct (op, shape) call of the step replayed on its own R times between CUDA events, multiplied by its count
    in the step, grouped by kernel and wgmma N.  Beside each tensor-core group: its floor, the least time the padded
    tiles the dispatcher plans (split-K, whole waves of CTAs on the SMs) take in 3 tf32 passes at the H100 SXM data-sheet
    dense TF32 rate (495 TFLOP/s).  The floor is a bound, never reached."""
import argparse
import ctypes as C
import os
import sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cc_b200 import synth, _lib, pyramid, nn as cnn     # noqa: E402
from cc_b200.train_step import Trainer                   # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('cfg', nargs='?', default='cfg3')
ap.add_argument('top', nargs='?', type=int, default=60)
ap.add_argument('--isolated', action='store_true', help='time each distinct call on its own instead of in the eager step')
ap.add_argument('--reps', type=int, default=20, help='replays of each distinct call between the events (--isolated)')
args = ap.parse_args()
B, H, W = 4, 256, 832
dev = torch.device('cuda:0')
tgt, refs = synth.frames(B, H, W, seed=1)
K, Kinv = synth.intrinsics(B, H, W)
tr = Trainer(args.cfg, dev)
step_args = (tgt.to(dev), [r.to(dev) for r in refs], K.to(dev), Kinv.to(dev))
real = _lib.lib()
OPS = {_lib.CONV_FPROP: 'fprop', _lib.CONV_DGRAD: 'dgrad', _lib.CONV_WGRAD: 'wgrad'}
TF32_FLOPS = 495e12
SMS = torch.cuda.get_device_properties(dev).multi_processor_count


def flops(shp):          # (B, Ci, Hi, Wi, Co, k, stride): algorithmic FLOP of the convolution, any op
    return 2.0 * shp[0] * shp[4] * shp[1] * shp[5] ** 2 * (shp[2] // shp[6]) * (shp[3] // shp[6])


def eager():
    records = []

    class Proxy:
        def __getattr__(self, name):
            fn = getattr(real, name)
            if not name.startswith('ccb_conv2d_'):
                return fn

            def wrapped(*a):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                rc = fn(*a)
                e.record()
                d = a[0]._obj
                records.append((name[len('ccb_conv2d_'):], (real.ccb_debug_last_conv_kernel() or b'').decode(),
                                (d.B, d.Ci, d.Hi, d.Wi, d.Co, d.kh, d.stride), s, e))
                return rc
            return wrapped

    for it in range(3):
        records.clear()
        _lib._lib = Proxy() if it == 2 else real
        pyramid.clear()
        tr.step(*step_args)
        _lib._lib = real
        torch.cuda.synchronize()
    rows = {}
    for op, kern, shp, s, e in records:
        r = rows.setdefault((op, kern, shp), [0.0, 0])
        r[0] += s.elapsed_time(e)
        r[1] += 1
    tot = sum(r[0] for r in rows.values())
    print('%d conv calls, %.2f ms (eager, events per call)' % (len(records), tot))
    by_k = {}
    for (op, kern, shp), (ms, n) in rows.items():
        k = by_k.setdefault(kern + ':' + op, [0.0, 0, 0.0])
        k[0] += ms; k[1] += n
        k[2] += n * flops(shp)
    for k, (ms, n, fl) in sorted(by_k.items(), key=lambda kv: -kv[1][0]):
        print('  %-24s %6.2f ms %5.1f%%  %3d calls  %6.1f TFLOP/s' % (k, ms, 100 * ms / tot, n, fl / ms / 1e9))
    print('top %d (op kernel B Ci HxW Co k s | calls ms us/call TFLOP/s):' % args.top)
    for (op, kern, shp), (ms, n) in sorted(rows.items(), key=lambda kv: -kv[1][0])[:args.top]:
        print('  %-5s %-16s B%d Ci%-4d %3dx%-3d Co%-4d k%d s%d | %2d %6.2f %7.1f %6.1f' % (
            (op, kern) + shp + (n, ms, 1e3 * ms / n, n * flops(shp) / ms / 1e9)))


# ---- the tensor-core floor of one call, from its shape and the dispatcher's plan (conv_tc.cu: tc_plan, tc_geometry)
def cdiv(a, b):
    return -(-a // b)


def tc_kp(ntaps, cc):    # k-tiles of 32 of `ntaps` taps of cc channels padded to 4; a class without taps runs one
    return cdiv(ntaps * cdiv(cc, 4) * 4, 32) * 32 if ntaps > 0 else 32


def wgmma_n(n):
    out = (C.c_int * 4)()
    assert real.ccb_debug_tc_plan(n, out) == 0
    return out[0]


def splits(d, op, head, numel):
    """the split-K count the dispatcher chose: its workspace is the head (prepared weights or padded copies) + the
    partials of every split when there is more than one"""
    work = _lib.call('ccb_conv_workspace_floats', d, op)
    return (work - head) // numel if work > head else 1


def launch_floor(rows, n, ktiles, nsplit):
    """seconds of one launch: whole waves of 128-row x wgmma-N CTAs, each 3 tf32 passes over its split's k-tiles"""
    waves = cdiv(cdiv(rows, 128) * cdiv(n, 128) * nsplit, SMS)
    return waves * cdiv(ktiles, nsplit) * 3 * 2.0 * 128 * wgmma_n(n) * 32 / (TF32_FLOPS / SMS)


def tc_floor(op, d):
    k, s = d.kh, d.stride
    if op == _lib.CONV_FPROP:
        kp = tc_kp(k * k, d.Ci)
        return launch_floor(d.B * d.Ho * d.Wo, d.Co, kp // 32, splits(d, op, 2 * d.Co * kp, d.B * d.Co * d.Ho * d.Wo))
    if op == _lib.CONV_DGRAD:       # one launch per stride-parity class, all with the plan's split count
        sp = splits(d, op, 2 * d.Ci * tc_kp(cdiv(k, s) ** 2, d.Co), d.B * d.Ci * d.Hi * d.Wi)
        t = 0.0
        for py in range(min(s, d.Hi)):
            for px in range(min(s, d.Wi)):
                ky0, kx0 = (py + d.pad) % s, (px + d.pad) % s
                nky, nkx = (cdiv(k - ky0, s) if k > ky0 else 0), (cdiv(k - kx0, s) if k > kx0 else 0)
                t += launch_floor(d.B * cdiv(d.Hi - py, s) * cdiv(d.Wi - px, s), d.Ci, tc_kp(nky * nkx, d.Co) // 32, sp)
        return t
    wo, wi = cdiv(d.Wo, 4) * 4, cdiv(d.Wi, 4) * 4     # a width that is not a multiple of 4 runs on padded copies
    head = 0 if wo == d.Wo else d.B * d.Ci * d.Hi * wi + d.B * d.Co * d.Ho * wo
    sp = splits(d, op, head, d.Co * d.Ci * k * k)
    return launch_floor(k * k * cdiv(d.Ci, 4) * 4, d.Co, cdiv(d.B * d.Ho * wo, 32), sp)


def isolated():
    calls = {}                  # (op, shape, act, operands present) -> [op, d, args, kernel, count]
    real_run = cnn._run

    def recording_run(op, d, *a):
        real_run(op, d, *a)
        key = (op, tuple(getattr(d, f) for f, _ in _lib.ConvDesc._fields_ if f not in ('slope', 'wcache')),
               tuple(x is None for x in a))
        c = calls.get(key)
        if c is None:           # the arguments stay referenced, so their memory outlives the step for the replays
            calls[key] = c = [op, d, a, (real.ccb_debug_last_conv_kernel() or b'').decode(), 0]
        c[4] += 1

    # the third step, as the eager mode times it: weight cache committed, Adam state warm
    for it in range(3):
        cnn._run = recording_run if it == 2 else real_run
        pyramid.clear()
        tr.step(*step_args)
        cnn._run = real_run
        torch.cuda.synchronize()
    rows = []
    for op, d, a, kern, n in calls.values():
        for _ in range(2):
            real_run(op, d, *a)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(args.reps):
            real_run(op, d, *a)
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e) / args.reps
        shp = (d.B, d.Ci, d.Hi, d.Wi, d.Co, d.kh, d.stride)
        tc = kern.startswith('conv_tc')
        nw = wgmma_n(d.Ci if op == _lib.CONV_DGRAD else d.Co) if tc else 0
        rows.append((OPS[op], kern, nw, shp, n, ms, 1e3 * tc_floor(op, d) if tc else float('nan')))
    tot = sum(r[4] * r[5] for r in rows)
    print('%s: %d conv calls, %d distinct; %.2f ms per step, each call timed alone (%d replays between CUDA events)' % (
        torch.cuda.get_device_name(dev), sum(r[4] for r in rows), len(rows), tot, args.reps))
    print('  %-16s %4s %6s %9s %7s %9s %7s %8s' % ('kernel', 'N', 'calls', 'ms/step', 'share', 'floor ms', 'floor%', 'GFLOP'))
    groups = {}
    for op, kern, nw, shp, n, ms, fl in rows:
        g = groups.setdefault((kern, nw), [0, 0.0, 0.0, 0.0])
        g[0] += n; g[1] += n * ms; g[2] += n * fl; g[3] += n * flops(shp) / 1e9
    for (kern, nw), (n, ms, fl, gf) in sorted(groups.items()):
        print('  %-16s %4s %6d %9.2f %6.1f%% %9.2f %6.1f%% %8.1f' % (
            kern, nw or '-', n, ms, 100 * ms / tot, fl, 100 * fl / ms, gf))
    print('top %d (op kernel N B Ci HxW Co k s | calls ms/step us/call floor-us/call TFLOP/s):' % args.top)
    for op, kern, nw, shp, n, ms, fl in sorted(rows, key=lambda r: -r[4] * r[5])[:args.top]:
        print('  %-5s %-13s %3s B%d Ci%-4d %3dx%-3d Co%-4d k%d s%d | %2d %6.2f %7.1f %7.1f %6.1f' % (
            (op, kern, nw or '-') + shp + (n, n * ms, 1e3 * ms, 1e3 * fl, flops(shp) / ms / 1e9)))


if args.isolated:
    isolated()
else:
    eager()
