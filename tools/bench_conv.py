#!/usr/bin/env python
"""Developer micro-benchmark: every conv layer shape of DispResNet6 / PoseNetB6 (b4, 256x832) through
libccb200 (fprop / dgrad / wgrad) next to torch/cuDNN with TF32 off and on."""
import argparse
import json
import os
import sys
import torch
import torch.nn.functional as F
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cc_b200 import nn as cnn, models as CM, _lib   # noqa: E402


def collect_shapes(net, inputs):
    shapes = []
    hooks = []

    def hook(m, inp, out):
        x = inp[0]
        shapes.append((type(m).__name__, tuple(x.shape), tuple(m.weight.shape), m.stride, m.padding,
                       getattr(m, 'output_padding', 0)))
    for m in net.modules():
        if isinstance(m, (cnn.Conv2d, cnn.ConvTranspose2d)):
            hooks.append(m.register_forward_hook(hook))
    with torch.no_grad():
        net(*inputs)
    for h in hooks:
        h.remove()
    return shapes


def timeit(fn, iters=5):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--impl', type=int, default=_lib.IMPL_AUTO, choices=(_lib.IMPL_AUTO, _lib.IMPL_FFMA, _lib.IMPL_TC),
                    help='0 auto, 1 FFMA kernels, 2 tensor-core kernels')
    ap.add_argument('--nets', default='disp,pose')
    args = ap.parse_args()
    cnn.CONV_IMPL = args.impl
    dev = torch.device('cuda:0')
    B, H, W = 4, 256, 832
    x = torch.randn(B, 3, H, W, device=dev)
    refs = [torch.randn(B, 3, H, W, device=dev) for _ in range(4)]
    shapes = []
    if 'disp' in args.nets:
        shapes += [('disp',) + s for s in collect_shapes(CM.DispResNet6().to(dev).train(), (x,))]
    if 'pose' in args.nets:
        shapes += [('pose',) + s for s in collect_shapes(CM.PoseNetB6(4).to(dev).train(), (x, refs))]
    if 'mask' in args.nets:
        shapes += [('mask',) + s for s in collect_shapes(CM.MaskNet6(4).to(dev).train(), (x, refs))]
    uniq = {}
    for s in shapes:
        uniq.setdefault(s[1:], [0, s[0]])[0] += 1
    tot = {'ours': 0.0, 'cudnn_fp32': 0.0, 'cudnn_tf32': 0.0}
    rows = []
    for key, (cnt, net) in uniq.items():
        kind, xs, ws, stride, pad, opad = key
        xin = torch.randn(*xs, device=dev, requires_grad=True)
        w = (torch.randn(*ws, device=dev) * 0.05).requires_grad_(True)
        k = ws[2]
        if kind == 'Conv2d':
            flops = 2 * xs[0] * ws[0] * ws[1] * k * k * ((xs[2] + 2 * pad - k) // stride + 1) * ((xs[3] + 2 * pad - k) // stride + 1)
            ours = lambda: cnn.conv2d(xin, w, None, None, stride, pad, None)
            ref = lambda: F.conv2d(xin, w, None, stride, pad)
        else:
            flops = 2 * xs[0] * xs[1] * ws[1] * k * k * xs[2] * xs[3]
            ours = lambda: cnn.conv_transpose2d(xin, w, None, stride, pad, opad, None)
            ref = lambda: F.conv_transpose2d(xin, w, None, stride, pad, opad)

        def fb(f):
            def run():
                y = f()
                y.backward(torch.ones_like(y))
                xin.grad = None
                w.grad = None
            return run
        t_f, t_fb = timeit(ours), timeit(fb(ours))
        torch.backends.cudnn.allow_tf32 = False
        r_f, r_fb = timeit(ref), timeit(fb(ref))
        torch.backends.cudnn.allow_tf32 = True
        q_f, q_fb = timeit(ref), timeit(fb(ref))
        rows.append(dict(net=net, kind=kind, x=xs, w=ws, s=stride, cnt=cnt, gflop_fwd=flops / 1e9,
                         ours_fwd_ms=t_f, ours_fb_ms=t_fb, ours_fwd_tflops=flops / t_f / 1e9,
                         cudnn_fp32_fwd_ms=r_f, cudnn_fp32_fb_ms=r_fb, cudnn_tf32_fwd_ms=q_f, cudnn_tf32_fb_ms=q_fb))
        tot['ours'] += cnt * t_fb
        tot['cudnn_fp32'] += cnt * r_fb
        tot['cudnn_tf32'] += cnt * q_fb
    rows.sort(key=lambda r: -r['ours_fb_ms'] * r['cnt'])
    for r in rows:
        print(json.dumps(r))
    print(json.dumps(dict(total_fwd_bwd_ms=tot)))


if __name__ == '__main__':
    main()
