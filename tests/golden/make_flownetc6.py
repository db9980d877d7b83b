#!/usr/bin/env python
"""Generate tests/golden/flownetc6_small*.npz from the UNMODIFIED reference FlowNetC6 (models/FlowNetC6.py) on CPU fp32.
Run:  python tests/golden/make_flownetc6.py   (the reference checkout is found as in make_golden.py; the other
fixtures are not touched).

make_golden.py's correlation stub takes Back2Future's arguments only.  FlowNetC6 calls spatial_correlation_sample with
patch_size=21, padding=0 and dilation_patch=2, so its module gets a stub with the full signature, computing the
restated semantics of oracle.nets.spatial_correlation_sample (the third-party op stays parity unpinned).

Contents: weights from synth.seeded_fill(FlowNetC6(), 310); B=2 64x128 frames (synth.frames seed 196), called as
train.py:465 does, flow_net(tgt, ref+): the six train-mode outputs, gradients of sum_i out_i * wts(500 + i) for a sample of
parameters (big ones strided, make_golden.compact), the eval-mode output and the state_dict keys with their shapes."""
import os
import sys
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG                      # noqa: E402  (reference import path, stubs, save helpers)
from oracle import nets as ON                 # noqa: E402

RF = sys.modules['models.FlowNetC6']          # the reference's module (imported by make_golden; `models.FlowNetC6` is the class)


def _corr_stub(in1, in2, kernel_size=1, patch_size=1, stride=1, padding=0, dilation_patch=1):
    assert kernel_size == 1 and stride == 1 and padding == 0, 'stub restates kernel_size=1, stride=1, padding=0 only'
    return ON.spatial_correlation_sample(in1, in2, patch_size, dilation_patch)


RF.spatial_correlation_sample = _corr_stub

B, H, W = 2, 64, 128
FRAME_SEED, WEIGHT_SEED, WTS_SEED = 196, 310, 500
GRAD_PARAMS = ['conv1.0.weight', 'conv3_1.0.weight', 'conv6_1.0.weight', 'deconv1.0.weight', 'predict_flow1.weight',
               'upsampled_flow6_to_5.weight']


def gen():
    tgt, refs = MG.synth.frames(B, H, W, seed=FRAME_SEED)
    net = MG.synth.seeded_fill(RF.FlowNetC6(), WEIGHT_SEED)
    net.train()
    outs = list(net(tgt, refs[2]))
    loss = sum((x * MG.wts(x.shape, WTS_SEED + i)).sum() for i, x in enumerate(outs))
    pd = dict(net.named_parameters())
    grads = torch.autograd.grad(loss, [pd[n] for n in GRAD_PARAMS])
    d = {}
    for i, x in enumerate(outs):
        d['out%d' % i] = x
    for n, g in zip(GRAD_PARAMS, grads):
        sfx, g = MG.compact(g)
        d['g_%s%s' % (n, sfx)] = g
    net.eval()
    with torch.no_grad():
        d['eval'] = net(tgt, refs[2])
    sd = net.state_dict()
    d['state_dict_keys'] = np.array(['%s:%s' % (k, ','.join(map(str, v.shape))) for k, v in sd.items()])
    d['nparams'] = np.array(sum(p.numel() for p in net.parameters()), dtype=np.int64)
    MG.save('flownetc6_small', d)


if __name__ == '__main__':
    gen()
