#!/usr/bin/env python
"""A SHA-256 digest of the output of every convolution call (fprop, dgrad, wgrad) of one eager training step at the
benchmark's size: two builds compute the same step bit for bit when their digest lists are equal.
python tools/conv_bits.py [cfg] [out.json]"""
import hashlib
import json
import os
import sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cc_b200 import synth, nn as cnn, _lib                # noqa: E402
from cc_b200.train_step import Trainer                   # noqa: E402

cfg = sys.argv[1] if len(sys.argv) > 1 else 'cfg3'
out_path = sys.argv[2] if len(sys.argv) > 2 else None
B, H, W = 4, 256, 832
dev = torch.device('cuda:0')
tgt, refs = synth.frames(B, H, W, seed=1)
K, Kinv = synth.intrinsics(B, H, W)
tr = Trainer(cfg, dev)
args = (tgt.to(dev), [r.to(dev) for r in refs], K.to(dev), Kinv.to(dev))
OPS = {_lib.CONV_FPROP: 'fprop', _lib.CONV_DGRAD: 'dgrad', _lib.CONV_WGRAD: 'wgrad'}
real_run = cnn._run
records = []


def hashed_run(op, d, *a):
    real_run(op, d, *a)
    out = a[2] if op == _lib.CONV_WGRAD else a[4]        # (x, dy, dw) or (x, w, bias, res, y)
    records.append({'op': OPS[op], 'shape': [d.B, d.Ci, d.Hi, d.Wi, d.Co, d.kh, d.stride],
                    'kernel': (_lib.lib().ccb_debug_last_conv_kernel() or b'').decode(),
                    'sha256': hashlib.sha256(out.detach().contiguous().cpu().numpy().tobytes()).hexdigest()})


# the third step, as tools/conv_calls.py times it: weight cache committed, Adam state warm
for it in range(3):
    records.clear()
    cnn._run = hashed_run if it == 2 else real_run
    tr.step(*args)
    cnn._run = real_run
    torch.cuda.synchronize()
total = hashlib.sha256(''.join(r['sha256'] for r in records).encode()).hexdigest()
print('%d conv calls (%s), digest of all outputs %s' % (len(records), ', '.join(
    '%d %s' % (sum(r['op'] == o for r in records), o) for o in OPS.values()), total))
if out_path:
    with open(out_path, 'w') as f:
        json.dump({'cfg': cfg, 'calls': records, 'digest': total}, f, indent=0)
