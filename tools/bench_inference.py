#!/usr/bin/env python
"""Developer benchmark of run_inference (cc_b200.run_inference; not bench.py).  Writes --photos seeded KITTI-size PNGs
(1242x375, tests/run_inference_cases.photo) into a temporary directory under --out, removed afterwards, and reports as
one JSON line, for a seeded DispNetS at 128x416 (the script's default) and 256x832:

  main_images_per_s    photos per second of main() end to end (--output-disp --output-depth, PNG outputs, --workers
                       host processes), host clock around the call
  device_images_per_s  infer() alone on the decoded photos in chunks of run_inference.CHUNK: the H2D copy, contrast
                       stretch and resize, normalisation, the net and both colorize calls, CUDA events around each call
  device_share         the device stages' time in main() (CUDA events around each infer() call) over main()'s time
and the card's name and power limit (tools/card.py).  A first main() on a few photos warms every shape up."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cc_b200 import run_inference as RI      # noqa: E402
from tests import run_inference_cases as RC  # noqa: E402
from tools.card import card                  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default='/tmp/ccb_bench_inference')
    ap.add_argument('--photos', type=int, default=256)
    ap.add_argument('--workers', type=int, default=RI.WORKERS)
    a = ap.parse_args()
    from PIL import Image
    dev = torch.device('cuda:0')
    os.makedirs(a.out, exist_ok=True)
    tmp = tempfile.mkdtemp(dir=a.out)
    try:
        photos = os.path.join(tmp, 'photos')
        os.makedirs(photos)
        frames = [RC.photo(375, 1242, 100 + k % 16) for k in range(a.photos)]
        for k, f in enumerate(frames):
            Image.fromarray(f).save(os.path.join(photos, '%06d.png' % k))
        ckpt = os.path.join(tmp, 'ckpt.pth.tar')
        torch.save(RC.checkpoint(), ckpt)
        net = RI.load_disp_net(ckpt, 'DispNetS', dev)
        res = {}
        for h, w in ((128, 416), (256, 832)):
            argv = ['--output-disp', '--output-depth', '--pretrained', ckpt, '--img-height', str(h), '--img-width', str(w),
                    '--dataset-dir', photos, '--output-dir', os.path.join(tmp, 'out')]
            events = []
            infer = RI.infer

            def timed(*args, **kw):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = infer(*args, **kw)
                e1.record()
                events.append((e0, e1))
                return out
            warm = os.path.join(tmp, 'warm')
            os.makedirs(warm, exist_ok=True)
            for k in range(4):
                shutil.copy(os.path.join(photos, '%06d.png' % k), warm)
            RI.main(argv[:-3] + [warm, '--output-dir', os.path.join(tmp, 'warm_out')], device=dev, workers=a.workers)
            RI.infer(net, frames[:RI.CHUNK], h, w)
            torch.cuda.synchronize()
            RI.infer = timed
            try:
                t0 = time.time()
                RI.main(argv, device=dev, workers=a.workers)
                torch.cuda.synchronize()
                dt = time.time() - t0
            finally:
                RI.infer = infer
            dev_s = sum(e0.elapsed_time(e1) for e0, e1 in events) / 1e3
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(0, len(frames), RI.CHUNK):
                RI.infer(net, frames[i:i + RI.CHUNK], h, w)
            e1.record()
            torch.cuda.synchronize()
            res['%dx%d' % (h, w)] = dict(main_images_per_s=round(len(frames) / dt, 2),
                                         device_images_per_s=round(len(frames) / (e0.elapsed_time(e1) / 1e3), 2),
                                         device_share=round(dev_s / dt, 4))
            shutil.rmtree(os.path.join(tmp, 'out'), ignore_errors=True)
        print(json.dumps(dict(metric='run_inference', photos=a.photos, source='1242x375 PNG', net='DispNetS',
                              workers=a.workers, results=res, card=card())))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == '__main__':
    main()
