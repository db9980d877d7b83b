#!/usr/bin/env python
"""Developer benchmark of the depth-evaluation command (cc_b200.test_disp; not bench.py).  Writes a seeded KITTI raw tree
into a temporary directory under --out, removed afterwards: two drives of 1242x375 and 1241x376 PNG frames
(tests/run_inference_cases.photo) with --points-point velodyne sweeps, and a list of --samples targets, half from each.
Runs main() with a seeded DispResNet6 and PoseNetB6 at seq 5 (4 reference frames) at 256x832, and reports as one JSON
line:

  main_samples_per_s    samples per second of main() end to end (--workers host processes), host clock around the call
  device_samples_per_s  the device stages alone (evaluate_chunk: the H2D copies, ground truth, stretch and resize, both
                        nets, zoom and errors), CUDA events around each call inside main()
  device_share          those stages' time over main()'s time
and the card's name and power limit (tools/card.py).  A first main() on a few samples warms every shape up."""
import argparse
import contextlib
import io
import json
import os
import shutil
import sys
import tempfile
import time
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cc_b200 import test_disp as TD              # noqa: E402
from oracle import nets as ON                    # noqa: E402
from tests import depth_command_cases as DC      # noqa: E402
from tools.card import card                      # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default='/tmp/ccb_bench_test_disp')
    ap.add_argument('--samples', type=int, default=200)
    ap.add_argument('--points', type=int, default=120000)
    ap.add_argument('--workers', type=int, default=TD.WORKERS)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    os.makedirs(a.out, exist_ok=True)
    tmp = tempfile.mkdtemp(dir=a.out)
    try:
        half = a.samples // 2
        drives = {('2011_09_26', '2011_09_26_drive_0001_sync'): (half + 4, ('image_02',)),
                  ('2011_09_30', '2011_09_30_drive_0003_sync'): (a.samples - half + 4, ('image_02',))}
        DC.write_kitti_tree(os.path.join(tmp, 'kitti'), a.points, DC.KITTI_SIZE_DATES, drives, seed=11)
        files = ['%s/%s/image_02/data/%010d.png' % (date, drive, 2 + i)
                 for (date, drive), (n, _) in sorted(drives.items()) for i in range(n - 4)]
        with open(os.path.join(tmp, 'list.txt'), 'w') as f:
            f.write('\n'.join(files) + '\n')
        with open(os.path.join(tmp, 'warm.txt'), 'w') as f:
            f.write('\n'.join(files[:2] + files[-2:]) + '\n')
        torch.save({'state_dict': ON.disp_params(DC.DISP_SEED)}, os.path.join(tmp, 'disp.pth.tar'))
        torch.save(DC.pose_checkpoint('PoseNetB6'), os.path.join(tmp, 'pose.pth.tar'))
        argv = ['--pretrained-dispnet', os.path.join(tmp, 'disp.pth.tar'), '--pretrained-posenet',
                os.path.join(tmp, 'pose.pth.tar'), '--posenet', 'PoseNetB6', '--dataset-dir', os.path.join(tmp, 'kitti')]
        events = []
        evaluate_chunk = TD.evaluate_chunk

        def timed(*args, **kw):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = evaluate_chunk(*args, **kw)
            e1.record()
            events.append((e0, e1))
            return out
        with contextlib.redirect_stdout(io.StringIO()):
            TD.main(argv + ['--dataset-list', os.path.join(tmp, 'warm.txt')], device=dev, workers=a.workers)
        torch.cuda.synchronize()
        TD.evaluate_chunk = timed
        buf = io.StringIO()
        try:
            with contextlib.redirect_stdout(buf):
                t0 = time.time()
                TD.main(argv + ['--dataset-list', os.path.join(tmp, 'list.txt')], device=dev, workers=a.workers)
                torch.cuda.synchronize()
                dt = time.time() - t0
        finally:
            TD.evaluate_chunk = evaluate_chunk
        dev_s = sum(e0.elapsed_time(e1) for e0, e1 in events) / 1e3
        print(json.dumps(dict(metric='test_disp', samples=len(files), source='1242x375 + 1241x376 PNG',
                              points_per_sweep=a.points, nets='DispResNet6 + PoseNetB6 (seq 5)', size='256x832',
                              workers=a.workers, main_samples_per_s=round(len(files) / dt, 2),
                              device_samples_per_s=round(len(files) / dev_s, 2), device_share=round(dev_s / dt, 4),
                              card=card())))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == '__main__':
    main()
