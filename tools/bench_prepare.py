#!/usr/bin/env python
"""Developer benchmark of the training-data preparation (cc_b200.prepare_train_data; not bench.py).  Writes a seeded
KITTI-size raw tree (tests/prepare_cases.write_kitti_tree: --drives drives x 2 cameras x --frames frames of 1242x375
and 1241x376, sweeps of --points points) into a temporary directory under --out, removed afterwards, and reports as one
JSON line:

  main_frames_per_s       {workers: frames written per second} of main() end to end with --with-gt at 832x256 (every
                          frame kept by a static-frames list), host clock, for --num-threads 1 and 4
  device_s, device_share  the device stages alone in the 4-worker run: CUDA events around each resize_chunk and
                          depth_chunk call (the H2D copy of the chunk included), their sum and its share of that run
  oracle_frames_per_s     oracle/prepare.py (numpy and Pillow, one process) on the first --oracle-frames frames of
                          each drive: the CPU baseline
and the card's name and power limit (tools/card.py).  A first main() on the oracle's small tree warms the device up."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cc_b200 import prepare_train_data as PT      # noqa: E402
from oracle import prepare as OP                  # noqa: E402
from tests import prepare_cases as PC             # noqa: E402
from tools.card import card                       # noqa: E402


def timed(fn, events):
    def run(*a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn(*a, **k)
        e1.record()
        events.append((e0, e1))
        return out
    return run


def write_tree(root, drives, frames, points):
    sizes = ((375, 1242), (376, 1241))
    dr = PC.kitti_size_drives(frames, sizes)[:drives]
    PC.write_kitti_tree(root, drives=dr, out_hw=(256, 832), points=points)
    PC.write_files(root, {'static.txt': PC.STATIC, 'test_scenes.txt': PC.TEST_SCENES})
    return root


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default='/tmp/ccb_bench_prepare')
    ap.add_argument('--drives', type=int, default=2)
    ap.add_argument('--frames', type=int, default=200)
    ap.add_argument('--points', type=int, default=120000)
    ap.add_argument('--oracle-frames', type=int, default=4)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    os.makedirs(a.out, exist_ok=True)
    tmp = tempfile.mkdtemp(dir=a.out)
    cwd = os.getcwd()
    try:
        big = write_tree(os.path.join(tmp, 'big'), a.drives, a.frames, a.points)
        small = write_tree(os.path.join(tmp, 'small'), a.drives, a.oracle_frames, a.points)
        argv = ['raw', '--dataset-format', 'kitti', '--dump-root', 'dump', '--with-gt', '--height', '256', '--width',
                '832', '--test-scenes', 'test_scenes.txt', '--static-frames', 'static.txt']

        def run(root, workers, dump='dump'):
            os.chdir(root)
            try:
                shutil.rmtree(dump, ignore_errors=True)
                t0 = time.time()
                PT.main(argv[:4] + [dump] + argv[5:] + ['--num-threads', str(workers)], device=dev)
                torch.cuda.synchronize()
                dt = time.time() - t0
            finally:
                os.chdir(cwd)
            n = sum(f.endswith('.jpg') for f in PC.dump_files(os.path.join(root, dump)))
            return n, dt

        run(small, 4, 'warmup')
        rates, device_s, share = {}, None, None
        for workers in (1, 4):
            events = []
            saved = PT.resize_chunk, PT.depth_chunk
            if workers == 4:
                PT.resize_chunk, PT.depth_chunk = timed(PT.resize_chunk, events), timed(PT.depth_chunk, events)
            try:
                n, dt = run(big, workers)
            finally:
                PT.resize_chunk, PT.depth_chunk = saved
            rates[workers] = round(n / dt, 2)
            if events:
                device_s = sum(e0.elapsed_time(e1) for e0, e1 in events) / 1e3
                share = device_s / dt
        os.chdir(small)
        try:
            t0 = time.time()
            rec = OP.prepare('raw', 'kitti', 'oracle_dump', 256, 832, 'static.txt', True, 'test_scenes.txt')
            oracle = len(rec['frames']) / (time.time() - t0)
        finally:
            os.chdir(cwd)
        print(json.dumps(dict(metric='prepare_train_data', size='832x256 from 1242x375 / 1241x376', with_gt=True,
                              frames=n, points_per_sweep=a.points, main_frames_per_s=rates,
                              device_s=round(device_s, 3), device_share=round(share, 4),
                              oracle_frames_per_s=round(oracle, 2), oracle_frames=len(rec['frames']), card=card())))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == '__main__':
    main()
