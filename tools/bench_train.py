#!/usr/bin/env python
"""Developer benchmark of the training driver (cc_b200.train; not bench.py).  Writes a synthetic sequential dump of
seeded cc_b200.synth frames (832x256 JPEGs, --scenes scenes of --frames frames) into --out, then trains on it with the
README command's hyper-parameters and fixed nets (--fix-masknet --fix-flownet, b4) through the driver's epoch loop
(cc_b200.train.run_epoch: DataLoader workers decoding into pinned uint8 batches, HostFeeder, DeviceAugment into the
captured step's inputs, replay, the device loss log read once per --print-freq steps), and reports:

  driver_triplets_per_s   B x steps over the device time between consecutive steps' completion events within each
                          epoch, the capture step excluded
  e2e_triplets_per_s      B x steps over the host time of the epochs after the first, epoch boundaries (worker start)
                          included, ending in a device synchronise
  replay_triplets_per_s   the same trainer's replay() alone on its device-resident inputs (what bench.py times), device
                          events, in the same process
  decode_frames_per_s     Pillow decodes of the dump's frames per second on one host process (one worker's rate)
  depth_validation_s      validate_depth over the dump's val.txt scenes at b4 (--with-depth-gt), host time ending in
                          the host read of the averages
and the card's name and power limit (tools/card.py), as one JSON line.  The README command itself chooses the best model
by --with-flow-gt's error, which needs KITTI-2015; this tool drives the same loop without that validation."""
import argparse
import json
import os
import sys
import time
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cc_b200 import train as T                    # noqa: E402
from cc_b200.input_pipeline import DeviceAugment  # noqa: E402
from cc_b200.train_step import Trainer            # noqa: E402
from tests import train_cases as TC               # noqa: E402
from tools.card import card                       # noqa: E402

README = ('DUMP --dispnet DispResNet6 --posenet PoseNetB6 --masknet MaskNet6 --flownet Back2Future -b4 -m0.1 -pf 0.5 '
          '-pc 1.0 -s0.1 -c0.3 --nlevels 6 --lr 1e-4 -wssim 0.997 --with-flow-gt --smoothness-type edgeaware '
          '--fix-masknet --fix-flownet --name bench').split()


class TimedLog(T.LossLog):
    """The driver's loss log, plus a completion event after every step."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.events = []

    def record(self, i, loss, terms):
        super().record(i, loss, terms)
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.events.append(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default='/tmp/ccb_bench_train')
    ap.add_argument('--scenes', type=int, default=4)
    ap.add_argument('--frames', type=int, default=54)
    ap.add_argument('--epochs', type=int, default=4)
    ap.add_argument('--workers', type=int, default=4)
    ap.add_argument('--print-freq', type=int, default=10)
    ap.add_argument('--replays', type=int, default=50)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    root = TC.write_synth_dump(os.path.join(a.out, 'dump'), scenes=a.scenes, frames=a.frames, H=256, W=832)
    args = T.parse_args(README)
    B = args.batch_size
    ds = T.FrameSet(T.sequence_samples(root, args.seed))
    steps = len(ds) // B
    tr = Trainer('cfg3', dev, T.hyper_parameters(args), seed=args.seed, fixed=T.fixed_nets(args))
    aug = DeviceAugment(dev, rotate=not args.fix_flownet, normalization=args.data_normalization)

    dev_ms, dev_steps, host_s, host_steps = 0.0, 0, 0.0, 0
    for epoch in range(a.epochs):
        order = T.epoch_order(len(ds), B, 0, args.seed, epoch)
        params = T.epoch_params(steps, B, 256, 832, args.seed, epoch, rotate=not args.fix_flownet)
        log = TimedLog(steps, dev, tr.hp['w2'] <= 0, B)
        t0 = time.time()
        T.run_epoch(tr, T.make_loader(ds, order, B, a.workers, True), params, aug, log, a.print_freq)
        torch.cuda.synchronize()
        if epoch > 0:
            host_s += time.time() - t0
            host_steps += steps
        ev = log.events
        dev_ms += ev[0].elapsed_time(ev[-1])            # steps 1 .. steps-1 of the epoch (step 0 of epoch 0 captures)
        dev_steps += len(ev) - 1

    st, sr, sK, sKi = tr.static_in
    for _ in range(3):
        tr.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.replays):
        tr.replay()
    e1.record()
    torch.cuda.synchronize()
    replay_ms = e0.elapsed_time(e1) / a.replays

    n_dec = min(40, len(ds))
    t0 = time.time()
    for i in range(n_dec):
        ds[i]
    decode = 5 * n_dec / (time.time() - t0)

    vs = T.DepthSet(T.validation_samples(root))
    loader = T.make_loader(vs, list(range(len(vs))), B, a.workers, True)
    T.validate_depth(tr.nets['disp'], loader, dev)                   # warm-up of the eval shapes
    t0 = time.time()
    errs = torch.stack(T.validate_depth(tr.nets['disp'], loader, dev)).tolist()
    val_s = time.time() - t0
    for n in tr.nets.values():
        n.train()

    drv = B * dev_steps / (dev_ms / 1e3)
    print(json.dumps(dict(metric='train_driver', batch=B, size='256x832', steps_per_epoch=steps, epochs=a.epochs,
                          workers=a.workers, driver_triplets_per_s=round(drv, 2),
                          e2e_triplets_per_s=round(B * host_steps / host_s, 2) if host_steps else None,
                          replay_triplets_per_s=round(B / (replay_ms / 1e3), 2),
                          driver_over_replay=round(drv / (B / (replay_ms / 1e3)), 4),
                          decode_frames_per_s=round(decode, 1), depth_validation_s=round(val_s, 3),
                          depth_validation_samples=len(vs), depth_errors=errs, card=card())))


if __name__ == '__main__':
    main()
