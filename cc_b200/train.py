"""The reference's train.py main() (train.py:141-417, train() :422-586, validate_depth_with_gt :588-636) on this stack:
`python -m cc_b200.train DATA --name NAME ...` trains the four nets of cfg3 on a dump written by data/prepare_train_data.py
and writes the reference's checkpoints and progress logs under checkpoints/NAME.

  samples      sequence_samples / stacked_samples / validation_samples: the lists the reference's SequenceFolder
               (sequential and stacked) and ValidationSet build, in their order; frames decoded with Pillow
               (np.asarray(Image.open(p)), what scipy.misc.imread returned) in DataLoader workers into pinned uint8
               batches [B,5,H,W,3] ([tgt, refs...]) and K.
  epoch        run_epoch: the captured step (Trainer.capture / replay) fed by HostFeeder one batch ahead, the uint8 batch
               augmented on the device (DeviceAugment) into the graph's input buffers; the per-step loss rows of
               progress_log_full.csv go to a device log that the host reads once per --print-freq steps.
  validation   validate_depth (validate_depth_with_gt) and validate_flow (validate_flow_with_gt through
               evaluate.flow_eval_batch), both averaged as the reference's AverageMeter does on 0-dim fp32 tensors.
  files        save_checkpoint (utils.py:55-63), the tab-separated logs (train.py:317-323,415-417,574-576).

Documented deviation: the reference draws its batch order from the DataLoader's global torch generator and its augmentation
from per-worker generators, so neither can be reproduced across worker counts.  Here epoch e's order comes from a
torch.Generator and its augmentation from a random.Random and a np.random.RandomState, all seeded from (seed, e)
(epoch_seed), and drawn on the main process: a run depends on (seed, epoch) alone, never on --workers."""
import argparse
import csv
import fnmatch
import os
import random
import shutil
import sys
import time
import numpy as np
import torch

from . import _lib, pyramid, loss_functions as LF, evaluate as EV
from .input_pipeline import DeviceAugment, draw_params, scale_frames, to_device
from .train_step import Trainer, HostFeeder, FLOWNETS

SEQUENCE_LENGTH = 5
NETS = ('disp', 'pose', 'mask', 'flow')
CKPT_PREFIXES = ('dispnet', 'posenet', 'masknet', 'flownet', 'optimizer')
SUMMARY_HEADER = ['train_loss', 'validation_loss']
FULL_HEADER = ['train_loss', 'photo_cam_loss', 'photo_flow_loss', 'explainability_loss', 'smooth_loss']
DEPTH_ERROR_NAMES = ['abs_diff', 'abs_rel', 'sq_rel', 'a1', 'a2', 'a3']
FLOW_ERROR_NAMES = ['epe_total', 'epe_rigid', 'epe_non_rigid', 'outliers', 'epe_total_with_gt_mask',
                    'epe_rigid_with_gt_mask', 'epe_non_rigid_with_gt_mask', 'outliers_gt_mask']


# ---- samples (datasets/sequence_folders.py, stacked_sequence_folders.py, validation_folders.py) ----------------------
def _list_lines(path):
    """The lines of a scene list as the reference reads them: each line minus its last character (`folder[:-1]`)."""
    with open(path) as f:
        return [line[:-1] for line in f]


def _files(folder, pattern):
    """path.Path(folder).files(pattern), sorted: the regular files of `folder` whose name matches."""
    return sorted(os.path.join(folder, f) for f in os.listdir(folder)
                  if fnmatch.fnmatch(f, pattern) and os.path.isfile(os.path.join(folder, f)))


def _read_cam(path):
    return np.genfromtxt(path, delimiter=',').astype(np.float32).reshape((3, 3))


def sequence_samples(root, seed=0, train=True, sequence_length=SEQUENCE_LENGTH):
    """SequenceFolder(root, seed, train, sequence_length).samples (sequence_folders.py:8-23,43-49): the scenes of
    train.txt / val.txt, targets demi_length .. len - demi_length of each scene's sorted jpgs (a scene with fewer frames
    than sequence_length is skipped), refs i-2, i-1, i+1, i+2; shuffled as random.seed(seed); random.shuffle(...) does.
    Each sample is dict(frames=[tgt, refs...], K=float32 [3,3])."""
    scenes = [os.path.join(root, s) for s in _list_lines(os.path.join(root, 'train.txt' if train else 'val.txt'))]
    demi = (sequence_length - 1) // 2
    samples = []
    for folder in scenes:
        K = _read_cam(os.path.join(folder, 'cam.txt'))
        imgs = _files(folder, '*.jpg')
        if len(imgs) < sequence_length:
            continue
        for i in range(demi, len(imgs) - demi):
            samples.append(dict(frames=[imgs[i]] + [imgs[i + j] for j in range(-demi, demi + 1) if j != 0], K=K))
    random.Random(seed).shuffle(samples)
    return samples


def stacked_samples(root, train=True):
    """The stacked SequenceFolder's samples (stacked_sequence_folders.py:41-56): one `scene frame` line of train.txt /
    val.txt per sample, in file order, dict(stack=<scene>/<frame>.jpg, K=<scene>/<frame>_cam.txt as float32 [3,3])."""
    samples = []
    for line in _list_lines(os.path.join(root, 'train.txt' if train else 'val.txt')):
        a, b = line.split(' ')
        base = os.path.join(root, a, b)
        samples.append(dict(stack=base + '.jpg', K=_read_cam(base + '_cam.txt')))
    return samples


def validation_samples(root):
    """ValidationSet(root) (validation_folders.py:8-20,64-69): every jpg of the val.txt scenes in sorted order with the
    .npy depth beside it -> [(jpg, npy)]."""
    out = []
    for folder in [os.path.join(root, s) for s in _list_lines(os.path.join(root, 'val.txt'))]:
        for img in _files(folder, '*.jpg'):
            d = img[:-4] + '.npy'
            assert os.path.isfile(d), 'depth file {} not found'.format(d)
            out.append((img, d))
    return out


def decode(path):
    """The uint8 frame scipy.misc.imread returned (Pillow's decoder): np.asarray(Image.open(path))."""
    from PIL import Image
    with Image.open(path) as im:
        return np.asarray(im)


def split_stack(stack, sequence_length=SEQUENCE_LENGTH):
    """A stacked jpg's frames (stacked_sequence_folders.py:21-27): slices of width int(w / sequence_length), ordered
    [tgt] + imgs[:tgt_index] + imgs[tgt_index + 1:]."""
    w_img = int(stack.shape[1] / sequence_length)
    imgs = [stack[:, i * w_img:(i + 1) * w_img] for i in range(sequence_length)]
    t = sequence_length // 2
    return [imgs[t]] + imgs[:t] + imgs[t + 1:]


class FrameSet(torch.utils.data.Dataset):
    """Samples -> (uint8 [5,H,W,3] frames in [tgt, refs...] order, float32 K [3,3]); decoded in the loader's workers,
    which draw no random numbers."""

    def __init__(self, samples):
        self.samples = samples

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        s = self.samples[i]
        frames = split_stack(decode(s['stack'])) if 'stack' in s else [decode(p) for p in s['frames']]
        return torch.from_numpy(np.ascontiguousarray(np.stack(frames))), torch.from_numpy(s['K'].copy())


class DepthSet(torch.utils.data.Dataset):
    """validation_samples -> (uint8 [1,H,W,3], float32 depth [H,W])."""

    def __init__(self, samples):
        self.samples = samples

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        img, d = self.samples[i]
        return torch.from_numpy(decode(img)[None].copy()), torch.from_numpy(np.load(d).astype(np.float32))


def epoch_seed(seed, epoch):
    """One 32-bit seed for epoch `epoch` of a run seeded `seed`."""
    return int(np.random.SeedSequence([int(seed), int(epoch)]).generate_state(1)[0])


def epoch_order(n_samples, batch_size, epoch_size, seed, epoch):
    """The sample indices of an epoch, batch after batch: a permutation from a torch.Generator seeded epoch_seed(seed,
    epoch), cut to whole batches (drop_last, train.py:228-230) and to the first epoch_size of them (0: all, :239-240)."""
    g = torch.Generator()
    g.manual_seed(epoch_seed(seed, epoch))
    perm = torch.randperm(n_samples, generator=g).tolist()
    n = n_samples // batch_size
    if epoch_size:
        n = min(n, epoch_size)
    return perm[:n * batch_size]


def epoch_params(n_batches, batch_size, Hs, Ws, seed, epoch, rotate):
    """The augmentation decisions of an epoch's batches in batch order (input_pipeline.draw_params), from a random.Random
    and a np.random.RandomState seeded epoch_seed(seed, epoch)."""
    s = epoch_seed(seed, epoch)
    rr, rn = random.Random(s), np.random.RandomState(s)
    return [draw_params(batch_size, Hs, Ws, rng_random=rr, rng_np=rn, rotate=rotate) for _ in range(n_batches)]


def make_loader(dataset, indices, batch_size, workers, pin):
    """A DataLoader over `indices` in their order, whole batches only.  It gets its own generator: creating its iterator
    draws a worker seed, which must not advance the global torch generator."""
    return torch.utils.data.DataLoader(dataset, batch_size=batch_size, sampler=indices, num_workers=workers,
                                       pin_memory=pin, drop_last=True, generator=torch.Generator())


# ---- decisive error (train.py:380-395) -------------------------------------------------------------------------------
def decisive_source(fixed):
    """(flag, column) of the error train.py:382-389 picks for the set of fixed nets: ('--with-flow-gt', -2) for a trained
    pose net, else ('--with-depth-gt', 0) for a trained disp net, else ('--with-flow-gt', -1) for a trained flow net, else
    ('--with-flow-gt', 3) for a trained mask net."""
    if 'pose' not in fixed:
        return '--with-flow-gt', -2
    if 'disp' not in fixed:
        return '--with-depth-gt', 0
    if 'flow' not in fixed:
        return '--with-flow-gt', -1
    return '--with-flow-gt', 3


def decisive_error(fixed, errors, flow_errors):
    flag, col = decisive_source(fixed)
    return (flow_errors if flag == '--with-flow-gt' else errors)[col]


class AverageMeter:
    """logger.AverageMeter's update: sum += val * n, avg = sum / count, elementwise over a list."""

    def __init__(self, i=1):
        self.sum, self.avg, self.val, self.count = [0] * i, [0] * i, [0] * i, 0

    def update(self, val, n=1):
        val = val if isinstance(val, list) else [val]
        self.count += n
        for i, v in enumerate(val):
            self.val[i] = v
            self.sum[i] += v * n
            self.avg[i] = self.sum[i] / self.count

    def __repr__(self, precision=3):
        fmt = lambda xs: ' '.join('{:.{}f}'.format(v, precision) for v in xs)      # noqa: E731
        return '{} ({})'.format(fmt(self.val), fmt(self.avg))


# ---- files (utils.py:55-63; train.py:317-323,415-417,574-576) --------------------------------------------------------
def write_rows(path, rows, mode='a'):
    with open(path, mode) as f:
        w = csv.writer(f, delimiter='\t')
        for r in rows:
            w.writerow(r)


def net_state(net):
    """A net's state dict with its own host copy of every tensor (the parameters are views into the flat Adam buffer,
    and torch.save would otherwise write that whole buffer into each file)."""
    return {k: v.detach().cpu().clone() for k, v in net.state_dict().items()}


def save_checkpoint(save_path, trainer, epoch, is_best):
    """utils.save_checkpoint: {prefix}_checkpoint.pth.tar = {'epoch': epoch, 'state_dict': ...} for the four nets and the
    optimizer (FlatAdam.state_dict: torch.optim.Adam's format over chain(disp, pose, mask, flow)), each copied to
    {prefix}_model_best.pth.tar when is_best."""
    states = [net_state(trainer.nets[n]) for n in NETS] + [trainer.opt.state_dict()]
    for prefix, state in zip(CKPT_PREFIXES, states):
        torch.save({'epoch': epoch, 'state_dict': state}, os.path.join(save_path, prefix + '_checkpoint.pth.tar'))
    if is_best:
        for prefix in CKPT_PREFIXES:
            shutil.copyfile(os.path.join(save_path, prefix + '_checkpoint.pth.tar'),
                            os.path.join(save_path, prefix + '_model_best.pth.tar'))


def load_resume(save_path, trainer):
    """--resume: the four nets from save_path's checkpoints and, when the file exists, the optimizer (the per-net Adam
    step counts through FlatAdam.load_state_dict); the weight cache is refreshed."""
    with torch.no_grad():
        for n, prefix in zip(NETS, CKPT_PREFIXES):
            sd = torch.load(os.path.join(save_path, prefix + '_checkpoint.pth.tar'), map_location='cpu')['state_dict']
            trainer.nets[n].load_state_dict(sd)
    opt = os.path.join(save_path, 'optimizer_checkpoint.pth.tar')
    if os.path.exists(opt):
        trainer.opt.load_state_dict(torch.load(opt, map_location='cpu')['state_dict'])
    trainer.refresh_weights()


# ---- one epoch (train.py:422-586) ------------------------------------------------------------------------------------
class LossLog:
    """The per-step rows of progress_log_full.csv on the device ([steps, 5]: loss, loss_1, loss_2, loss_3, loss_4), read
    by the host in one copy per flush, and the epoch's loss meter (AverageMeter(loss.item(), B) in step order)."""

    def __init__(self, steps, device, w2_zero, batch_size):
        self.rows = torch.zeros(steps, 5, device=device)
        self.zero = torch.zeros((), device=device)
        self.w2_zero, self.batch_size = w2_zero, batch_size
        self.done, self.written = 0, []
        self.meter = AverageMeter()

    def record(self, i, loss, terms):
        t = [loss, terms['loss_1'], self.zero if self.w2_zero else terms['loss_2'], terms['loss_3'], terms['loss_4']]
        torch.stack([x.reshape(()) for x in t], out=self.rows[i])

    def flush(self, upto, on_row=None):
        """Rows done..upto-1 to the host (one copy) -> the csv rows, the meter updated row by row; on_row(j) is called
        after row j's update (the meter then holds the state the reference's meter has after step j)."""
        host = self.rows[self.done:upto].cpu().tolist()
        out = []
        for j, r in enumerate(host, self.done):
            if self.w2_zero:
                r[2] = 0                                       # the reference writes the int 0 (train.py:576)
            self.meter.update(r[0], self.batch_size)
            out.append(r)
            if on_row is not None:
                on_row(j)
        self.done = upto
        return out


def run_epoch(trainer, loader, params, aug, log, print_freq=10, full_log=None, printer=None):
    """One epoch of train(): batch i of `loader` augmented with params[i] and stepped; on CUDA the first step of the
    trainer's life captures the step graph and every step replays it; on the simulator build the step runs eagerly.
    Returns the epoch's train loss (losses.avg[0]).

    printer gets the reference's 'Train: Time ... Data ... Loss ...' line for every step j with j % print_freq == 0
    (train.py:579-580), written when the log is flushed.  Its Loss meter is the reference's as of step j.  The steps are
    not timed one by one (that would synchronise every step): Time is the mean step time of the flush window on the
    host clock, and Data, the reference's wait for its loader, is not measured and shows 0."""
    cuda = torch.device(trainer.device).type == 'cuda'
    n = len(params)
    it = iter(loader)
    Ks = {}
    t0, t_flush = time.time(), 0
    batch_time = AverageMeter()

    def batch_of(i):
        frames, K = next(it)
        Ks[i] = K.numpy()
        return [frames]

    feeder = None
    for i in range(n):
        if cuda:
            if feeder is None:
                first = batch_of(0)
                static_u8 = torch.empty(first[0].shape, dtype=torch.uint8, device=trainer.device)
                feeder = HostFeeder([static_u8], lambda j, f=first: f if j == 0 else batch_of(j))
            feeder.feed(i, prefetch=i + 1 < n)
            src = static_u8
        else:
            src = batch_of(i)[0]
        tgt, refs, K, Kinv = aug(src, Ks.pop(i), params=params[i], tgt_index=0)
        if cuda:
            if trainer.graph is None:
                trainer.capture(tgt, refs, K, Kinv)             # this batch's tensors become the graph's inputs
            else:
                st, sr, sK, sKi = trainer.static_in
                for s, v in zip([st] + sr + [sK, sKi], [tgt] + refs + [K, Kinv]):
                    s.copy_(v)
            loss = trainer.replay()
            terms = trainer.static_terms
        else:
            loss, terms = trainer.step(tgt, refs, K, Kinv)
        log.record(i, loss, terms)
        if (i + 1) % print_freq == 0 or i == n - 1:
            step_s = (time.time() - t0) / (i + 1 - log.done)

            def on_row(j):
                batch_time.update(step_s)
                if printer is not None and j % print_freq == 0:
                    printer('Train: Time {} Data {} Loss {}'.format(batch_time, AverageMeter(), log.meter.__repr__(4)))
            rows = log.flush(i + 1, on_row)
            t0 = time.time()
            if full_log is not None:
                write_rows(full_log, rows)
    return log.meter.avg[0]


# ---- validation ------------------------------------------------------------------------------------------------------
@torch.no_grad()
def validate_depth(disp_net, loader, device, normalization='global'):
    """validate_depth_with_gt: the disp net in eval mode at batch B on the validation transform (ArrayToTensor and
    normalize: scale_frames at the frames' own size), 1 / disp, then compute_errors(gt, depth.squeeze(1)); the six
    metrics summed on the device in batch order and divided by the count (AverageMeter over 0-dim fp32 tensors) -> list
    of six 0-dim device tensors.  The net is left in eval mode."""
    disp_net.eval()
    acc, count = torch.zeros(6, device=device), 0
    for frames, depth in loader:
        H, W = frames.shape[2:4]
        tgt = scale_frames(to_device(frames, device), H, W, normalization)[0][0]
        out = 1 / disp_net(tgt)
        acc += torch.stack(LF.compute_errors(to_device(depth, device), out.squeeze(1)))
        count += 1
    assert count > 0, 'the validation set holds fewer samples than one batch'
    avg = acc / count
    return [avg[k] for k in range(6)]


@torch.no_grad()
def validate_flow(nets, framework, batch_size, THRESH=0.01, normalization='global'):
    """validate_flow_with_gt: evaluate.flow_eval_batch over the KITTI-2015 samples (batches of one frame size, at most
    batch_size each) with the four nets in eval mode at 256x832, the frames normalised as training normalises them
    (train.py:165-170,189-190: --data-normalization); the 8 columns summed on the device in sample order and
    divided by the count -> list of eight 0-dim device tensors.  The nets are left in eval mode."""
    n = len(framework['samples'])
    rows = [None] * n
    for idx in framework['groups'].values():
        for c in range(0, len(idx), batch_size):
            chunk = idx[c:c + batch_size]
            s = EV.load_kitti_flow_samples(framework, chunk)
            out = EV.flow_eval_batch(nets['disp'], nets['pose'], nets['mask'], nets['flow'], s['frames'], s['K'],
                                     s['gt'], s['obj'], THRESH=THRESH, normalization=normalization)
            for k, i in enumerate(chunk):
                rows[i] = out[k]
    acc = torch.zeros(8, device=rows[0].device)
    for r in rows:
        acc += r
    avg = acc / n
    return [avg[k] for k in range(8)]


# ---- command line (train.py:34-135) ----------------------------------------------------------------------------------
def build_parser():
    p = argparse.ArgumentParser(description='Competitive Collaboration training on KITTI and CityScapes Dataset',
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    a = p.add_argument
    a('data', metavar='DIR', help='path to dataset')
    a('--kitti-dir', dest='kitti_dir', type=str, default='kitti/kitti2015')
    a('--DEBUG', action='store_true')
    a('--name', dest='name', type=str, default='demo', required=True)
    a('--dataset-format', default='sequential', metavar='STR', choices=['sequential', 'stacked'])
    a('--sequence-length', type=int, metavar='N', default=5)
    a('--rotation-mode', type=str, choices=['euler', 'quat'], default='euler')
    a('--padding-mode', type=str, choices=['zeros', 'border'], default='zeros')
    a('--with-depth-gt', action='store_true')
    a('--with-flow-gt', action='store_true')
    a('-j', '--workers', default=4, type=int, metavar='N')
    a('--epochs', default=200, type=int, metavar='N')
    a('--epoch-size', default=0, type=int, metavar='N')
    a('-b', '--batch-size', default=4, type=int, metavar='N')
    a('--lr', '--learning-rate', default=2e-4, type=float, metavar='LR')
    a('--momentum', default=0.9, type=float, metavar='M')
    a('--beta', default=0.999, type=float, metavar='M')
    a('--weight-decay', '--wd', default=0, type=float, metavar='W')
    a('--print-freq', default=10, type=int, metavar='N')
    a('-e', '--evaluate', dest='evaluate', action='store_true')
    a('--smoothness-type', dest='smoothness_type', type=str, default='regular', choices=['edgeaware', 'regular'])
    a('--data-normalization', dest='data_normalization', type=str, default='global', choices=['local', 'global'])
    a('--nlevels', dest='nlevels', type=int, default=6)
    a('--dispnet', dest='dispnet', type=str, default='DispResNet6', choices=['DispResNet6'])
    a('--posenet', dest='posenet', type=str, default='PoseNetB6', choices=['PoseNetB6'])
    a('--masknet', dest='masknet', type=str, default='MaskNet6', choices=['MaskNet6'])
    a('--flownet', dest='flownet', type=str, default='Back2Future', choices=list(FLOWNETS))
    for k in ('disp', 'mask', 'pose', 'flow'):
        a('--pretrained-' + k, dest='pretrained_' + k, default=None, metavar='PATH')
    for k in ('spatial-normalize', 'robust', 'no-non-rigid-mask', 'joint-mask-for-depth', 'fix-masknet', 'fix-posenet',
              'fix-flownet', 'fix-dispnet', 'alternating', 'clamp-masks', 'fix-posemasknet'):
        a('--' + k, dest=k.replace('-', '_'), action='store_true')
    a('--seed', default=0, type=int)
    a('--log-summary', default='progress_log_summary.csv', metavar='PATH')
    a('--log-full', default='progress_log_full.csv', metavar='PATH')
    a('-qch', '--qch', type=float, metavar='W', default=0.5)
    a('-wrig', '--wrig', type=float, metavar='W', default=1.0)
    a('-wbce', '--wbce', type=float, metavar='W', default=0.5)
    a('-wssim', '--wssim', type=float, metavar='W', default=0.0)
    a('-pc', '--cam-photo-loss-weight', type=float, metavar='W', default=1)
    a('-pf', '--flow-photo-loss-weight', type=float, metavar='W', default=1)
    a('-m', '--mask-loss-weight', type=float, metavar='W', default=0)
    a('-s', '--smooth-loss-weight', type=float, metavar='W', default=0.1)
    a('-c', '--consensus-loss-weight', type=float, metavar='W', default=0.1)
    a('--THRESH', '--THRESH', type=float, metavar='W', default=0.01)
    a('--lambda-oob', type=float, default=0)
    a('--log-output', action='store_true')
    a('--log-terminal', action='store_true')
    a('--resume', action='store_true')
    a('-f', '--training-output-freq', type=int, metavar='N', default=0)
    return p


def fixed_nets(args):
    return tuple(n for n in NETS if getattr(args, 'fix_%snet' % n))


def parse_args(argv):
    """The reference's flags; the ones this trainer cannot honour are refused (parser.error, naming the flag):
    --robust and --joint-mask-for-depth are broken in the reference, --no-non-rigid-mask and --spatial-normalize are not
    implemented by the Trainer, the image logging (--log-output, -f, --DEBUG) needs tensorboardX and matplotlib; and so is
    a flag combination whose decisive error (train.py:382-389) the validation flags do not compute, which the reference
    only finds after its first epoch (NameError)."""
    parser = build_parser()
    args = parser.parse_args(argv)
    for flag, bad, why in (
            ('--robust', args.robust, 'its robust losses are missing from the reference'),
            ('--joint-mask-for-depth', args.joint_mask_for_depth, 'it is broken in the reference'),
            ('--no-non-rigid-mask', args.no_non_rigid_mask, 'the Trainer does not implement it'),
            ('--spatial-normalize', args.spatial_normalize, 'the Trainer does not implement it'),
            ('--sequence-length', args.sequence_length != 5, 'only 5 is supported'),
            ('--nlevels', args.nlevels != 6, 'only 6 is supported'),
            ('--weight-decay', args.weight_decay != 0, 'only 0 is supported'),
            ('--log-output', args.log_output, 'image logging needs tensorboardX and matplotlib'),
            ('-f/--training-output-freq', args.training_output_freq > 0, 'image logging needs tensorboardX and matplotlib'),
            ('--DEBUG', args.DEBUG, 'its image logging needs tensorboardX and matplotlib')):
        if bad:
            parser.error('%s is not supported: %s' % (flag, why))
    fixed = fixed_nets(args)
    if len(fixed) == len(NETS):
        parser.error('--fix-dispnet --fix-posenet --fix-masknet --fix-flownet: every net is fixed, nothing to train')
    flag, _ = decisive_source(fixed)
    if not getattr(args, flag[2:].replace('-', '_')):
        parser.error('%s is required: with these --fix-* flags the best model is chosen by an error it computes' % flag)
    return args


def hyper_parameters(args):
    return dict(w1=args.cam_photo_loss_weight, w2=args.mask_loss_weight, w3=args.smooth_loss_weight,
                w4=args.flow_photo_loss_weight, w5=args.consensus_loss_weight, wssim=args.wssim, qch=args.qch,
                lambda_oob=args.lambda_oob, THRESH=args.THRESH, wbce=args.wbce, wrig=args.wrig, lr=args.lr,
                beta1=args.momentum, beta2=args.beta, smoothness=args.smoothness_type)


def main(argv=None, device=None):
    """train.py main(): returns dict(save_path, train_losses, decisive_errors, trainer)."""
    args = parse_args(sys.argv[1:] if argv is None else argv)
    dev = device or _lib.device()
    cuda = dev.type == 'cuda'
    save_path = os.path.join('checkpoints', args.name)
    print('=> will save everything to {}'.format(save_path))
    os.makedirs(save_path, exist_ok=True)
    say = print if args.log_terminal else (lambda *a: None)

    if args.dataset_format == 'stacked':
        train_samples = stacked_samples(args.data)
    else:
        train_samples = sequence_samples(args.data, args.seed)
    train_set = FrameSet(train_samples)
    val_loader = None
    if args.with_depth_gt:
        val_set = DepthSet(validation_samples(args.data.replace('cityscapes', 'kitti')))
        if len(val_set) < args.batch_size:
            raise SystemExit('--with-depth-gt: %d validation samples in %s, fewer than one batch of %d' % (
                len(val_set), args.data.replace('cityscapes', 'kitti'), args.batch_size))
        val_loader = make_loader(val_set, list(range(len(val_set))), args.batch_size, args.workers, cuda)
    framework = EV.kitti_flow_framework(args.kitti_dir) if args.with_flow_gt else None
    print('{} samples found in train scenes'.format(len(train_set)))
    n_batches = len(train_set) // args.batch_size
    epoch_size = min(n_batches, args.epoch_size) if args.epoch_size else n_batches
    if epoch_size == 0:
        raise SystemExit('fewer than one batch of %d samples in %s' % (args.batch_size, args.data))

    print('=> creating model')
    sds = {}
    for n in NETS:
        path = getattr(args, 'pretrained_' + n)
        if path:
            sds[n] = torch.load(path, map_location='cpu')['state_dict']
    fixed = fixed_nets(args)
    trainer = Trainer('cfg3', dev, hyper_parameters(args), state_dicts=sds, seed=args.seed, flownet=args.flownet,
                      fixed=fixed)
    if args.resume:
        print('=> resuming from checkpoint')
        load_resume(save_path, trainer)

    summary, full = os.path.join(save_path, args.log_summary), os.path.join(save_path, args.log_full)
    write_rows(summary, [SUMMARY_HEADER], 'w')
    write_rows(full, [FULL_HEADER], 'w')
    aug = DeviceAugment(dev, rotate=not args.fix_flownet, normalization=args.data_normalization)
    best_error, train_losses, decisive = -1, [], []
    Hs = Ws = None
    for epoch in range(args.epochs):
        for net in trainer.nets.values():
            net.train()
        order = epoch_order(len(train_set), args.batch_size, epoch_size, args.seed, epoch)
        loader = make_loader(train_set, order, args.batch_size, args.workers, cuda)
        if Hs is None:
            Hs, Ws = train_set[order[0]][0].shape[1:3]
        params = epoch_params(epoch_size, args.batch_size, Hs, Ws, args.seed, epoch, rotate=not args.fix_flownet)
        log = LossLog(epoch_size, dev, trainer.hp['w2'] <= 0, args.batch_size)
        train_loss = run_epoch(trainer, loader, params, aug, log, args.print_freq, full, say)
        train_losses.append(train_loss)
        say(' * Avg Loss : {:.3f}'.format(train_loss))

        flow_errors = errors = None
        if framework is not None:
            flow_errors = validate_flow(trainer.nets, framework, args.batch_size, args.THRESH, args.data_normalization)
        if val_loader is not None:
            errors = validate_depth(trainer.nets['disp'], val_loader, dev, args.data_normalization)
            host = torch.stack(errors).tolist()
            error_string = ', '.join('{} : {:.3f}'.format(name, e) for name, e in zip(DEPTH_ERROR_NAMES, host))
            if args.log_terminal:
                say(' * Avg {}'.format(error_string))
            else:
                print('Epoch {} completed'.format(epoch))
        for net in trainer.nets.values():
            net.train()
        pyramid.clear()

        d = decisive_error(fixed, errors, flow_errors)
        if best_error < 0:
            best_error = d
        is_best = bool(d <= best_error)
        best_error = min(best_error, d)
        save_checkpoint(save_path, trainer, epoch + 1, is_best)
        write_rows(summary, [[train_loss, d]])
        decisive.append(d)
    return dict(save_path=save_path, train_losses=train_losses, decisive_errors=decisive, trainer=trainer)


if __name__ == '__main__':
    main()
