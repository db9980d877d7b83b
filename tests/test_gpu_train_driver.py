"""The training driver (cc_b200.train) on the H100: main() end to end with depth validation, the driver's graph-replayed
epoch against eager Trainer.steps on the same augmented batches, no host synchronisation between log flushes, --resume,
--workers, and both validations against their restatements."""
import os
import numpy as np
import pytest
import torch

from cc_b200 import train as T, nn as cnn, evaluate as EV, loss_functions as LF
from cc_b200.input_pipeline import DeviceAugment
from cc_b200.train_step import Trainer
from oracle import metrics as OM
from tests import train_cases as TC, flow_eval_cases as FC
from tests.step_cases import _record, _assert_same
from tests.util import device_lib, assert_close      # noqa: F401  (module fixture: the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]
DEV = torch.device('cuda:0')
CANON = ('mask', 'flow')


@pytest.fixture(autouse=True)
def _graph_live():
    saved = cnn.GRAPH_LIVE
    yield
    cnn.GRAPH_LIVE = saved
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _epoch_inputs(root, B, steps, seed=0, epoch=0, workers=0, rotate=False):
    ds = T.FrameSet(T.sequence_samples(root, seed))
    order = T.epoch_order(len(ds), B, steps, seed, epoch)
    assert len(order) == B * steps, (len(ds), B, steps)
    H, W = ds[0][0].shape[1:3]
    params = T.epoch_params(steps, B, H, W, seed, epoch, rotate)
    return ds, order, params


def _graph_epoch(root, B, steps, fixed=CANON, workers=0, log_cls=T.LossLog, print_freq=10, epoch=0):
    ds, order, params = _epoch_inputs(root, B, steps, epoch=epoch, rotate='flow' not in fixed)
    tr = Trainer('cfg3', DEV, fixed=fixed)
    aug = DeviceAugment(DEV, rotate='flow' not in fixed)
    log = log_cls(steps, DEV, tr.hp['w2'] <= 0, B)
    loss = T.run_epoch(tr, T.make_loader(ds, order, B, workers, True), params, aug, log, print_freq)
    torch.cuda.synchronize()
    return tr, log, loss


def _eager_epoch(root, B, steps, fixed=CANON, epoch=0):
    ds, order, params = _epoch_inputs(root, B, steps, epoch=epoch, rotate='flow' not in fixed)
    tr = Trainer('cfg3', DEV, fixed=fixed)
    aug = DeviceAugment(DEV, rotate='flow' not in fixed)
    rows = []
    for i in range(steps):
        batch = [ds[j] for j in order[i * B:(i + 1) * B]]
        frames, K = torch.stack([b[0] for b in batch]), torch.stack([b[1] for b in batch])
        tgt, refs, Kd, Kinv = aug(frames.to(DEV), K.numpy(), params=params[i], tgt_index=0)
        loss, aux = tr.step(tgt, refs, Kd, Kinv)
        rows.append(torch.stack([loss, aux['loss_1'], torch.zeros((), device=DEV) if tr.hp['w2'] <= 0 else aux['loss_2'],
                                 aux['loss_3'], aux['loss_4']]).detach())
    torch.cuda.synchronize()
    return tr, torch.stack(rows)


@pytest.mark.parametrize('size', [(2, 64, 128, 2, CANON), (4, 256, 832, 3, CANON), (2, 64, 128, 3, ('mask',))],
                         ids=lambda s: 'b%d_%dx%d_fixed_%s' % (s[:3] + ('_'.join(s[4]),)))
def test_graph_epoch_equals_eager(tmp_path, size):
    """The driver's epoch (capture on the first batch, HostFeeder, DeviceAugment into the graph's inputs, replay) equals
    eager Trainer.steps on the same augmented batches bit for bit: parameters, gradients, Adam moments and step counts,
    BatchNorm buffers and the logged loss rows.  With the flow net trained, the augmentation rotates (RandomRotate)."""
    B, H, W, steps, fixed = size
    epoch = 0 if 'flow' in fixed else 1                    # seed 0's epoch 1 rotates samples of its first batches
    root = TC.write_synth_dump(str(tmp_path / 'dump'), scenes=1, frames=B * steps + 4, H=H, W=W)
    if 'flow' not in fixed:
        assert any(p['rotate'].any() for p in _epoch_inputs(root, B, steps, epoch=epoch, rotate=True)[2]), 'no rotation'
    tr, rows = _eager_epoch(root, B, steps, fixed, epoch)
    want = _record(tr)
    want_rows = rows.clone()
    del tr
    torch.cuda.empty_cache()
    tr, log, loss = _graph_epoch(root, B, steps, fixed, workers=2, epoch=epoch)
    assert tr.graph is not None
    _assert_same(_record(tr), want, 'driver epoch vs eager steps', skip=('flat_g',))
    assert torch.equal(tr.opt.flat_g, want['flat_g'])
    assert torch.equal(log.rows, want_rows), (log.rows, want_rows)
    host = want_rows.cpu().tolist()
    m = T.AverageMeter()
    for r in host:
        m.update(r[0], B)
    assert loss == m.avg[0]
    assert tr.opt.group_steps() == [0 if n in fixed else steps for n in T.NETS]


@pytest.mark.parametrize('fixed', [CANON, ('mask',)], ids=lambda f: 'fixed_' + '_'.join(f))
def test_no_host_sync_between_flushes(tmp_path, fixed):
    """Steady-state steps (after the capture) run under torch.cuda.set_sync_debug_mode('error'); only the log flush, once
    per --print-freq steps, reads the device.  With the flow net trained the augmentation rotates."""

    class Guarded(T.LossLog):
        def record(self, i, loss, terms):
            super().record(i, loss, terms)
            if i == 0:
                torch.cuda.set_sync_debug_mode('error')     # the capture (step 0) synchronises; the rest must not

        def flush(self, upto, on_row=None):
            torch.cuda.set_sync_debug_mode(0)
            try:
                return super().flush(upto, on_row)
            finally:
                torch.cuda.set_sync_debug_mode('error')

    root = TC.write_synth_dump(str(tmp_path / 'dump'), scenes=1, frames=16, H=64, W=128)
    epoch = 0 if 'flow' in fixed else 1
    if 'flow' not in fixed:
        assert any(p['rotate'].any() for p in _epoch_inputs(root, 2, 6, epoch=epoch, rotate=True)[2][1:]), 'no rotation'
    try:
        tr, log, _ = _graph_epoch(root, 2, 6, fixed, workers=2, log_cls=Guarded, print_freq=3, epoch=epoch)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert log.done == 6
    if 'flow' in fixed:
        # on this synthetic dump the reference's photometric loss is infinite for the first rotated batch at the initial
        # weights (oracle.step.loss_cfg3 on the CPU gives the same), so only the unrotated run is held to finite losses
        assert bool(torch.isfinite(log.rows).all())


def test_resume_step_equals_uninterrupted(tmp_path):
    """A trainer rebuilt from written checkpoints (--resume) takes one step on batch X equal to the uninterrupted trainer's
    next step on X bit for bit, with the canonical fixed set (per-net Adam step counts 2, 2, 0, 0)."""
    root = TC.write_synth_dump(str(tmp_path / 'dump'), scenes=1, frames=10, H=64, W=128)
    ds, order, params = _epoch_inputs(root, 2, 3)
    aug = DeviceAugment(DEV)

    def batch(i):
        b = [ds[j] for j in order[2 * i:2 * i + 2]]
        return aug(torch.stack([x[0] for x in b]).to(DEV), torch.stack([x[1] for x in b]).numpy(), params=params[i],
                   tgt_index=0)

    a = Trainer('cfg3', DEV, fixed=CANON)
    for i in range(2):
        a.step(*batch(i))
    save = str(tmp_path / 'ck')
    os.makedirs(save)
    T.save_checkpoint(save, a, 1, True)
    b = Trainer('cfg3', DEV, seed=7, fixed=CANON)
    T.load_resume(save, b)
    assert b.opt.group_steps() == [2, 2, 0, 0]
    x = batch(2)
    la, _ = a.step(*x)
    lb, _ = b.step(*x)
    _assert_same(_record(b, lb), _record(a, la), 'resumed step vs uninterrupted step')


def _main(tmp_path, tag, root, workers, extra=()):
    cwd = os.getcwd()
    os.makedirs(tmp_path / tag, exist_ok=True)
    os.chdir(tmp_path / tag)
    try:
        return T.main([root, '--name', 'x', '-b', '2', '--epochs', '2', '--epoch-size', '2', '--workers', str(workers),
                       '--with-depth-gt', '--fix-posenet', '--fix-masknet', '--fix-flownet', '--print-freq', '1',
                       '--log-terminal'] + list(extra), device=DEV)
    finally:
        os.chdir(cwd)


def test_main_files_and_workers(tmp_path):
    """main() on the fixture's tree: two epochs of two steps with depth validation write the five checkpoints, the best
    copies and both logs; --workers 0 and 2 write identical checkpoint tensors and loss rows; the files load through
    the evaluation loaders."""
    root = os.path.join(TC.write_tree(str(tmp_path / 'tree')), 'seq')
    runs = {}
    for w in (0, 2):
        out = _main(tmp_path, 'w%d' % w, root, w)
        runs[w] = os.path.join(tmp_path, 'w%d' % w, out['save_path'])
        assert len(out['decisive_errors']) == 2 and out['decisive_errors'][0].dim() == 0
        del out
        torch.cuda.empty_cache()
    names = set(os.listdir(runs[0]))
    for p in T.CKPT_PREFIXES:
        assert {p + '_checkpoint.pth.tar', p + '_model_best.pth.tar'} <= names
    for p in T.CKPT_PREFIXES:
        a = torch.load(os.path.join(runs[0], p + '_checkpoint.pth.tar'), map_location='cpu')
        b = torch.load(os.path.join(runs[2], p + '_checkpoint.pth.tar'), map_location='cpu')
        assert a['epoch'] == b['epoch'] == 2
        sa, sb = a['state_dict'], b['state_dict']
        if p == 'optimizer':
            sa, sb = sa['state'], sb['state']
            assert sa.keys() == sb.keys() and len(sa) > 0
            for k in sa:
                for kk in sa[k]:
                    assert torch.equal(sa[k][kk].cpu(), sb[k][kk].cpu()), (p, k, kk)
        else:
            for k in sa:
                assert torch.equal(sa[k], sb[k]), (p, k)
    for f in ('progress_log_full.csv', 'progress_log_summary.csv'):
        with open(os.path.join(runs[0], f)) as fa, open(os.path.join(runs[2], f)) as fb:
            assert fa.read() == fb.read(), f
    with open(os.path.join(runs[0], 'progress_log_full.csv')) as f:
        lines = f.read().splitlines()
    assert lines[0] == '\t'.join(T.FULL_HEADER) and len(lines) == 5
    assert all(len(r.split('\t')) == 5 and r.split('\t')[2] == '0' for r in lines[1:])
    with open(os.path.join(runs[0], 'progress_log_summary.csv')) as f:
        lines = f.read().splitlines()
    assert lines[0] == 'train_loss\tvalidation_loss' and len(lines) == 3
    assert lines[1].split('\t')[1].startswith('tensor(') and "device='cuda:0'" in lines[1]
    ck = lambda p: os.path.join(runs[0], p + '_checkpoint.pth.tar')     # noqa: E731
    nets = EV.load_flow_eval_nets(ck('dispnet'), ck('posenet'), ck('masknet'), ck('flownet'))
    pose, seq = EV.load_pose_net(ck('posenet'))
    assert seq == 5 and len(nets) == 4


def test_depth_validation(tmp_path):
    """validate_depth against compute_errors' oracle on the same predictions, and its device sums against a host
    restatement of AverageMeter over the same per-batch 0-dim tensors."""
    root = os.path.join(TC.write_tree(str(tmp_path / 'tree')), 'seq')
    tr = Trainer('cfg3', DEV, fixed=CANON)
    vs = T.DepthSet(T.validation_samples(root))
    loader = T.make_loader(vs, list(range(len(vs))), 2, 0, True)
    got = T.validate_depth(tr.nets['disp'], loader, DEV)
    aug = DeviceAugment(DEV, flip=False, scale_crop=False)
    meter = T.AverageMeter(6)
    with torch.no_grad():
        for frames, depth in loader:
            tgt = aug(frames.to(DEV), np.tile(np.eye(3, dtype=np.float32), (frames.shape[0], 1, 1)))[0]
            pred = (1 / tr.nets['disp'](tgt)).squeeze(1)
            errs = LF.compute_errors(depth.to(DEV), pred)
            meter.update(errs)
            want = torch.stack([torch.as_tensor(v) for v in OM.compute_errors(depth, pred.cpu())])
            assert_close(torch.stack(errs).cpu(), want, 1e-5, 'compute_errors on the driver predictions')
    assert meter.count == len(vs) // 2
    for g, w in zip(got, meter.avg):
        assert torch.equal(g, w), (g, w)
    assert str(got[0]) == str(meter.avg[0])


def test_flow_validation(tmp_path):
    """validate_flow on a written KITTI-2015 tree equals AverageMeter over flow_eval_batch's rows in sample order, and the
    canonical fixed set's decisive error is column -2, epe_non_rigid_with_gt_mask (train.py:641; the comment at
    train.py:383 misnames it).  With --data-normalization local the frames are normalised locally: the averages differ
    from the global ones and equal AverageMeter over flow_eval_batch's local rows, whose frames match a restatement of
    NormalizeLocally."""
    root = str(tmp_path / 'kitti')
    FC.write_flow_tree(root)
    fw = EV.kitti_flow_framework(root, N=FC.TREE_N)
    tr = Trainer('cfg3', DEV, fixed=CANON)
    avgs = {}
    for norm in ('global', 'local'):
        got = T.validate_flow(tr.nets, fw, 2, normalization=norm)
        rows = {}
        for idx in fw['groups'].values():
            for c in range(0, len(idx), 2):
                s = EV.load_kitti_flow_samples(fw, idx[c:c + 2])
                out = EV.flow_eval_batch(tr.nets['disp'], tr.nets['pose'], tr.nets['mask'], tr.nets['flow'], s['frames'],
                                         s['K'], s['gt'], s['obj'], normalization=norm)
                rows.update({i: out[k] for k, i in enumerate(idx[c:c + 2])})
        meter = T.AverageMeter(8)
        for i in range(FC.TREE_N):
            meter.update([rows[i][k] for k in range(8)])
        for g, w in zip(got, meter.avg):
            assert torch.equal(g, w), (norm, g, w)
        avgs[norm] = torch.stack(got)
        assert T.decisive_error(CANON, None, got) is got[6]
        assert T.decisive_error(('pose', 'disp', 'mask'), None, got) is got[7]
    assert not torch.equal(avgs['global'], avgs['local'])
    # NormalizeLocally (custom_transforms.py:33-44) restated in fp64 on the globally normalised frames of one batch
    s = EV.load_kitti_flow_samples(fw, fw['groups'][next(iter(fw['groups']))][:2])
    glob = EV._flow_frames(s['frames'], 256, 832, 'global')
    loc = EV._flow_frames(s['frames'], 256, 832, 'local')
    v = torch.stack(glob, 1).double() * 0.5 + 0.5                      # [B,F,3,h,w] in [0, 1]
    flat = v.transpose(1, 2).reshape(v.shape[0], 3, -1)
    want = (v - flat.mean(2)[:, None, :, None, None]) / flat.std(2)[:, None, :, None, None]
    assert_close(torch.stack(loc, 1), want, 1e-5, 'local flow-validation frames')
