"""The training driver (cc_b200.train) without a GPU: the reference loaders' sample lists and decoded frames, the epoch's
order and augmentation draws, the decisive-error chain, the command line, and the reference's log and checkpoint files.
The driver's end-to-end epochs, its validation and --resume run on the H100 (tests/test_gpu_train_driver.py): a cfg3
step under the CPU simulator build takes minutes."""
import os
import numpy as np
import pytest
import torch

from cc_b200 import train as T
from tests import train_cases as TC
from tests.util import golden

README = ('DUMP --dispnet DispResNet6 --posenet PoseNetB6 --masknet MaskNet6 --flownet Back2Future '
          '--pretrained-disp d.tar --pretrained-pose p.tar --pretrained-flow f.tar --pretrained-mask m.tar '
          '-b4 -m0.1 -pf 0.5 -pc 1.0 -s0.1 -c0.3 --epoch-size 1000 -f 0 --nlevels 6 --lr 1e-4 -wssim 0.997 '
          '--with-flow-gt --with-depth-gt --epochs 100 --smoothness-type edgeaware  --fix-masknet --fix-flownet '
          '--log-terminal --name EXPERIMENT_NAME').split()


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    return TC.write_tree(str(tmp_path_factory.mktemp('train_tree')))


def _rel(root, samples):
    return np.array([[os.path.relpath(p, root) for p in s['frames']] for s in samples])


def test_tree_rebuilds_from_fixture(tree):
    g = golden('train_data_small')
    for i, n in enumerate(g['tree_names']):
        with open(os.path.join(tree, str(n)), 'rb') as f:
            assert f.read() == g['tree_%d' % i].tobytes(), n


@pytest.mark.parametrize('tag,seed,train', [('seq0', 0, True), ('seq3', 3, True), ('seqval', 0, False)])
def test_sequence_samples(tree, tag, seed, train):
    g = golden('train_data_small')
    root = os.path.join(tree, 'seq')
    s = T.sequence_samples(root, seed, train=train)
    np.testing.assert_array_equal(_rel(root, s), g[tag + '_frames'])
    np.testing.assert_array_equal(np.stack([x['K'] for x in s]), g[tag + '_K'])
    assert all(x['K'].dtype == np.float32 for x in s)


def test_stacked_and_validation_samples(tree):
    g = golden('train_data_small')
    root = os.path.join(tree, 'stacked')
    s = T.stacked_samples(root)
    np.testing.assert_array_equal([os.path.relpath(x['stack'], root) for x in s], g['stacked_files'])
    np.testing.assert_array_equal(np.stack([x['K'] for x in s]), g['stacked_K'])
    frames, K = T.FrameSet(s)[0]
    assert frames.dtype == torch.uint8
    np.testing.assert_array_equal(frames.numpy(), g['stacked0_frames'])
    np.testing.assert_array_equal(K.numpy(), g['stacked_K'][0])
    seq = os.path.join(tree, 'seq')
    v = T.validation_samples(seq)
    np.testing.assert_array_equal([os.path.relpath(a, seq) for a, _ in v], g['val_imgs'])
    np.testing.assert_array_equal([os.path.relpath(b, seq) for _, b in v], g['val_depth'])
    img, depth = T.DepthSet(v)[0]
    np.testing.assert_array_equal(img.numpy()[0], g['val0_img'])
    np.testing.assert_array_equal(depth.numpy(), g['val0_depth'])


def test_decoded_frames(tree):
    g = golden('train_data_small')
    ds = T.FrameSet(T.sequence_samples(os.path.join(tree, 'seq'), 0))
    for i in range(2):
        frames, K = ds[i]
        np.testing.assert_array_equal(frames.numpy(), g['seq0_%d_frames' % i])
        np.testing.assert_array_equal(K.numpy(), g['seq0_%d_K' % i])
        np.testing.assert_allclose(np.linalg.inv(K.numpy()), g['seq0_%d_Kinv' % i], rtol=1e-6)


def _epoch_batches(tree, workers, seed, epoch, B=2, epoch_size=0):
    ds = T.FrameSet(T.sequence_samples(os.path.join(tree, 'seq'), seed))
    order = T.epoch_order(len(ds), B, epoch_size, seed, epoch)
    return order, [(f.clone(), k.clone()) for f, k in T.make_loader(ds, order, B, workers, False)]


def test_epoch_depends_on_seed_and_epoch_only(tree):
    torch.manual_seed(123)
    state = torch.get_rng_state()
    o0, b0 = _epoch_batches(tree, 0, seed=4, epoch=1)
    o2, b2 = _epoch_batches(tree, 2, seed=4, epoch=1)
    assert torch.equal(torch.get_rng_state(), state), 'the epoch advanced the global torch generator'
    assert o0 == o2 and len(b0) == len(b2) == 2                 # 5 samples at B=2: drop_last leaves 2 batches
    for (f0, k0), (f2, k2) in zip(b0, b2):
        assert torch.equal(f0, f2) and torch.equal(k0, k2)
    assert f0.shape == (2, 5, TC.H, TC.W, 3) and f0.dtype == torch.uint8
    assert T.epoch_order(5, 2, 1, 4, 1) == o0[:2]              # --epoch-size cuts whole batches
    assert T.epoch_order(5, 2, 0, 4, 2) != o0 or T.epoch_order(5, 2, 0, 5, 1) != o0
    p1 = T.epoch_params(3, 2, TC.H, TC.W, 4, 1, rotate=True)
    random_state = np.random.get_state()
    p2 = T.epoch_params(3, 2, TC.H, TC.W, 4, 1, rotate=True)
    assert np.random.get_state()[1].tolist() == random_state[1].tolist()
    for a, b in zip(p1, p2):
        for k in a:
            np.testing.assert_array_equal(a[k], b[k])
    p3 = T.epoch_params(3, 2, TC.H, TC.W, 4, 2, rotate=True)
    assert any(not np.array_equal(a['offset_x'], b['offset_x']) or not np.array_equal(a['angle'], b['angle'])
               for a, b in zip(p1, p3))


def _chain(fix_pose, fix_disp, fix_flow, fix_mask, errors, flow_errors):
    """train.py:382-389 as written."""
    if not fix_pose:
        decisive_error = flow_errors[-2]
    elif not fix_disp:
        decisive_error = errors[0]
    elif not fix_flow:
        decisive_error = flow_errors[-1]
    elif not fix_mask:
        decisive_error = flow_errors[3]
    return decisive_error


def test_decisive_error_chain():
    import itertools
    errors, flow_errors = list(range(100, 106)), list(range(200, 208))
    for bits in itertools.product((False, True), repeat=4):
        fixed = tuple(n for n, b in zip(T.NETS, bits) if b)
        if len(fixed) == 4:
            continue
        flags = dict(zip(T.NETS, bits))
        want = _chain(flags['pose'], flags['disp'], flags['flow'], flags['mask'], errors, flow_errors)
        assert T.decisive_error(fixed, errors, flow_errors) == want, fixed
        # the reference raises NameError after its first epoch when the chain reads an error it did not compute
        for depth_gt, flow_gt in itertools.product((False, True), repeat=2):
            try:                                          # an empty list stands for the undefined name
                _chain(flags['pose'], flags['disp'], flags['flow'], flags['mask'], errors if depth_gt else [],
                       flow_errors if flow_gt else [])
                ref_ok = True
            except IndexError:
                ref_ok = False
            argv = ['D', '--name', 'x'] + ['--fix-%snet' % n for n in fixed] + \
                (['--with-depth-gt'] if depth_gt else []) + (['--with-flow-gt'] if flow_gt else [])
            if ref_ok:
                T.parse_args(argv)
            else:
                with pytest.raises(SystemExit):
                    T.parse_args(argv)


@pytest.mark.parametrize('flag,name', [
    ('--robust', '--robust'), ('--joint-mask-for-depth', '--joint-mask-for-depth'),
    ('--no-non-rigid-mask', '--no-non-rigid-mask'), ('--spatial-normalize', '--spatial-normalize'),
    ('--sequence-length 3', '--sequence-length'), ('--nlevels 5', '--nlevels'), ('--weight-decay 0.1', '--weight-decay'),
    ('--log-output', '--log-output'), ('-f 2', '--training-output-freq'), ('--DEBUG', '--DEBUG'),
    ('--dispnet DispNetS', '--dispnet'), ('--posenet PoseNet', '--posenet'), ('--masknet MaskNet', '--masknet'),
    ('--flownet FlowNetS', '--flownet')])
def test_refused_flags(flag, name, capsys):
    with pytest.raises(SystemExit):
        T.parse_args(['D', '--name', 'x', '--with-flow-gt'] + flag.split())
    assert name in capsys.readouterr().err


def test_readme_command_parses():
    args = T.parse_args(README)
    assert (args.dispnet, args.posenet, args.masknet, args.flownet) == ('DispResNet6', 'PoseNetB6', 'MaskNet6', 'Back2Future')
    assert T.fixed_nets(args) == ('mask', 'flow') and args.batch_size == 4 and args.epoch_size == 1000
    hp = T.hyper_parameters(args)
    assert (hp['w1'], hp['w2'], hp['w3'], hp['w4'], hp['w5']) == (1.0, 0.1, 0.1, 0.5, 0.3)
    assert hp['wssim'] == 0.997 and hp['smoothness'] == 'edgeaware' and hp['lr'] == 1e-4
    ignored = T.parse_args(README + ['--alternating', '--clamp-masks', '--fix-posemasknet', '-e', '--rotation-mode', 'quat',
                                     '--padding-mode', 'border'])
    assert T.fixed_nets(ignored) == ('mask', 'flow')


def test_meter_and_csv_bytes(tmp_path):
    g = golden('train_data_small')
    m = T.AverageMeter(6)
    acc, n = torch.zeros(6), 0
    for row in g['meter_in']:
        m.update([torch.tensor(v) for v in row])
        acc += torch.from_numpy(row)
        n += 1
    dev_avg = acc / n                                        # validate_depth's device restatement
    np.testing.assert_array_equal(np.array([float(a) for a in m.avg], np.float32), g['meter_avg'])
    np.testing.assert_array_equal(dev_avg.numpy(), g['meter_avg'])
    assert str(dev_avg[0]) == str(g['meter_str'])
    full, summary = tmp_path / 'full.csv', tmp_path / 'summary.csv'
    T.write_rows(full, [T.FULL_HEADER], 'w')
    log = T.LossLog(3, 'cpu', False, 4)
    log.rows.copy_(torch.from_numpy(g['csv_full_rows']))
    rows = log.flush(3)
    rows[1][2] = 0                                           # the fixture's second row was written with w2 == 0
    T.write_rows(full, rows)
    assert full.read_bytes() == g['csv_full'].tobytes()
    T.write_rows(summary, [T.SUMMARY_HEADER], 'w')
    T.write_rows(summary, [[float(g['csv_full_rows'][0, 0]), dev_avg[0]]])
    assert summary.read_bytes() == g['csv_summary'].tobytes()
    w2_zero = T.LossLog(2, 'cpu', True, 4)
    w2_zero.rows.copy_(torch.from_numpy(g['csv_full_rows'][:2]))
    r = w2_zero.flush(2)
    assert r[0][2] == 0 and type(r[0][2]) is int and type(r[0][0]) is float
    losses = [float(v) for v in g['csv_full_rows'][:2, 0]]
    assert w2_zero.meter.avg[0] == (losses[0] * 4 + losses[1] * 4) / 8


def test_flush_reports_the_meter_as_of_each_step():
    """The terminal line of step j shows the loss meter after step j (train.py:563,579-580), not after the flush."""
    log = T.LossLog(4, 'cpu', True, 2)
    log.rows[:, 0] = torch.tensor([1.0, 2.0, 3.0, 4.0])
    seen = {}
    log.flush(3, lambda j: seen.__setitem__(j, (log.meter.val[0], log.meter.avg[0])))
    assert seen == {0: (1.0, 1.0), 1: (2.0, 1.5), 2: (3.0, 2.0)}
    log.flush(4, lambda j: seen.__setitem__(j, (log.meter.val[0], log.meter.avg[0])))
    assert seen[3] == (4.0, 2.5) and log.done == 4


def test_checkpoint_files_and_optimizer(tmp_path, sim_lib):
    from cc_b200.train_step import Trainer
    import itertools
    tr = Trainer('cfg3', 'cpu', fixed=('mask', 'flow'))
    k = sum(p.numel() for n in ('disp', 'pose') for p in tr.nets[n].parameters())
    with torch.no_grad():                                    # a fake step's Adam state for disp and pose
        tr.opt.exp_avg[:k].uniform_(-1, 1)
        tr.opt.exp_avg_sq[:k].uniform_(0, 1)
        tr.opt.state.view(-1, 4)[:2, 0] = 3
    T.save_checkpoint(str(tmp_path), tr, 2, is_best=True)
    T.save_checkpoint(str(tmp_path), tr, 3, is_best=False)
    names = sorted(os.listdir(tmp_path))
    assert names == sorted(['%s_%s' % (p, s) for p in T.CKPT_PREFIXES for s in ('checkpoint.pth.tar', 'model_best.pth.tar')])
    for n, prefix in zip(T.NETS, T.CKPT_PREFIXES):
        ck = torch.load(tmp_path / (prefix + '_checkpoint.pth.tar'))
        best = torch.load(tmp_path / (prefix + '_model_best.pth.tar'))
        assert set(ck) == {'epoch', 'state_dict'} and ck['epoch'] == 3 and best['epoch'] == 2
        sd = ck['state_dict']
        assert list(sd) == list(tr.nets[n].state_dict()) and not any(k.startswith('module.') for k in sd)
        for k, v in tr.nets[n].state_dict().items():
            assert torch.equal(sd[k], v.cpu())
            assert sd[k].untyped_storage().nbytes() == sd[k].numel() * sd[k].element_size(), k
    opt = torch.load(tmp_path / 'optimizer_checkpoint.pth.tar')['state_dict']
    params = [torch.nn.Parameter(p.detach().clone()) for p in itertools.chain(*(tr.nets[n].parameters() for n in T.NETS))]
    adam = torch.optim.Adam(params, lr=1e-4)
    adam.load_state_dict(opt)
    n_dp = sum(1 for n in ('disp', 'pose') for _ in tr.nets[n].parameters())
    assert len(adam.state) == n_dp and float(adam.state[params[0]]['step']) == 3
    # a reference-format (torch.optim.Adam) state dict loads back through --resume
    fresh = Trainer('cfg3', 'cpu', seed=1, fixed=('mask', 'flow'))
    T.load_resume(str(tmp_path), fresh)
    assert fresh.opt.group_steps() == [3, 3, 0, 0]
    assert torch.equal(fresh.opt.exp_avg, tr.opt.exp_avg) and torch.equal(fresh.opt.flat_p, tr.opt.flat_p)


from tests.util import sim_lib      # noqa: E402,F401  (module fixture: the simulator library)
