"""KITTI-2015 flow evaluation without a GPU: the oracle (oracle/flow_eval.py) against the numbers frozen from the
reference's own ValidationFlow, flow_read_png, compute_all_epes and test_flow.py's sample body
(tests/golden/flow_eval_small.npz), the loaders of cc_b200.evaluate and of the oracle against the frozen framework on the
same tree, the printed row and the output files, then ccb_flow_eval compiled by g++ against the CPU execution-model
simulator (tests/sim) against the fixture and the oracle.  The same kernel cases run on the H100 in
tests/test_gpu_flow_eval.py."""
import os
import numpy as np
import pytest
import torch
from cc_b200 import evaluate as CE
from oracle import flow_eval as OF
from tests import flow_eval_cases as FC, workspace_cases as WC
from tests.util import sim_lib      # noqa: F401  (module fixture: the simulator library)

CPU = torch.device('cpu')


@pytest.mark.parametrize('name', list(FC.CASES))
def test_oracle_equals_reference(name):
    d = FC.g()
    T, ET = FC.CASES[name][4:6]
    ins = FC.case_inputs(name)
    if name in FC.STORED:
        assert all(np.array_equal(a, b) for a, b in zip(ins, FC.stored_inputs(name))), 'the seeded inputs moved'
    errs, comb = OF.sample_errors(*(torch.from_numpy(a) for a in ins), THRESH=T, epe_thresh=ET)
    assert np.array_equal(np.array(errs), d[name + '_out'])
    assert np.array_equal(np.array(OF.back2future_errors(*(torch.from_numpy(ins[k]) for k in (2, 3, 4)), epe_thresh=ET)),
                          d[name + '_b2f'])
    want = d[name + '_mask'] if name != 'kitti' else \
        np.unpackbits(d['kitti_mask_bits'])[:256 * 832].reshape(1, 1, 256, 832).astype(np.float32)
    assert np.array_equal(comb.numpy(), want)


@pytest.fixture(scope='module')
def written_tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('kitti2015'))
    FC.write_flow_tree(root)
    return root


def test_oracle_loader_rebuilds_the_reference(written_tree):
    d = FC.g()
    for i in range(FC.TREE_N):
        tgt, refs, K, Kinv, gt, obj = OF.load_sample(written_tree, i)
        assert np.array_equal(np.stack([tgt] + refs), d['tree_%d_frames' % i])
        assert np.array_equal(gt, d['tree_%d_gt' % i]) and np.array_equal(K, d['tree_%d_K' % i])
        assert np.array_equal(Kinv, d['tree_%d_Kinv' % i]) and Kinv.dtype == d['tree_%d_Kinv' % i].dtype
        assert obj.dtype == d['tree_%d_obj' % i].dtype and np.array_equal(obj, d['tree_%d_obj' % i])
    assert np.array_equal(OF.load_sample(written_tree, 0, occ='flow_noc')[4], d['tree_noc_gt0'])


def test_framework_rebuilds_the_reference(written_tree):
    """kitti_flow_framework and load_kitti_flow_samples on the same tree: files, frame sizes and their groups, and per
    size group the frames, gt, obj (ones where obj_map is missing) and K bit for bit."""
    d = FC.g()
    fw = CE.kitti_flow_framework(written_tree, N=FC.TREE_N)
    assert fw['groups'] == {(14, 40): [0, 1, 3], (12, 44): [2]}
    assert [s['size'] for s in fw['samples']] == [FC.TREE_SIZES[i] for i in range(FC.TREE_N)]
    assert [os.path.basename(f) for f in fw['samples'][1]['frames']] == ['000001_%s.png' % k for k in ('10', '08', '09', '11', '12')]
    assert fw['samples'][2]['obj'] is None and all(fw['samples'][i]['obj'] for i in (0, 1, 3))
    for idx in fw['groups'].values():
        s = CE.load_kitti_flow_samples(fw, idx)
        for k, i in enumerate(idx):
            assert np.array_equal(s['frames'][k], d['tree_%d_frames' % i]) and s['frames'].dtype == np.uint8
            assert np.array_equal(s['gt'][k], d['tree_%d_gt' % i]) and s['gt'].dtype == np.float32
            assert np.array_equal(s['obj'][k], d['tree_%d_obj' % i]) and s['obj_found'][k] == (i != 2)
            assert np.array_equal(s['K'][k], d['tree_%d_K' % i]) and s['K'].dtype == np.float32
    noc = CE.kitti_flow_framework(written_tree, occ='flow_noc', N=1)
    assert np.array_equal(CE.load_kitti_flow_samples(noc, [0])['gt'][0], d['tree_noc_gt0'])
    with pytest.raises(AssertionError, match='one frame size'):
        CE.load_kitti_flow_samples(fw, [1, 2])


def test_summary_is_the_printed_row():
    """flow_summary of the tree samples' numbers equals AverageMeter's averages bit for bit, and the row is the script's."""
    d = FC.g()
    per = np.stack([d['tree_%d_out' % i] for i in range(FC.TREE_N)]).astype(np.float32)
    avg, row = CE.flow_summary(per)
    assert avg == d['tree_avg'].tolist() and OF.summary(per.tolist()) == d['tree_avg'].tolist()
    assert row == 'Errors \t ' + ', '.join('{:10.4f}'.format(v) for v in d['tree_avg'])
    avg4, row4 = CE.flow_summary(per[:, 4:])
    assert avg4 == d['tree_avg'][4:].tolist() and row4.startswith('Averge EPE [')


def test_output_files(tmp_path):
    d = FC.g()
    tgt, mask = torch.rand(1, 3, 8, 16), torch.from_numpy(d['tree_0_mask'])
    for i, found in ((0, True), (2, False)):
        obj = d['tree_%d_obj' % i][None]
        CE.write_flow_eval_outputs(str(tmp_path), i, tgt, mask, obj, found)
        got = np.load(str(tmp_path / 'gt' / ('%03d.npy' % i)))
        assert got.dtype == d['tree_%d_obj' % i].dtype and np.array_equal(got, d['tree_%d_obj' % i])
    assert np.array_equal(np.load(str(tmp_path / 'mask' / '000.npy')), d['tree_0_mask'][0])
    assert np.array_equal(np.load(str(tmp_path / 'images' / '002.npy')), tgt[0].numpy())


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('case', FC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(CPU)


@pytest.mark.usefixtures('sim_lib')
def test_tree_samples():
    """The tree samples' frozen script-body numbers and masks from ccb_flow_eval, one batch per frame size."""
    d = FC.g()
    for idx in ([0, 1, 3], [2]):
        ins = [FC.tree_net_outputs(i) for i in idx]
        emask, cam, fwd = (torch.from_numpy(np.concatenate(a)) for a in zip(*ins))
        gt = torch.from_numpy(np.stack([d['tree_%d_gt' % i] for i in idx]))
        obj = torch.from_numpy(np.stack([d['tree_%d_obj' % i] for i in idx]).astype(np.float32))
        out, mask = CE.flow_eval(emask, cam, fwd, gt, obj, 0.01, want_mask=True)
        for k, i in enumerate(idx):
            assert np.array_equal(mask[k].numpy(), d['tree_%d_mask' % i][0])
            FC._close(out[k].numpy(), d['tree_%d_out' % i], FC.BAR, i)


@pytest.mark.usefixtures('sim_lib')
def test_workspace_row(monkeypatch):
    WC.check_row(CPU, WC.Row('flow_eval', 16, 17, [15, 18], FC._flow_eval_row,
                             ('ccb_flow_eval_workspace_bytes', (1, 16, 0, 25, 61))), monkeypatch)


@pytest.mark.parametrize('choice', [('DispResNet6', 'PoseNetB6', 'MaskNet6', 'Back2Future'),
                                    ('DispNetS6', 'PoseNet6', 'MaskResNet6', 'FlowNetC6')])
def test_load_flow_eval_nets(choice, tmp_path):
    """The four checkpoints loaded strictly from ['state_dict'], pose and mask nets built for 4 references."""
    from cc_b200 import models as CM, synth
    paths = []
    for k, name in enumerate(choice):
        kw = {'nb_ref_imgs': 4} if k in (1, 2) else {'nlevels': 6} if k == 3 else {}
        net = synth.seeded_fill(getattr(CM, name)(**kw), 10 + k)
        paths.append(str(tmp_path / ('%d.pth.tar' % k)))
        torch.save({'state_dict': net.state_dict(), 'epoch': 1}, paths[-1])
    nets = CE.load_flow_eval_nets(*paths, *choice, device=CPU)
    for k, net in enumerate(nets):
        assert type(net).__name__ == (choice[k] if choice[k] != 'Back2Future' else 'Model') and not net.training
        src = torch.load(paths[k])['state_dict']
        assert all(torch.equal(v, src[n]) for n, v in net.state_dict().items())
    assert nets[1].nb_ref_imgs == 4
