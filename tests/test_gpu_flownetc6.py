"""FlowNetC6 on the H100: the cost-volume kernels at the benchmark shape, the network against the fixture frozen from
the reference module, the training step with --flownet FlowNetC6 against the CPU oracle, CUDA-graph replay against eager
steps, and the flow evaluation."""
import numpy as np
import pytest
import torch
from cc_b200 import _lib, nn as cnn, models as CM, pyramid, synth, evaluate as CE
from cc_b200.train_step import Trainer, HP
from oracle import step as OS, evaluate as OE, nets as ON
from tests import flownetc6_cases as FC, flownetc6_oracle as O6, step_cases as SC
from tests.util import rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


@pytest.fixture(scope='module', autouse=True)
def cuda_lib():
    _lib._lib = None                      # the real library, not a simulator build
    assert not _lib.is_simulator(), 'GPU tests must run on the sm_90a library'
    pyramid.clear()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def test_corr441d_benchmark_shape_vs_fp64():
    """[4,256,32,104] (conv3 of a 256x832 frame) and the small shapes: element-wise bound, bit-identical reruns.
    The kernels take no workspace, so there is no workspace size for a result to depend on."""
    worst = FC.case_corr441d(DEV, shapes=FC.CORR_SHAPES + [(4, 256, 32, 104)])
    print('corr441d worst r:', {s: {k: round(v, 3) for k, v in r.items()} for s, r in worst.items()})


def test_flownetc6_vs_fixture():
    """Default dispatch (wgmma tensor-core convolutions): outputs and eval output within 1e-4, gradients within 2e-3."""
    saved = cnn.CONV_IMPL
    cnn.CONV_IMPL = _lib.IMPL_AUTO
    try:
        net = CM.FlowNetC6()
        net.load_state_dict(FC.fixture_weights())
        net = net.to(DEV).train()
        tgt, ref = FC.fixture_inputs(DEV)
        outs = net(tgt, ref)
        assert len(outs) == 6
        loss = sum((x * FC._wts(x.shape, FC.WTS_SEED + i, DEV)).sum() for i, x in enumerate(outs))
        pd = dict(net.named_parameters())
        names = FC.grad_names()
        grads = dict(zip(names, torch.autograd.grad(loss, [pd[n] for n in names])))
        net.eval()
        with torch.no_grad():
            ev = net(tgt, ref)
        FC.check_against_fixture(outs, grads, ev, 1e-4, 2e-3)
    finally:
        cnn.CONV_IMPL = saved


GRAPH_CASES = [('cfg2', 2, 64, 128, 1e-3), ('cfg3', 2, 64, 128, 1e-3), ('cfg3', 4, 256, 832, None)]


@pytest.mark.parametrize('cfg,B,H,W,loss_tol', GRAPH_CASES, ids=['%s-b%d-%dx%d' % c[:4] for c in GRAPH_CASES])
def test_flownetc6_step_graph_replay_vs_eager(cfg, B, H, W, loss_tol):
    """Trainer(cfg, flownet='FlowNetC6'): three capture()d replays equal three eager steps bit for bit (loss, flat gradient,
    parameters, Adam moments and state, buffers); each replay's Adam update against fp64; the eager losses of steps 0-2
    against the CPU oracle step (loss_tol, the bar tests/test_gpu_parity.py GRAPH_CASES uses at that size)."""
    batches = []
    for i in range(3):
        tgt, refs = synth.frames(B, H, W, seed=80 + i)
        batches.append([tgt] + refs + list(synth.intrinsics(B, H, W)))
    P = O6.make_params(cfg)
    sd = SC._oracle_params_as_state_dicts(P)
    saved = (cnn.GRAPH_LIVE, cnn.CONV_IMPL)
    tr = None
    try:
        cnn.CONV_IMPL = _lib.IMPL_AUTO
        tr = Trainer(cfg, DEV, state_dicts=sd, flownet='FlowNetC6')
        assert isinstance(tr.nets['flow'], CM.FlowNetC6)
        eager = []
        for b in batches:
            d = [t.to(DEV) for t in b]
            loss, _ = tr.step(d[0], d[1:5], d[5], d[6])
            eager.append(SC._record(tr, loss))
        del tr, loss, d
        tr = None
        torch.cuda.empty_cache()

        tr = Trainer(cfg, DEV, state_dicts=sd, flownet='FlowNetC6')
        static = [t.to(DEV) for t in batches[0]]
        snap = SC._record(tr)
        tr.capture(static[0], static[1:5], static[5], static[6])
        SC._assert_same(SC._record(tr), snap, f'{cfg}: state after capture()', skip=('flat_g',))
        assert tr.wcache is not None and tr.wcache.committed
        prev, o = snap, tr.opt
        for i, b in enumerate(batches):
            for s, h in zip(static, b):
                s.copy_(h)
            cur = SC._record(tr, tr.replay())
            SC._assert_same(cur, eager[i], f'{cfg}: replay {i} vs eager step {i}')
            SC.assert_adam_step((prev['flat_p'], prev['exp_avg'], prev['exp_avg_sq']),
                                (cur['flat_p'], cur['exp_avg'], cur['exp_avg_sq'], cur['state']), cur['flat_g'], i + 1,
                                o.lr, o.betas, o.eps, o.grad_scale, f'{cfg}: Adam of replay {i}')
            prev = cur
        stats = tr.wcache.stats()
        assert stats['hits'] > 0 and stats['misses'] == 0, stats
    finally:
        if tr is not None:
            tr.graph = None
        tr = None
        torch.cuda.synchronize()
        cnn.GRAPH_LIVE, cnn.CONV_IMPL = saved
        pyramid.clear()
    if loss_tol is not None:
        oopt = OS.Adam(OS.all_params(P), HP['lr'], HP['beta1'], HP['beta2'])
        errs = []
        with O6.with_flownetc6():
            for i, b in enumerate(batches):
                lo, _ = OS.train_step(cfg, P, oopt, b[0], b[1:5], b[5], b[6])
                errs.append(rel_err(eager[i]['loss'], lo))
        assert max(errs) <= loss_tol, f'{cfg} {B}x{H}x{W} FlowNetC6: relative loss errors of steps 0-2 vs the oracle ' \
                                      f'{["%.2e" % e for e in errs]}, bar {loss_tol:.0e}'
        print(f'{cfg} {B}x{H}x{W} FlowNetC6: loss vs oracle {["%.2e" % e for e in errs]}')


def test_flow_sample_errors_flownetc6():
    """evaluate.flow_sample_errors with a FlowNetC6 (called as test_flow.py:125) against the oracle evaluation."""
    H, W = 64, 128
    tgt, refs = synth.frames(1, H, W, seed=73)
    K, Kinv = synth.intrinsics(1, H, W)
    rs = np.random.RandomState(7)
    Hg, Wg = 96, 200
    flow_gt = torch.from_numpy(np.concatenate([3 * rs.randn(1, 2, Hg, Wg), (rs.rand(1, 1, Hg, Wg) > 0.2)], 1).astype(np.float32))
    obj = torch.from_numpy((rs.rand(1, Hg, Wg) > 0.7).astype(np.float32))
    # flows of about a pixel (flownetc6_oracle.step_flow_params), so that the census and the rigid / non-rigid split
    # are not all one-sided
    P = dict(disp=ON.disp_params(), pose=ON.pose_params(), mask=ON.mask_params(), flow=O6.step_flow_params())

    def load(net, p):
        net.load_state_dict({k: v.clone() for k, v in p.items()})
        return net.to(DEV)

    nets = dict(disp=load(CM.DispResNet6(), P['disp']), pose=load(CM.PoseNetB6(nb_ref_imgs=4), P['pose']),
                mask=load(CM.MaskNet6(nb_ref_imgs=4, output_exp=True), P['mask']), flow=load(CM.FlowNetC6(), P['flow']))
    d = lambda t: t.to(DEV)      # noqa: E731
    errs, total = CE.flow_sample_errors(nets['disp'], nets['pose'], nets['mask'], nets['flow'], d(tgt), [d(r) for r in refs],
                                        d(K), d(Kinv), d(flow_gt), d(obj), THRESH=0.01)
    with O6.with_flownetc6():
        errs_o, total_o = OE.flow_sample_errors(P, tgt, refs, K, Kinv, flow_gt, obj, THRESH=0.01)
    assert np.allclose(np.array(errs, np.float64), np.array([float(e) for e in errs_o]), rtol=1e-3, atol=1e-4), (errs, errs_o)
    bad = ((total.cpu() - total_o).abs() > 1e-3 * total_o.abs().max()).float().mean().item()
    assert bad <= 1e-2, 'composed flow: %.2e of the pixels differ' % bad
