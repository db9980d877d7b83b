"""FlowNetC6 on the H100: the cost-volume kernels at the benchmark shape, the network against the fixture frozen from
the reference module, the training step with --flownet FlowNetC6 against the CPU oracle, CUDA-graph replay against eager
steps, every layer and loss-layer call of that step at b4 256x832 against fp64 (the layer and loss audits), and the flow
evaluation."""
import numpy as np
import pytest
import torch
from cc_b200 import _lib, models as CM, synth, evaluate as CE
from oracle import evaluate as OE, nets as ON
from tests import flownetc6_cases as FC, step_cases as SC, fullsize_cases as FS
from tests.util import conv_impl, device_lib      # noqa: F401  (device_lib: module fixture, the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]
DEV = torch.device('cuda:0')


def test_corr441d_benchmark_shape_vs_fp64():
    """[4,256,32,104] (conv3 of a 256x832 frame) and the small shapes: element-wise bound, bit-identical reruns.
    The kernels take no workspace, so there is no workspace size for a result to depend on."""
    worst = FC.case_corr441d(DEV, shapes=FC.CORR_SHAPES + [(4, 256, 32, 104)])
    print('corr441d worst r:', {s: {k: round(v, 3) for k, v in r.items()} for s, r in worst.items()})


def test_flownetc6_vs_fixture():
    """Default dispatch (wgmma tensor-core convolutions): outputs and eval output within 1e-4, gradients within 2e-3."""
    with conv_impl(_lib.IMPL_AUTO):
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


GRAPH_CASES = [('cfg2', 2, 64, 128, 1e-3), ('cfg3', 2, 64, 128, 1e-3), ('cfg3', 4, 256, 832, None)]


@pytest.mark.parametrize('cfg,B,H,W,loss_tol', GRAPH_CASES, ids=['%s-b%d-%dx%d' % c[:4] for c in GRAPH_CASES])
def test_flownetc6_step_graph_replay_vs_eager(cfg, B, H, W, loss_tol):
    """Trainer(cfg, flownet='FlowNetC6'): step_cases.case_step_graph_vs_eager, the eager losses against the CPU oracle
    step at the bar tests/test_gpu_parity.py GRAPH_CASES uses at that size."""
    SC.case_step_graph_vs_eager(DEV, cfg, B, H, W, loss_tol=loss_tol, seed=80, flownet='FlowNetC6')


def test_layer_audit_flownetc6_step():
    """Every layer call of the cfg3 b4 256x832 step with --flownet FlowNetC6 (second step, committed weight cache,
    production dispatch) against fp64, element by element: the dilated cost volumes included
    (fullsize_cases.audit_step)."""
    with conv_impl(_lib.IMPL_AUTO):
        FS.audit_step(DEV, flownet='FlowNetC6')


def test_loss_audit_flownetc6_step():
    """Every loss-layer call of the cfg3 b4 256x832 step with --flownet FlowNetC6 against fp64, element by element
    (fullsize_cases.loss_audit_step)."""
    with conv_impl(_lib.IMPL_AUTO):
        FS.loss_audit_step(DEV, flownet='FlowNetC6')


def test_flow_sample_errors_flownetc6():
    """evaluate.flow_sample_errors with a FlowNetC6 (called as test_flow.py:125) against the oracle evaluation."""
    H, W = 64, 128
    tgt, refs = synth.frames(1, H, W, seed=73)
    K, Kinv = synth.intrinsics(1, H, W)
    rs = np.random.RandomState(7)
    Hg, Wg = 96, 200
    flow_gt = torch.from_numpy(np.concatenate([3 * rs.randn(1, 2, Hg, Wg), (rs.rand(1, 1, Hg, Wg) > 0.2)], 1).astype(np.float32))
    obj = torch.from_numpy((rs.rand(1, Hg, Wg) > 0.7).astype(np.float32))
    # flows of about a pixel (flownetc6_cases.step_flow_params), so that the census and the rigid / non-rigid split
    # are not all one-sided
    P = dict(disp=ON.disp_params(), pose=ON.pose_params(), mask=ON.mask_params(), flow=FC.step_flow_params())

    def load(net, p):
        net.load_state_dict({k: v.clone() for k, v in p.items()})
        return net.to(DEV)

    nets = dict(disp=load(CM.DispResNet6(), P['disp']), pose=load(CM.PoseNetB6(nb_ref_imgs=4), P['pose']),
                mask=load(CM.MaskNet6(nb_ref_imgs=4, output_exp=True), P['mask']), flow=load(CM.FlowNetC6(), P['flow']))
    d = lambda t: t.to(DEV)      # noqa: E731
    errs, total = CE.flow_sample_errors(nets['disp'], nets['pose'], nets['mask'], nets['flow'], d(tgt), [d(r) for r in refs],
                                        d(K), d(Kinv), d(flow_gt), d(obj), THRESH=0.01)
    errs_o, total_o = OE.flow_sample_errors(P, tgt, refs, K, Kinv, flow_gt, obj, THRESH=0.01, flownet='FlowNetC6')
    assert np.allclose(np.array(errs, np.float64), np.array([float(e) for e in errs_o]), rtol=1e-3, atol=1e-4), (errs, errs_o)
    bad = ((total.cpu() - total_o).abs() > 1e-3 * total_o.abs().max()).float().mean().item()
    assert bad <= 1e-2, 'composed flow: %.2e of the pixels differ' % bad
