"""FlowNetC6 without a GPU: the oracle restatement against the fixture frozen from the reference module, the mirrored
module's state_dict contract, and the dilated cost-volume kernels compiled for the CPU simulator (tests/sim) against
fp64, including planted defects the bound must catch.  The whole network runs on the H100 in
tests/test_gpu_flownetc6.py (on the simulator it would take far longer than the rest of this suite)."""
import time
import pytest
import torch
import torch.nn.functional as F

from cc_b200 import models as CM
from cc_b200.train_step import build_nets
from oracle import nets as ON
from tests import flownetc6_cases as FC, layer_audit as LA
from tests.util import golden, sim_lib    # noqa: F401  (sim_lib: module fixture, the simulator library)

NTOL = 2e-5        # tests/test_oracle_golden.py: module vs functional conv algorithms


def test_oracle_matches_fixture():
    P = {k: v.detach().clone().requires_grad_(True) for k, v in FC.fixture_weights().items()}
    assert sum(v.numel() for v in P.values()) == ON.C6_NPARAMS == int(golden(FC.FIXTURE)['nparams'])
    tgt, ref = FC.fixture_inputs('cpu')
    outs = ON.flownetc6_forward(P, tgt, ref)
    loss = sum((x * FC._wts(x.shape, FC.WTS_SEED + i, 'cpu')).sum() for i, x in enumerate(outs))
    names = FC.grad_names()
    grads = dict(zip(names, torch.autograd.grad(loss, [P[n] for n in names])))
    with torch.no_grad():
        ev = ON.flownetc6_forward(P, tgt, ref, training=False)
    FC.check_against_fixture(outs, grads, ev, NTOL, NTOL)


def test_init_weights_is_the_references():
    """FlowNetC6.py:84-94: xavier_uniform weights, U[0,1) biases on every conv and transposed conv."""
    torch.manual_seed(0)
    net = CM.FlowNetC6()
    net.init_weights()
    for k, v in net.state_dict().items():
        if k.endswith('bias'):
            assert 0 <= v.min() and 0 < v.max() < 1, k
        else:
            bound = (6.0 / ((v.shape[0] + v.shape[1]) * v[0, 0].numel())) ** 0.5
            assert v.abs().max() <= bound and v.abs().max() > 0.9 * bound, k


def test_module_state_dict_matches_reference():
    net = CM.FlowNetC6()
    assert {k: tuple(v.shape) for k, v in net.state_dict().items()} == FC.fixture_state_dict_keys()
    assert list(net.state_dict()) == list(FC.fixture_state_dict_keys())
    assert sum(p.numel() for p in net.parameters()) == ON.C6_NPARAMS
    with pytest.raises(NotImplementedError):
        CM.FlowNetC6(batchNorm=True)
    with pytest.raises(NotImplementedError):
        CM.FlowNetC6(full_res=False)


def test_build_nets_flownet_choice():
    nets = build_nets('cfg2', 'cpu', flownet='FlowNetC6')
    assert isinstance(nets['flow'], CM.FlowNetC6) and nets['flow'].training
    assert isinstance(build_nets('cfg2', 'cpu')['flow'], CM.Back2Future)
    with pytest.raises(ValueError):
        build_nets('cfg2', 'cpu', flownet='SpyNet')


def test_corr441d_sim_vs_fp64(sim_lib):
    t0 = time.time()
    worst = FC.case_corr441d(torch.device('cpu'))
    print('corr441d on the simulator: %.1f s; worst r per shape %s' % (time.time() - t0, {
        s: {k: round(v, 3) for k, v in r.items()} for s, r in worst.items()}))


def _r(checks, what):
    """Worst r of one check and whether the layer audit's bound (family corr441d) flags it."""
    res, _, bad = LA.evaluate('corr441d', checks)
    return res[what][0], any(b.startswith(what + ' ') for b in bad)


def test_corr441d_planted_defects_fail_the_bound(sim_lib):
    B, C, h, w = 3, 13, 8, 16
    N = LA.CORR441D_N
    f1, f2, go = FC._inputs(B, C, h, w, 'cpu', 5)
    out, d1, d2 = FC.run_corr441d(f1, f2, go)
    fwd = lambda o: _r(LA.corr441d_fwd_checks(f1, f2, o)[0], 'z')       # noqa: E731
    assert not fwd(out)[1]
    j0 = 13
    # forward: one horizontal displacement skipped by the j loop (its 21 channels never accumulate)
    bad = out.clone()
    bad[:, j0::N] = 0
    assert fwd(bad)[1]
    # forward: the second staged channel group (channels 8..12) missing from every sum
    part = LA.corr441d_sample(f1[:, :8], f2[:, :8]) / C
    assert fwd(F.leaky_relu(part, 0.1))[1]
    # d f1: the terms of displacement column j0 dropped for every i
    dz = torch.where(out > 0, go, go * LA.CORR441D_SLOPE32)
    col = torch.zeros_like(dz)
    col[:, j0::N] = dz[:, j0::N]
    miss1, _ = LA.corr441d_adjoint(col, f1, f2)
    r, flagged = _r(LA.corr441d_bwd_checks(f1, f2, out, go, d1=d1 - miss1 / C)[0], 'd_f1')
    assert flagged and r > LA.R['corr441d'], r
    # d f2: one channel chunk never written (left at zero)
    bad2 = d2.clone()
    bad2[:, 8:] = 0
    r, flagged = _r(LA.corr441d_bwd_checks(f1, f2, out, go, d2=bad2)[0], 'd_f2')
    assert flagged and r > LA.R['corr441d'], r
    # and the correct results pass
    rs, bad = FC.corr441d_ratios(f1, f2, out, go, d1, d2)
    assert not bad and max(rs.values()) <= LA.R['corr441d'], rs
