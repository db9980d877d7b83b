"""FlowNetC6 cases, run on the CPU simulator build (tests/test_flownetc6.py) and on the H100
(tests/test_gpu_flownetc6.py).

The cost volume (cc_b200.nn.corr441d) is checked against fp64 element by element with the layer audit's checks and
error model (tests/layer_audit.py corr441d_fwd_checks / corr441d_bwd_checks, family corr441d).  One dropped term of
typical size moves an element by ||t||_2 / sqrt(K) (r ~ 1 / (u K) >= 3.8e4 at K = 441, 6.5e4 at C = 256), so a missing
displacement or channel chunk cannot hide under R['corr441d']."""
import torch
from cc_b200 import nn as cnn, models as CM, synth
from tests.util import golden, assert_close, key_with_stride, pick
from tests import layer_audit as LA

N = LA.CORR441D_N
# (B, C, h, w): maps smaller and larger than the 41-pixel displacement span, one staged channel group and several
CORR_SHAPES = [(1, 1, 3, 5), (3, 13, 3, 5), (3, 13, 8, 16), (1, 256, 8, 16), (3, 13, 45, 50), (1, 256, 32, 104)]


def corr441d_ratios(f1, f2, out, g=None, d1=None, d2=None):
    """{check: worst r} of the forward output and, given g, of d f1 / d f2; the failures against the audit's bound."""
    checks = LA.corr441d_fwd_checks(f1, f2, out)[0]
    if g is not None:
        checks += LA.corr441d_bwd_checks(f1, f2, out, g, d1, d2)[0]
    res, _, bad = LA.evaluate('corr441d', checks)
    return {k: v[0] for k, v in res.items()}, bad


def _inputs(B, C, h, w, device, seed):
    g = torch.Generator().manual_seed(seed)
    f1, f2 = torch.randn(B, C, h, w, generator=g), torch.randn(B, C, h, w, generator=g)
    go = torch.randn(B, N * N, h, w, generator=g)
    return f1.to(device), f2.to(device), go.to(device)


def run_corr441d(f1, f2, go):
    """Forward and both input gradients through the autograd Function."""
    a, b = f1.clone().requires_grad_(True), f2.clone().requires_grad_(True)
    out = cnn.corr441d(a, b)
    d1, d2 = torch.autograd.grad(out, [a, b], go)
    return out.detach(), d1, d2


def case_corr441d(device, shapes=CORR_SHAPES, seed=11):
    """Every shape: forward, d f1 and d f2 within the layer audit's bound, negative correlations present (the leaky
    branch), and a second run bit-identical.  Returns the worst ratios per shape."""
    worst = {}
    for k, (B, C, h, w) in enumerate(shapes):
        f1, f2, go = _inputs(B, C, h, w, device, seed + k)
        out, d1, d2 = run_corr441d(f1, f2, go)
        assert (out < 0).any() and (out > 0).any(), 'both branches of the activation must be exercised'
        rs, bad = corr441d_ratios(f1, f2, out, go, d1, d2)
        assert not bad, f'corr441d {(B, C, h, w)}: {bad}'
        again = run_corr441d(f1, f2, go)
        for what, x, y in zip(('out', 'd_f1', 'd_f2'), (out, d1, d2), again):
            assert torch.equal(x, y), f'corr441d {(B, C, h, w)} {what}: a second run differs'
        worst[(B, C, h, w)] = rs
    return worst


# ---------------------------------------------------------------------------------------------------------------------
FIXTURE = 'flownetc6_small'
B_FIX, H_FIX, W_FIX, FRAME_SEED, WEIGHT_SEED, WTS_SEED = 2, 64, 128, 196, 310, 500      # tests/golden/make_flownetc6.py


def fixture_state_dict_keys():
    g = golden(FIXTURE)
    return {s.split(':')[0]: tuple(int(v) for v in s.split(':')[1].split(',')) for s in g['state_dict_keys']}


def fixture_weights(seed=WEIGHT_SEED):
    """The fixture's weights: synth.seeded_fill over FlowNetC6's state_dict (same keys on both sides)."""
    return synth.seeded_fill(CM.FlowNetC6(), seed).state_dict()


def _wts(shape, seed, device):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(device)


def check_against_fixture(outs, grads, ev, tol, gtol):
    """outs: the six train-mode outputs, grads: {param name: gradient}, ev: the eval output."""
    g = golden(FIXTURE)
    for i, x in enumerate(outs):
        assert_close(x, g['out%d' % i], tol, 'FlowNetC6 out%d' % i)
    for n, gg in grads.items():
        key, st = key_with_stride(g, 'g_' + n)
        assert_close(pick(gg, st), g[key], gtol, 'FlowNetC6 grad ' + n)
    assert_close(ev, g['eval'], tol, 'FlowNetC6 eval')


def fixture_inputs(device):
    tgt, refs = synth.frames(B_FIX, H_FIX, W_FIX, seed=FRAME_SEED)
    return tgt.to(device), refs[2].to(device)


def grad_names():
    g = golden(FIXTURE)
    return [k[2:].split('@')[0] for k in g if k.startswith('g_')]


def step_flow_params(seed=320, head_scale=0.05):
    """FlowNetC6 weights for step tests: synth.seeded_fill, the six predict_flow heads scaled by head_scale.
    Every output is 20 x a head upsampled, so the flows of the reference init (xavier, U[0,1) biases) or of seeded_fill
    alone are several pixels even on the 2x4 coarsest level of a 64x128 frame: every pixel of that level then samples
    outside the frame and the flow photometric loss is inf (in the reference as here).  Scaled heads keep the flows
    below a pixel there."""
    sd = synth.seeded_fill(CM.FlowNetC6(), seed).state_dict()
    for k in sd:
        if k.startswith('predict_flow'):
            sd[k] = sd[k] * head_scale
    return sd
