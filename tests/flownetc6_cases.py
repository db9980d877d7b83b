"""FlowNetC6 cases, run on the CPU simulator build (tests/test_flownetc6.py) and on the H100
(tests/test_gpu_flownetc6.py).

The cost volume (cc_b200.nn.corr441d) is checked against fp64 element by element with the error model of
tests/layer_audit.py (u = 2^-24; a long reduction of K products of random sign is off by about u sqrt(K) ||t||_2):
  forward   the kernel sums the C products f1 f2 of an output in fp32, divides by C and applies LeakyReLU(0.1).  The
            activation is inverted exactly in fp64 (out / 0.1f where out <= 0: the slope multiply adds u |z|), and the
            pre-activation z is held to  s = (u sqrt(C) + C_PROD) ||t||_2 / C + 3u |z| + TINY32.
  d f1/d f2 sums of the 441 products dz f (dz = g * leaky'(out), taken from the sign of the forward's own output),
            divided by C:  s = (u sqrt(441) + C_PROD) ||t||_2 / C + 2u |ref| + TINY32.
r = |kernel - fp64| / s must stay below R_CORR441D.  One dropped term of typical size moves an element by ||t||_2 / sqrt(K)
(r ~ 1 / (u K) >= 2.3e4 at K = 441, 6.5e4 at C = 256), so a missing displacement or channel chunk cannot hide."""
import torch
import torch.nn.functional as F
from cc_b200 import nn as cnn, models as CM, synth
from tests.util import golden, assert_close, key_with_stride, pick
from oracle import nets as ON
from tests.layer_audit import U, C_PROD, TINY32

R_CORR441D = 6.0
N, R = 21, 20
SLOPE32 = float(torch.tensor(0.1, dtype=torch.float32))
# (B, C, h, w): maps smaller and larger than the 41-pixel displacement span, one staged channel group and several
CORR_SHAPES = [(1, 1, 3, 5), (3, 13, 3, 5), (3, 13, 8, 16), (1, 256, 8, 16), (3, 13, 45, 50), (1, 256, 32, 104)]


def corr441d_sample(a, b):
    """The restated third-party correlation at FlowNetC6's call (patch 21, dilation 2) as [B,441,h,w], not divided by C."""
    B, _, h, w = a.shape
    return ON.spatial_correlation_sample(a, b, patch=N, dilation=2).reshape(B, N * N, h, w)


def corr441d_ref(f1, f2):
    """fp64 pre-activation z [B,441,h,w] and ||t||_2 / C of its terms."""
    a, b = f1.double(), f2.double()
    B, C, h, w = a.shape
    z = corr441d_sample(a, b) / C
    tn = corr441d_sample(a * a, b * b).sqrt() / C
    return z, tn


def corr441d_adjoint(G, f1, f2):
    """(sum_k G_k f2(. + d_k), sum_k G_k(. - d_k) f1(. - d_k)) over the 441 displacements d_k, no 1/C."""
    B, C, h, w = f1.shape
    f2p = F.pad(f2, (R, R, R, R))
    d1 = torch.zeros_like(f1)
    d2p = torch.zeros_like(f2p)
    for i in range(N):
        for j in range(N):
            gk = G[:, N * i + j:N * i + j + 1]
            sl = (slice(None), slice(None), slice(2 * i, 2 * i + h), slice(2 * j, 2 * j + w))
            d1 += gk * f2p[sl]
            d2p[sl] += gk * f1
    return d1, d2p[:, :, R:R + h, R:R + w]


def corr441d_fwd_ratio(f1, f2, out):
    """Worst r of the forward output (module docstring)."""
    z, tn = corr441d_ref(f1, f2)
    o = out.double()
    zk = torch.where(o > 0, o, o / SLOPE32)
    s = (U * f1.shape[1] ** 0.5 + C_PROD) * tn + 3 * U * z.abs() + TINY32
    return ((zk - z).abs() / s).max().item()


def corr441d_bwd_ratios(f1, f2, out, g, d1=None, d2=None):
    """Worst r of d f1 and d f2 (module docstring)."""
    C = f1.shape[1]
    a, b, gd = f1.double(), f2.double(), g.double()
    dz = torch.where(out > 0, gd, gd * SLOPE32)
    r1, r2 = corr441d_adjoint(dz, a, b)
    t1, t2 = corr441d_adjoint(dz * dz, a * a, b * b)
    res = {}
    for what, got, ref, tn in (('d_f1', d1, r1, t1), ('d_f2', d2, r2, t2)):
        if got is not None:
            ref = ref / C
            s = (U * N + C_PROD) * tn.sqrt() / C + 2 * U * ref.abs() + TINY32
            res[what] = ((got.double() - ref).abs() / s).max().item()
    return res


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
    """Every shape: forward, d f1 and d f2 within the bound, negative correlations present (the leaky branch), and a
    second run bit-identical.  Returns the worst ratios per shape."""
    worst = {}
    for k, (B, C, h, w) in enumerate(shapes):
        f1, f2, go = _inputs(B, C, h, w, device, seed + k)
        out, d1, d2 = run_corr441d(f1, f2, go)
        assert (out < 0).any() and (out > 0).any(), 'both branches of the activation must be exercised'
        rs = dict(out=corr441d_fwd_ratio(f1, f2, out), **corr441d_bwd_ratios(f1, f2, out, go, d1, d2))
        for what, r in rs.items():
            assert r <= R_CORR441D, f'corr441d {(B, C, h, w)} {what}: r = {r:.3g} > {R_CORR441D}'
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
