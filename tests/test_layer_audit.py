"""The layer audit's checker (tests/layer_audit.py), without a GPU.

fp32 torch ops stand in for the kernels: correct fp32 results must pass every bound, and each of six typical kernel
bugs applied to an otherwise correct result must be flagged; so must three faults of the tensor-core convolutions'
3xTF32 stage ring, emulated on the CPU, that rel_err's 1e-4 bar alone can miss.  The wrappers must restore the autograd
Functions on exit, also when the audit raises.  Then the audit runs on the CPU simulator build of the product kernels
over the four networks, one forward and one backward each (DispResNet6 and PoseNetB6 at b2 64x128, MaskNet6 and Back2Future at
b1 64x64, FlowNetC6 at b1 64x128), which covers the CUDA-core convolutions and the BatchNorm, upsample, cost-volume and
feature-warp kernels; and over the evaluation forwards in eval mode, which covers the eval-mode BatchNorm kernel.  Three
mistakes in an eval-mode BatchNorm result (eps, the running mean, invstd) must each be flagged."""
import pytest
import torch
import torch.nn.functional as F
from tests import layer_audit as LA, flownetc6_cases as FC6, fullsize_cases as FS
from tests.util import conv_impl, sim_lib      # noqa: F401  (sim_lib: module fixture, the simulator library)
from cc_b200 import nn as cnn, _lib, synth, models as CM
from oracle import nets as ON

pytestmark = pytest.mark.usefixtures('sim_lib')


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _flagged(op, checks, what):
    res, r, bad = LA.evaluate(op, checks)
    return any(b.startswith(what + ' ') for b in bad), res[what]


def _passes(op, checks):
    res, r, bad = LA.evaluate(op, checks)
    assert not bad, (op, bad, res)
    return r


def test_conv_forward_border_tap_dropped():
    g = _gen(1)
    x = torch.randn(2, 16, 12, 20, generator=g)
    w = torch.randn(24, 16, 3, 3, generator=g) / 12
    b = torch.randn(24, generator=g)
    y = F.leaky_relu(F.conv2d(x, w, b, 1, 1), 0.2)
    _passes('conv', LA.conv_fwd_checks(x, w, b, None, 1, 1, _lib.ACT_LEAKY, 0.2, y)[0])
    # output pixel (0, 0) of channel 5: its tap (1, 1) reads x[:, :, 0, 0]; drop that tap's contribution
    z = F.conv2d(x, w, b, 1, 1)
    z[1, 5, 0, 0] -= (x[1, :, 0, 0] * w[5, :, 1, 1]).sum()
    flagged, (r, rel, _) = _flagged('conv', LA.conv_fwd_checks(x, w, b, None, 1, 1, _lib.ACT_LEAKY, 0.2, F.leaky_relu(z, 0.2))[0], 'y')
    assert flagged and r > 1e3, r


def _tf32(t):
    """fp32 -> tf32, round to nearest with ties away from zero (cvt.rna.tf32.f32), by bit mask."""
    return ((t.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def _conv_3xtf32(x, w, stride, pad, fault=None):
    """The wgmma convolution's arithmetic, emulated on the CPU: the im2col operand A [pixels, K] and the weights B [K, Co]
    in the kernel's K order (tap-major, channels inner), split into tf32 hi and lo, k-stages of 32 whose
    hi*hi + hi*lo + lo*hi products are summed in fp64, the result rounded to fp32.  fault: 'cross terms dropped' - the
    last k-stage keeps hi*hi only; 'stale lo' - the last k-stage multiplies the previous stage's A lo; '2xTF32' - every
    stage drops lo*hi.  The first two are what one ring-phase or buffer-parity slip does to a single stage."""
    B, Ci, H, W = x.shape
    Co, _, k, _ = w.shape
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    a = F.unfold(x, k, padding=pad, stride=stride).view(B, Ci, k * k, Ho * Wo).permute(0, 3, 2, 1).reshape(B * Ho * Wo, -1)
    b = w.permute(0, 2, 3, 1).reshape(Co, -1).t()
    ah, bh = _tf32(a), _tf32(b)
    al, bl = _tf32(a - ah), _tf32(b - bh)
    ah, bh, al, bl = ah.double(), bh.double(), al.double(), bl.double()
    K = a.shape[1]
    acc = torch.zeros(a.shape[0], Co, dtype=torch.float64)
    last = (K - 1) // 32 * 32
    for k0 in range(0, K, 32):
        sl = slice(k0, k0 + 32)
        acc += ah[:, sl] @ bh[sl]
        if fault == 'cross terms dropped' and k0 == last:
            continue
        alo = al[:, k0 - 32:k0 - 32 + (min(K, k0 + 32) - k0)] if fault == 'stale lo' and k0 == last else al[:, sl]
        acc += ah[:, sl] @ bl[sl]
        if fault != '2xTF32':
            acc += alo @ bh[sl]
    return acc.float().view(B, Ho * Wo, Co).permute(0, 2, 1).reshape(B, Co, Ho, Wo)


@pytest.mark.parametrize('fault', ['cross terms dropped', 'stale lo', '2xTF32'])
def test_conv_tf32_stage_fault_flagged(fault):
    """Three plausible faults of the 3xTF32 stage ring, emulated on the CPU (no device kernel is touched) on shapes of
    the ring tests' plan grid: the element-wise bound flags each on every shape (the correct emulation passes), while
    rel_err's 1e-4 bar alone lets a one-stage fault through on at least one of them - why the convolution edge tests
    hold every result to the bound."""
    missed = []
    for i, (B, Ci, H, W, Co, k, s, p) in enumerate([(2, 64, 16, 16, 64, 3, 1, 1), (2, 32, 8, 8, 20, 3, 1, 1),
                                                     (1, 512, 8, 8, 64, 3, 1, 1)]):
        g = _gen(30 + i)
        x = torch.randn(B, Ci, H, W, generator=g)
        w = torch.randn(Co, Ci, k, k, generator=g) / (Ci * k * k) ** 0.5
        r_ok = _passes('conv', LA.conv_fwd_checks(x, w, None, None, s, p, _lib.ACT_NONE, 0.0, _conv_3xtf32(x, w, s, p))[0])
        assert r_ok < 1, r_ok
        flagged, (r, rel, _) = _flagged('conv', LA.conv_fwd_checks(x, w, None, None, s, p, _lib.ACT_NONE, 0.0,
                                                                    _conv_3xtf32(x, w, s, p, fault))[0], 'y')
        assert flagged and r > LA.R['conv'], (fault, (B, Ci, H, W, Co, k, s, p), r, rel)
        if rel <= LA.REL_BAR:
            missed.append(((B, Ci, H, W, Co, k, s, p), r, rel))
    assert missed or fault == '2xTF32', (fault, 'rel_err alone catches it on every shape')


def test_dgrad_parity_class_shifted():
    g = _gen(2)
    x = torch.randn(2, 8, 16, 24, generator=g)
    w = torch.randn(12, 8, 3, 3, generator=g) / 8
    dz = torch.randn(2, 12, 8, 12, generator=g)
    dx = torch.nn.grad.conv2d_input(x.shape, w, dz, 2, 1)
    _passes('conv', LA.conv_bwd_checks(x, w, None, dz, 2, 1, _lib.ACT_NONE, 0.0, dx=dx)[0])
    bad = dx.clone()
    bad[:, :, 1::2, 1::2] = torch.roll(dx[:, :, 1::2, 1::2], 1, dims=3)      # odd-odd class one pixel to the right
    flagged, (r, _, _) = _flagged('conv', LA.conv_bwd_checks(x, w, None, dz, 2, 1, _lib.ACT_NONE, 0.0, dx=bad)[0], 'dx')
    assert flagged and r > 1e3, r


def test_wgrad_pixel_missing_at_long_k():
    g = _gen(3)
    B, C, H, W = 2, 4, 256, 256                       # K = B H W = 131072 >= 1e5 products per weight
    x = torch.relu(torch.randn(B, C, H, W, generator=g))
    w = torch.randn(4, C, 3, 3, generator=g) / 6
    dz = torch.randn(B, 4, H, W, generator=g)
    dw = torch.nn.grad.conv2d_weight(x, w.shape, dz, 1, 1)
    checks, K = LA.conv_bwd_checks(x, w, None, dz, 1, 1, _lib.ACT_NONE, 0.0, dw=dw)
    assert K == B * H * W and LA.R['conv'] < 1 / (LA.U * K)
    _passes('conv', checks)
    dz_missing = dz.clone()
    dz_missing[1, :, 100, 37] = 0                     # one output pixel left out of the reduction
    bad = torch.nn.grad.conv2d_weight(x, w.shape, dz_missing, 1, 1)
    flagged, (r, _, _) = _flagged('conv', LA.conv_bwd_checks(x, w, None, dz, 1, 1, _lib.ACT_NONE, 0.0, dw=bad)[0], 'dw')
    assert flagged, r


def _bn_fp32(x, gamma, beta, g, eps=1e-5):
    mean = x.mean((0, 2, 3))
    var = ((x - mean.view(1, -1, 1, 1)) ** 2).mean((0, 2, 3))
    inv = 1 / torch.sqrt(var + eps)
    xh = (x - mean.view(1, -1, 1, 1)) * inv.view(1, -1, 1, 1)
    y = xh * gamma.view(1, -1, 1, 1) + beta.view(1, -1, 1, 1)
    db, dg = g.sum((0, 2, 3)), (g * xh).sum((0, 2, 3))
    N = x.numel() // x.shape[1]
    gi = (gamma * inv).view(1, -1, 1, 1)
    dx = gi * (g - db.view(1, -1, 1, 1) / N - xh * dg.view(1, -1, 1, 1) / N)
    return torch.stack([mean, inv], 1), y, dx, dg, db, gi


def test_bn_dx_mean_term_removed():
    g = _gen(4)
    x = torch.randn(3, 5, 40, 70, generator=g) * 2 + 3
    gamma, beta = torch.rand(5, generator=g) + 0.5, torch.randn(5, generator=g)
    gout = torch.randn(3, 5, 40, 70, generator=g) + 0.3
    stats, y, dx, dg, db, gi = _bn_fp32(x, gamma, beta, gout)
    rm, rv = torch.zeros(5), torch.ones(5)
    N = 3 * 40 * 70
    var = x.var((0, 2, 3), unbiased=True)
    rm1, rv1 = 0.9 * rm + 0.1 * stats[:, 0], 0.9 * rv + 0.1 * var
    _passes('bn', LA.bn_fwd_checks(x, gamma, beta, rm, rv, rm1, rv1, stats, y, 1e-5, 0.1)[0])
    _passes('bn', LA.bn_bwd_checks(x, gamma, stats, gout, dx=dx, dgamma=dg, dbeta=db)[0])
    bad = dx.clone()
    bad[:, 2] += gi[0, 2] * db[2] / N                 # channel 2 without its mean term
    flagged, (r, _, _) = _flagged('bn', LA.bn_bwd_checks(x, gamma, stats, gout, dx=bad)[0], 'dx')
    assert flagged and r > 1e3, r


def _bn_eval_case(seed=8):
    """An eval-mode BatchNorm call with running statistics far from their defaults, and its fp32 result."""
    g = _gen(seed)
    x = torch.randn(2, 6, 20, 30, generator=g) * 1.5 + 0.4
    gamma, beta = torch.rand(6, generator=g) + 0.5, torch.randn(6, generator=g) * 0.1
    rm, rv = 0.5 * torch.randn(6, generator=g), 0.25 + 3.75 * torch.rand(6, generator=g)
    v = lambda t: t.view(1, -1, 1, 1)       # noqa: E731
    y = (x - v(rm)) * v(1 / torch.sqrt(rv + 1e-5)) * v(gamma) + v(beta)
    return x, gamma, beta, rm, rv, y, v


def test_bn_eval_eps_mean_and_invstd_mistakes_flagged():
    """The eval-mode bound is a rounding count (R = 1): a correct fp32 result passes; eps left out of the square root,
    the running mean ignored, and the running variance used where invstd belongs are each flagged."""
    x, gamma, beta, rm, rv, y, v = _bn_eval_case()
    r = _passes('bn_eval', LA.bn_eval_checks(x, gamma, beta, rm, rv, y, 1e-5)[0])
    assert r <= LA.R['bn_eval'], r
    bad = {'eps omitted': (x - v(rm)) * v(1 / torch.sqrt(rv)) * v(gamma) + v(beta),
           'running mean ignored': x * v(1 / torch.sqrt(rv + 1e-5)) * v(gamma) + v(beta),
           'running_var for invstd': (x - v(rm)) * v(rv + 1e-5) * v(gamma) + v(beta)}
    for what, yb in bad.items():
        flagged, (r, _, _) = _flagged('bn_eval', LA.bn_eval_checks(x, gamma, beta, rm, rv, yb, 1e-5)[0], 'y')
        assert flagged and r > LA.R['bn_eval'], (what, r)


def test_bn_eval_kernel_vs_fp64():
    """The eval-mode BatchNorm kernel of the simulator build through cc_b200.nn, audited as one call: a row of family
    bn_eval within R = 1."""
    x, gamma, beta, rm, rv, _, _ = _bn_eval_case(9)
    bn = cnn.BatchNorm2d(6)
    with torch.no_grad():
        bn.weight.copy_(gamma)
        bn.bias.copy_(beta)
        bn.running_mean.copy_(rm)
        bn.running_var.copy_(rv)
    bn.eval()
    with LA.LayerAudit(nets={'bn': bn}, report=False) as audit:
        with torch.no_grad():
            bn(x)
    assert [(r['op'], r['name'], r['phase']) for r in audit.rows] == [('bn_eval', 'bn', 'fwd')], audit.rows
    assert audit.rows[0]['r'] <= LA.R['bn_eval']


def test_corr81_displacement_channels_swapped():
    g = _gen(5)
    f1, f2 = torch.randn(2, 24, 9, 13, generator=g), torch.randn(2, 24, 9, 13, generator=g)
    for rev, idx in ((False, ON.IDX_FWD), (True, ON.IDX_BWD)):
        out = ON.correlate(f1, f2).index_select(1, torch.tensor(idx))
        _passes('corr81', LA.corr81_fwd_checks(f1, f2, rev, out)[0])
        bad = out.clone()
        bad[:, [10, 11]] = out[:, [11, 10]]
        flagged, (r, _, _) = _flagged('corr81', LA.corr81_fwd_checks(f1, f2, rev, bad)[0], 'out')
        assert flagged and r > 1e3, r
    # backward through torch fp32 autograd of the same definition
    a, b = f1.clone().requires_grad_(True), f2.clone().requires_grad_(True)
    G = torch.randn(2, 81, 9, 13, generator=g)
    d1, d2 = torch.autograd.grad((ON.correlate(a, b).index_select(1, torch.tensor(ON.IDX_FWD)) * G).sum(), [a, b])
    _passes('corr81', LA.corr81_bwd_checks(f1, f2, False, G, d1, d2)[0])


def _warp_case(seed=6, B=2, C=5, h=12, w=17):
    g = _gen(seed)
    x = torch.randn(B, C, h, w, generator=g)
    flo = torch.randn(B, 2, h, w, generator=g) * 3
    # pixel (3, 4) of sample 0 samples at (x, y) = (5, 2) to within fp32 rounding of the flow: a tie in both components
    # (Back2Future's normalisation with align_corners=False: ix = (x + u) w / (w - 1) - 1/2)
    flo[0, :, 3, 4] = torch.tensor([5.5 * (w - 1) / w - 4, 2.5 * (h - 1) / h - 3])
    gout = torch.randn(B, C, h, w, generator=g)
    return x, flo, gout


def test_featwarp_sampler_matches_grid_sample():
    """The audit's fp64 bilinear sampler against torch's grid_sample (the oracle's Model.warp) in fp64."""
    x, flo, gout = _warp_case()
    xd, fd = x.double().requires_grad_(True), flo.double().requires_grad_(True)
    ref = ON.b2f_warp(xd, fd)
    dx_ref, df_ref = torch.autograd.grad((ref * gout.double()).sum(), [xd, fd])
    B, C, h, w = x.shape
    ix, iy, _, _ = LA._warp_coords(flo, h, w)
    sp = LA._Samp(ix, iy, h, w)
    c = sp.corners(x.double())
    out = sum(wq.unsqueeze(1) * cq for wq, cq in zip(sp.w, c))
    assert (out - ref.detach()).abs().max() < 1e-12
    dx = sp.scatter([gout.double() * wq.unsqueeze(1) for wq in sp.w])
    assert (dx - dx_ref).abs().max() < 1e-12
    tie = ((ix - ix.round()).abs() < 1e-9).unsqueeze(1) | ((iy - iy.round()).abs() < 1e-9).unsqueeze(1)
    dfx = (gout.double() * sp.dx(c)).sum(1) * sp.gx * (2.0 / (w - 1))
    dfy = (gout.double() * sp.dy(c)).sum(1) * sp.gy * (2.0 / (h - 1))
    d = (torch.stack([dfx, dfy], 1) - df_ref).abs().masked_fill(tie, 0)
    assert d.max() < 1e-12


def test_featwarp_scatter_corner_dropped():
    x, flo, gout = _warp_case()
    xr, fr = x.clone().requires_grad_(True), flo.clone().requires_grad_(True)
    out = ON.b2f_warp(xr, fr)
    dx, df = torch.autograd.grad((out * gout).sum(), [xr, fr])
    _passes('featwarp', LA.featwarp_fwd_checks(x, flo, out.detach())[0])
    checks, K, extra = LA.featwarp_bwd_checks(x, flo, gout, dx=dx, dflow=df)
    _passes('featwarp', checks)
    assert extra['ties'] >= 2 and extra['fx_term_max'] > 0
    # drop the (y0, x0) corner of output pixel (5, 6) of sample 1: its contribution to every channel
    B, C, h, w = x.shape
    ix, iy, _, _ = LA._warp_coords(flo, h, w)
    sp = LA._Samp(ix, iy, h, w)
    bad = dx.clone()
    i = int(sp.idx[0][1, 5 * w + 6])
    bad.view(B, C, h * w)[1, :, i] -= (gout[1, :, 5, 6].double() * sp.w[0][1, 5, 6]).float()
    flagged, (r, _, _) = _flagged('featwarp', LA.featwarp_bwd_checks(x, flo, gout, dx=bad)[0], 'd_x')
    assert flagged and r > 10 * LA.R['featwarp'], r


def test_audit_restores_functions():
    """The wrappers are in place inside the context only, and are removed on exit - also when the body raises and when
    the audit itself raises because a call is over its bound."""
    names = list(LA.LayerAudit.FNS.values())
    before = {n: (getattr(cnn, n).__dict__['forward'], getattr(cnn, n).__dict__['backward']) for n in names}
    run = cnn._run

    def same():
        return all(getattr(cnn, n).__dict__['forward'] is before[n][0] and getattr(cnn, n).__dict__['backward'] is before[n][1]
                   for n in names) and cnn._run is run

    x = torch.randn(1, 3, 5, 7, generator=_gen(7)).requires_grad_(True)
    with LA.LayerAudit(report=False) as audit:
        assert not same()
        cnn.upsample2x(x).sum().backward()
    assert same() and len(audit.rows) == 2 and all(not r['bad'] for r in audit.rows)
    with pytest.raises(RuntimeError, match='body'):
        with LA.LayerAudit(report=False):
            raise RuntimeError('body')
    assert same()
    saved = LA.R['bn']
    try:
        LA.R['bn'] = -1.0                             # every BatchNorm call now misses its bound
        bn = cnn.BatchNorm2d(3)
        with pytest.raises(AssertionError, match='layer calls over their bound'):
            with LA.LayerAudit(report=False):
                bn(x)
    finally:
        LA.R['bn'] = saved
    assert same()


def _wts(shape, seed):
    return torch.randn(shape, generator=_gen(seed))


def _net_outputs(which):
    if which == 'disp':
        net = CM.DispResNet6()
        net.load_state_dict(ON.disp_params())
        tgt, _ = synth.frames(2, 64, 128, seed=40)
        return net, lambda: list(net(tgt))
    if which == 'pose':
        net = CM.PoseNetB6(nb_ref_imgs=4)
        net.load_state_dict(ON.pose_params())
        tgt, refs = synth.frames(2, 64, 128, seed=40)
        return net, lambda: [net(tgt, refs)]
    if which == 'mask':
        net = CM.MaskNet6(nb_ref_imgs=4, output_exp=True)
        net.load_state_dict(ON.mask_params())
        tgt, refs = synth.frames(1, 64, 64, seed=42)
        return net, lambda: list(net(tgt, refs))
    if which == 'flownetc6':
        net = CM.FlowNetC6()
        net.load_state_dict(FC6.step_flow_params())
        tgt, refs = synth.frames(1, 64, 128, seed=42)
        return net, lambda: list(net(tgt, refs[2]))
    net = CM.Back2Future(nlevels=6, compute_occ=False)
    net.load_state_dict(ON.flow_params())
    tgt, refs = synth.frames(1, 64, 64, seed=42)
    return net, lambda: (lambda ff, fb, _: list(ff) + list(fb))(*net(tgt, refs[1:3]))


@pytest.mark.parametrize('which', ['disp', 'pose', 'mask', 'flow', 'flownetc6'])
def test_audit_simulator_nets(which):
    """One forward and one backward (of a seeded weighted sum of the outputs) of each net on the simulator build, every
    layer call audited; every Conv2d / ConvTranspose2d / BatchNorm2d module is audited forward and backward, and the
    flow nets' cost volumes and feature warps are all there."""
    with conv_impl(_lib.IMPL_FFMA):
        net, run = _net_outputs(which)
        net.train()
        with LA.LayerAudit(nets={which: net}, tag='sim_' + which) as audit:
            outs = run()
            sum((o * _wts(o.shape, 500 + i)).sum() for i, o in enumerate(outs)).backward()
    want = {which + ('.' + n if n else '') for n, m in net.named_modules()     # occlusion decoders: not run in training
            if isinstance(m, (cnn.Conv2d, cnn.ConvTranspose2d, cnn.BatchNorm2d)) and not n.startswith('decoder_occ')}
    for phase in ('fwd', 'bwd'):
        got = {r['name'] for r in audit.rows if r['phase'] == phase and r['op'] in ('conv', 'convT', 'bn')}
        assert got == want, (phase, sorted(want - got)[:10], sorted(got - want)[:10])
    calls = dict(flow=dict(corr81=10, featwarp=8), flownetc6=dict(corr441d=1)).get(which, {})
    for op in ('corr81', 'corr441d', 'featwarp'):
        for phase in ('fwd', 'bwd'):
            assert sum(r['op'] == op and r['phase'] == phase for r in audit.rows) == calls.get(op, 0), (op, phase)


def test_audit_simulator_eval_forwards():
    """evaluate._flow_nets in eval mode over the four nets (Back2Future as the flow net) at b1 64x128 on the simulator
    build, every BatchNorm's running statistics seeded far from the defaults: every layer call audited, the eval-mode
    BatchNorms included (fullsize_cases.audit_eval_forwards).  FlowNetC6 in eval mode is audited on the H100."""
    with conv_impl(_lib.IMPL_FFMA):
        FS.audit_eval_forwards(torch.device('cpu'), 'Back2Future', H=64, W=128)
