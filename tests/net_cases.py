"""Parity cases for the convolution kernels and the networks (shared by the simulator tests and the
GPU tests): product modules vs the golden fixtures frozen from the reference and vs the oracle."""
import torch
import torch.nn.functional as F
from tests.util import golden, T, assert_close, key_with_stride, pick
from cc_b200 import synth, nn as cnn, models as CM
from oracle import nets as ON

TOL = 1e-4


def _wts(shape, seed, device):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(device)


def case_conv_shapes(device, big=False):
    """conv2d / conv_transpose2d forward + all gradients against torch on odd shapes."""
    g = torch.Generator().manual_seed(0)
    cases = [  # B, Ci, H, W, Co, k, s, p, act, bias, res
        (2, 3, 13, 17, 8, 7, 2, 3, 'relu', True, False),
        (2, 15, 12, 20, 16, 5, 2, 2, 'relu', True, False),
        (1, 17, 9, 11, 16, 3, 1, 1, 'relu', False, True),
        (2, 8, 10, 14, 1, 3, 1, 1, 'sigmoid', True, False),
        (2, 16, 8, 12, 24, 1, 1, 0, None, True, False),
        (2, 32, 7, 9, 64, 1, 2, 0, None, False, False),
        (2, 65, 6, 10, 32, 3, 2, 1, 'leaky', True, False),
        (1, 4, 16, 16, 70, 3, 1, 1, 'leaky', True, True),
    ]
    if big:
        cases += [(4, 32, 32, 104, 32, 7, 1, 3, 'relu', True, False), (4, 196, 16, 52, 128, 3, 1, 1, 'leaky', True, False),
                  (4, 512, 2, 7, 512, 3, 1, 1, 'relu', False, True), (4, 16, 64, 208, 1, 3, 1, 1, 'sigmoid', True, False)]
    for (B, Ci, H, W, Co, k, s, p, act, bias, res) in cases:
        x = torch.randn(B, Ci, H, W, generator=g).to(device).requires_grad_(True)
        w = (torch.randn(Co, Ci, k, k, generator=g) * 0.2).to(device).requires_grad_(True)
        b = torch.randn(Co, generator=g).to(device).requires_grad_(True) if bias else None
        Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
        r = torch.randn(B, Co, Ho, Wo, generator=g).to(device).requires_grad_(True) if res else None
        y = cnn.conv2d(x, w, b, r, s, p, act, 0.2)
        z = F.conv2d(x, w, b, s, p)
        if res:
            z = z + r
        z = {'relu': F.relu, 'sigmoid': torch.sigmoid, 'leaky': lambda t: F.leaky_relu(t, 0.2), None: lambda t: t}[act](z)
        tag = f'conv {Ci}->{Co} k{k} s{s}'
        assert_close(y, z, TOL, tag)
        wt = _wts(y.shape, 1, device)
        ins = [t for t in (x, w, b, r) if t is not None]
        ga = torch.autograd.grad((y * wt).sum(), ins)
        gb = torch.autograd.grad((z * wt).sum(), ins)
        for a_, b_, nm in zip(ga, gb, ('dx', 'dw', 'db/dres', 'dres')):
            assert_close(a_, b_, TOL, tag + ' ' + nm)
    tcases = [(2, 16, 5, 7, 8, 3, 2, 1, 1, 'relu'), (2, 24, 4, 6, 12, 4, 2, 1, 0, 'relu'), (1, 8, 3, 3, 5, 3, 1, 1, 0, None)]
    if big:
        tcases += [(4, 512, 2, 7, 512, 3, 2, 1, 1, 'relu'), (4, 96, 32, 104, 32, 4, 2, 1, 0, 'relu')]
    for (B, Ci, H, W, Co, k, s, p, op, act) in tcases:
        x = torch.randn(B, Ci, H, W, generator=g).to(device).requires_grad_(True)
        w = (torch.randn(Ci, Co, k, k, generator=g) * 0.2).to(device).requires_grad_(True)
        b = torch.randn(Co, generator=g).to(device).requires_grad_(True)
        y = cnn.conv_transpose2d(x, w, b, s, p, op, act)
        z = F.conv_transpose2d(x, w, b, s, p, op)
        z = F.relu(z) if act == 'relu' else z
        tag = f'convT {Ci}->{Co} k{k} s{s}'
        assert_close(y, z, TOL, tag)
        wt = _wts(y.shape, 2, device)
        ga = torch.autograd.grad((y * wt).sum(), [x, w, b])
        gb = torch.autograd.grad((z * wt).sum(), [x, w, b])
        for a_, b_, nm in zip(ga, gb, ('dx', 'dw', 'db')):
            assert_close(a_, b_, TOL, tag + ' ' + nm)


def case_conv_tc(device):
    """wgmma tensor-core path against torch fp64 on real layer shapes: fprop, dgrad (incl. strided parity classes /
    ConvTranspose forward) and wgrad.  IMPL_TC = 3xTF32 (fp32 parity), IMPL_TC_TF32 = single TF32 (what cuDNN
    runs by default for the reference).  GPU only (the simulator has no tensor cores)."""
    from cc_b200 import _lib
    g = torch.Generator().manual_seed(7)
    shapes = [(2, 32, 16, 24, 64, 3, 1, 1), (2, 17, 13, 20, 40, 3, 2, 1), (4, 128, 32, 104, 128, 3, 1, 1),
              (4, 32, 64, 208, 32, 7, 1, 3), (4, 65, 32, 104, 32, 1, 1, 0), (2, 256, 16, 52, 160, 3, 1, 1),
              (2, 16, 64, 208, 1, 3, 1, 1), (4, 3, 64, 208, 32, 7, 2, 3),
              (4, 512, 8, 26, 512, 3, 1, 1), (4, 256, 16, 52, 512, 3, 2, 1)]      # small-M layers: split-K
    saved = cnn.CONV_IMPL
    try:
        for (B, Ci, H, W, Co, k, s, p) in shapes:
            x = torch.randn(B, Ci, H, W, generator=g).to(device).requires_grad_(True)
            w = (torch.randn(Co, Ci, k, k, generator=g) / (Ci * k * k) ** 0.5).to(device).requires_grad_(True)
            b = torch.randn(Co, generator=g).to(device).requires_grad_(True)
            xd, wd, bd = [t.detach().double().requires_grad_(True) for t in (x, w, b)]
            for impl, tol in ((_lib.IMPL_TC, 1e-4), (_lib.IMPL_TC_TF32, 5e-3)):
                tag = f'tc impl {impl} {Ci}->{Co} k{k} s{s}'
                cnn.CONV_IMPL = impl
                # fused epilogue (bias + LeakyReLU) in the forward ...
                assert_close(cnn.conv2d(x, w, b, None, s, p, 'leaky', 0.2), F.leaky_relu(F.conv2d(xd, wd, bd, s, p), 0.2), tol,
                             tag + ' fprop+leaky')
                # ... gradients with a linear epilogue: a forward difference of 1e-6 flips LeakyReLU masks of
                # near-zero pre-activations, which changes dx by ~1e-2 for ANY two implementations
                zd = F.conv2d(xd, wd, bd, s, p)
                wt = _wts(zd.shape, 5, device)
                gd = torch.autograd.grad((zd * wt.double()).sum(), [xd, wd, bd])
                y = cnn.conv2d(x, w, b, None, s, p, None, 0.2)
                assert_close(y, zd, tol, tag + ' fprop')
                gx, gw, gb = torch.autograd.grad((y * wt).sum(), [x, w, b])
                assert_close(gx, gd[0], tol, tag + ' dgrad')
                assert_close(gw, gd[1], tol, tag + ' wgrad')
                assert_close(gb, gd[2], tol, tag + ' bias grad')
        # ConvTranspose2d forward == strided dgrad parity classes
        x = torch.randn(4, 96, 8, 28, generator=g).to(device).requires_grad_(True)      # small M per parity class: split-K
        b = torch.randn(32, generator=g).to(device)
        cnn.CONV_IMPL = _lib.IMPL_TC
        for (k, op) in ((4, 0), (3, 1)):
            w = (torch.randn(96, 32, k, k, generator=g) * 0.05).to(device).requires_grad_(True)
            xd, wd = x.detach().double().requires_grad_(True), w.detach().double().requires_grad_(True)
            zd = F.conv_transpose2d(xd, wd, b.double(), 2, 1, op)
            y = cnn.conv_transpose2d(x, w, b, 2, 1, op, None)
            assert_close(y, zd, 1e-4, f'tc convT k{k} s2')
            wt = _wts(zd.shape, 6, device)
            ga = torch.autograd.grad((y * wt).sum(), [x, w])
            gb_ = torch.autograd.grad((zd * wt.double()).sum(), [xd, wd])
            assert_close(ga[0], gb_[0], 1e-4, f'tc convT k{k} dx')
            assert_close(ga[1], gb_[1], 1e-4, f'tc convT k{k} dw')
    finally:
        cnn.CONV_IMPL = saved


def _conv_cross_check(device, shapes, seed, name):
    """Every shape through both convolution families - the wgmma tensor-core kernels (IMPL_TC, 3xTF32) and the CUDA-core
    FFMA kernels - each against torch fp64 and against each other: two independent implementations of the same
    convolution, forward with a fused bias + LeakyReLU epilogue and with a linear one, data / weight / bias gradients."""
    from cc_b200 import _lib
    g = torch.Generator().manual_seed(seed)
    saved = cnn.CONV_IMPL
    try:
        for (B, Ci, H, W, Co, k, s, p) in shapes:
            tag = f'{name} {Ci}->{Co} k{k} s{s} {H}x{W}'
            x = torch.randn(B, Ci, H, W, generator=g).to(device).requires_grad_(True)
            w = (torch.randn(Co, Ci, k, k, generator=g) / (Ci * k * k) ** 0.5).to(device).requires_grad_(True)
            b = torch.randn(Co, generator=g).to(device).requires_grad_(True)
            xd, wd, bd = [t.detach().double().requires_grad_(True) for t in (x, w, b)]
            zd = F.conv2d(xd, wd, bd, s, p)
            wt = _wts(zd.shape, 9, device)
            gd = torch.autograd.grad((zd * wt.double()).sum(), [xd, wd, bd])
            outs = {}
            for impl in (_lib.IMPL_TC, _lib.IMPL_FFMA):
                cnn.CONV_IMPL = impl
                assert_close(cnn.conv2d(x, w, b, None, s, p, 'leaky', 0.2), F.leaky_relu(zd, 0.2), 1e-4, f'{tag} impl {impl} fprop+leaky')
                y = cnn.conv2d(x, w, b, None, s, p, None, 0.2)
                gx, gw, gb = torch.autograd.grad((y * wt).sum(), [x, w, b])
                outs[impl] = (y.detach(), gx, gw, gb)
                for got, ref, what in zip(outs[impl], (zd,) + tuple(gd), ('fprop', 'dgrad', 'wgrad', 'bias grad')):
                    assert_close(got, ref, 1e-4, f'{tag} impl {impl} {what}')
            for a_, b_, what in zip(outs[_lib.IMPL_TC], outs[_lib.IMPL_FFMA], ('fprop', 'dgrad', 'wgrad', 'bias grad')):
                assert_close(a_, b_, 1e-4, f'{tag} tensor-core vs CUDA-core kernels {what}')
    finally:
        cnn.CONV_IMPL = saved


def case_conv_tma_family(device):
    """(Named after the removed TMA-fed Blackwell kernels whose dispatch branches these shapes reached.)  Thin and odd layer
    geometries: ragged channels / rows / columns, stride-2 thin input (PoseNet conv1), one output
    channel (disparity head), ragged tile bottoms, several 32-channel K blocks with column tails, narrow maps whose width is
    not a multiple of 4 (weight gradient through padded rows), 1x1 with N > 128.  GPU only."""
    _conv_cross_check(device, [(6, 13, 100, 260, 20, 3, 1, 1),
                               (4, 15, 256, 832, 16, 7, 2, 3),
                               (4, 16, 252, 832, 1, 3, 1, 1),
                               (4, 32, 126, 416, 32, 3, 1, 1),
                               (2, 160, 12, 36, 72, 3, 1, 1),
                               (2, 24, 9, 22, 40, 3, 1, 1),
                               (2, 40, 16, 64, 136, 1, 1, 0)], 11, 'thin/odd')


def case_conv_nhwc(device):
    """(Named after the removed channels-last Blackwell slab kernel these shapes exercised.)  The layer geometries of the four networks' heavy convolutions: the ResBlock shape, a 7x7 halo (DispResNet6 conv1b),
    channel tails (196 = 6 x 32 + 4), 5x5 with an N tail, few tiles with a long K (split-K, 2 N tiles), stride-2 DGRAD
    parity classes, the MaskNet6 deconv geometry (k4 s2 p1).  GPU only."""
    _conv_cross_check(device, [(2, 64, 32, 40, 64, 3, 1, 1),
                               (2, 32, 48, 72, 32, 7, 1, 3),
                               (2, 196, 20, 44, 128, 3, 1, 1),
                               (2, 100, 33, 23, 72, 5, 1, 2),
                               (1, 512, 16, 24, 200, 3, 1, 1),
                               (2, 64, 48, 64, 48, 3, 2, 1),
                               (2, 96, 40, 56, 64, 4, 2, 1)], 13, 'network')


ALT_NETS = [  # mirrors tests/golden/make_golden.py:ALT_NETS (name, kwargs, input size, frozen gradients)
    ('DispNetS', {}, (2, 64, 128), ['conv1.0.weight', 'conv7.2.bias', 'upconv4.0.weight', 'iconv3.0.weight', 'predict_disp4.0.weight']),
    ('DispNetS6', {}, (2, 64, 128), ['conv1.2.weight', 'conv5.0.bias', 'upconv7.0.weight', 'iconv1.0.weight', 'predict_disp6.0.bias']),
    ('DispResNetS6', {}, (2, 64, 128), ['conv1.0.weight', 'conv4.2.conv2.weight', 'iconv5.1.conv1.weight', 'iconv7.0.downsample.1.bias',
                                       'predict_disp1.0.weight']),
    ('PoseNet6', dict(nb_ref_imgs=4), (2, 128, 128), ['conv0.0.weight', 'conv1.0.weight', 'conv7.0.bias', 'pose_pred.weight']),
    ('PoseExpNet', dict(nb_ref_imgs=4, output_exp=True), (2, 64, 128), ['conv1.0.weight', 'conv6.0.weight', 'upconv5.0.weight',
                                                                      'upconv1.0.bias', 'predict_mask4.weight', 'pose_pred.bias']),
    ('MaskResNet6', dict(nb_ref_imgs=4, output_exp=True), (2, 128, 128), ['conv1.0.weight', 'conv3.0.downsample.1.weight', 'conv6.1.conv2.weight',
                                                                        'deconv6.0.weight', 'deconv1.0.bias', 'pred_mask1.weight']),
]


def _alt_outputs(name, net, tgt, refs):
    if name.startswith('Disp'):
        return list(net(tgt))
    if name == 'PoseNet6':
        return [net(tgt, refs)]
    if name == 'PoseExpNet':
        masks, pose = net(tgt, refs)
        return list(masks) + [pose]
    return list(net(tgt, refs))


def case_alt_nets(device, names=None, grads=True):
    """The reference's alternate architectures (SURVEY N4; cc_b200/models/alternates.py) against fixtures frozen from the
    reference's own modules (tests/golden/alt_nets_small.npz): weights come from synth.seeded_fill on both sides (state_dict
    key names and shapes must therefore agree), train-mode outputs at 1e-4, a sample of parameter gradients, eval output.
    Gradient bars: 2e-3 for the plain nets; the two residual nets carry BatchNorm over 2-16 values at this toy input size
    (DispResNetS6's conv7 sees a 1x2 map) and are held to 1e-1 (chaotic conditioning, see tests/fullsize_cases.py; measured on
    DispResNet6; the exact-fp32 simulator run already shows 6e-2 against torch on one tensor)."""
    g = golden('alt_nets_small')
    for k, (name, kw, (B, H, W), pn) in enumerate(ALT_NETS):
        if names is not None and name not in names:
            continue
        tgt, refs = synth.frames(B, H, W, seed=190 + k)
        tgt, refs = tgt.to(device), [r.to(device) for r in refs]
        net = getattr(CM, name)(**kw)
        ref_keys = {kk[len(name) + 3:].split('@')[0] for kk in g if kk.startswith(name + '_g_')}
        assert ref_keys <= set(dict(net.named_parameters())), f'{name}: state_dict keys differ from the reference'
        net = synth.seeded_fill(net, 300 + k).to(device)
        net.train()
        outs = _alt_outputs(name, net, tgt, refs)
        for i, x in enumerate(outs):
            assert_close(x, g[f'{name}_out{i}'], TOL, f'{name} out{i}')
        if grads:
            loss = sum((x * _wts(x.shape, 400 + 10 * k + i, device)).sum() for i, x in enumerate(outs))
            pd = dict(net.named_parameters())
            gs = torch.autograd.grad(loss, [pd[n] for n in pn])
            gtol = 1e-1 if 'Res' in name else 2e-3
            for n, gg in zip(pn, gs):
                key, st = key_with_stride(g, f'{name}_g_{n}')
                assert_close(pick(gg, st), g[key], gtol, f'{name} grad {n}')
        net.eval()
        with torch.no_grad():
            e = net(tgt) if name.startswith('Disp') else net(tgt, refs)
        e = e if torch.is_tensor(e) else (e[1] if name == 'PoseExpNet' else e[0])
        assert_close(e, g[f'{name}_eval'], TOL, f'{name} eval')


def case_alt_pose_nets(device):
    case_alt_nets(device, names=('PoseNet6', 'PoseExpNet'))


def case_bn_upsample(device):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(3, 6, 5, 7, generator=g).to(device).requires_grad_(True)
    bn = cnn.BatchNorm2d(6).to(device)
    ref = torch.nn.BatchNorm2d(6).to(device)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(6, generator=g) + 0.5); bn.bias.copy_(torch.randn(6, generator=g))
        ref.weight.copy_(bn.weight); ref.bias.copy_(bn.bias)
    y, z = bn(x), ref(x)
    assert_close(y, z, TOL, 'bn fwd')
    wt = _wts(y.shape, 3, device)
    ga = torch.autograd.grad((y * wt).sum(), [x, bn.weight, bn.bias])
    gb = torch.autograd.grad((z * wt).sum(), [x, ref.weight, ref.bias])
    for a_, b_, nm in zip(ga, gb, ('dx', 'dgamma', 'dbeta')):
        assert_close(a_, b_, TOL, 'bn ' + nm)
    assert_close(bn.running_mean, ref.running_mean, TOL, 'bn running_mean')
    assert_close(bn.running_var, ref.running_var, TOL, 'bn running_var')
    bn.eval(); ref.eval()
    assert_close(bn(x), ref(x), TOL, 'bn eval')
    # multi-split path (B*plane > 8192 values per channel) incl. a large common offset (Chan merge stability)
    xb = (torch.randn(2, 3, 80, 70, generator=g) + 30.0).to(device).requires_grad_(True)
    bn2, ref2 = cnn.BatchNorm2d(3).to(device), torch.nn.BatchNorm2d(3).to(device)
    y, z = bn2(xb), ref2(xb)
    assert_close(y, z, TOL, 'bn multi-split fwd')
    wt = _wts(y.shape, 8, device)
    for a_, b_, nm in zip(torch.autograd.grad((y * wt).sum(), [xb, bn2.weight, bn2.bias]),
                          torch.autograd.grad((z * wt).sum(), [xb, ref2.weight, ref2.bias]), ('dx', 'dgamma', 'dbeta')):
        assert_close(a_, b_, TOL, 'bn multi-split ' + nm)
    assert_close(bn2.running_var, ref2.running_var, TOL, 'bn multi-split running_var')
    x2 = torch.randn(2, 3, 5, 9, generator=g).to(device).requires_grad_(True)
    u = cnn.upsample2x(x2)
    v = F.interpolate(x2, scale_factor=2, mode='bilinear', align_corners=False)
    assert_close(u, v, 1e-6, 'upsample2x')
    wt = _wts(u.shape, 4, device)
    assert_close(torch.autograd.grad((u * wt).sum(), [x2])[0], torch.autograd.grad((v * wt).sum(), [x2])[0], 1e-6, 'upsample2x bwd')


def _load(mod, params, device):
    mod.load_state_dict({k: v.clone() for k, v in params.items()}, strict=True)
    return mod.to(device)


def _check_grads(g, prefix, names, pd, grads, tol):
    for n, gg in zip(names, grads):
        k, stride = key_with_stride(g, prefix + n)
        assert_close(pick(gg, stride), g[k], tol, k)


def case_disp_pose_golden(device):
    """DispResNet6 + PoseNetB6 modules (reference state_dict keys) vs fixtures from the reference nets.
    Strict (grads 5e-4) with the exact-fp32 FFMA kernels; with the default (tensor-core, 3xTF32) path the
    OUTPUTS meet the 1e-4 bar, while first-layer weight gradients are only held to 5e-2 at this tiny size: the
    deepest BatchNorms normalise over 2-8 values and amplify the ~1e-5 tensor-core accumulation error ~500x
    (same net at 128x416 and up: see tests/step_cases.py)."""
    from cc_b200 import _lib
    saved = cnn.CONV_IMPL
    try:
        cnn.CONV_IMPL = _lib.IMPL_FFMA
        _disp_pose_golden(device, 5e-4)
        if device.type == 'cuda':
            cnn.CONV_IMPL = _lib.IMPL_AUTO
            _disp_pose_golden(device, 5e-2)
    finally:
        cnn.CONV_IMPL = saved


def _disp_pose_golden(device, gtol):
    g = golden('nets_small')
    tgt, refs = synth.frames(2, 64, 128, seed=40)
    tgt, refs = tgt.to(device), [r.to(device) for r in refs]
    net = _load(CM.DispResNet6(), ON.disp_params(), device)
    net.train()
    disps = net(tgt)
    for i, x in enumerate(disps):
        assert_close(x, g[f'disp_out{i}'], TOL, f'disp{i}')
    names = ['conv1.0.weight', 'conv1.2.bias', 'conv2.0.conv1.weight', 'conv2.0.downsample.0.weight',
             'conv2.0.downsample.1.weight', 'conv2.0.downsample.1.bias', 'conv7.1.conv2.weight',
             'upconv7.0.weight', 'upconv1.0.bias', 'iconv1.0.conv1.weight', 'iconv3.0.downsample.0.weight',
             'predict_disp1.0.weight', 'predict_disp6.0.bias']
    pd = dict(net.named_parameters())
    loss = sum((x * _wts(x.shape, 50 + i, device)).sum() for i, x in enumerate(disps))
    _check_grads(g, 'disp_g_', names, pd, torch.autograd.grad(loss, [pd[n] for n in names]), gtol)
    sd = net.state_dict()
    assert_close(sd['conv2.0.downsample.1.running_mean'], g['disp_rm'], TOL, 'running_mean')
    assert_close(sd['iconv1.0.downsample.1.running_var'], g['disp_rv'], TOL, 'running_var')
    net.eval()
    with torch.no_grad():
        assert_close(net(tgt), g['disp_eval'], TOL, 'disp eval')
        net.train()
        t2, _ = synth.frames(2, 24, 40, seed=41)
        for i, x in enumerate(net(t2.to(device))):
            assert_close(x, g[f'disp_odd_out{i}'], TOL, f'disp odd {i}')
    pnet = _load(CM.PoseNetB6(nb_ref_imgs=4), ON.pose_params(), device)
    pose = pnet(tgt, refs)
    assert_close(pose, g['pose_out'], TOL, 'pose')
    pn = ['conv1.0.weight', 'conv2.0.weight', 'conv8.0.bias', 'pose_pred.weight', 'pose_pred.bias']
    ppd = dict(pnet.named_parameters())
    _check_grads(g, 'pose_g_', pn, ppd, torch.autograd.grad((pose * _wts(pose.shape, 60, device)).sum(), [ppd[n] for n in pn]), gtol)


def case_mask_golden(device):
    g = golden('nets_small')
    tgt, refs = synth.frames(1, 64, 64, seed=42)
    tgt, refs = tgt.to(device), [r.to(device) for r in refs]
    mnet = _load(CM.MaskNet6(nb_ref_imgs=4, output_exp=True), ON.mask_params(), device)
    mnet.train()
    ms = mnet(tgt, refs)
    for i, x in enumerate(ms):
        assert_close(x, g[f'mask_out{i}'], TOL, f'mask{i}')
    mn = ['conv1.0.weight', 'conv6.0.weight', 'deconv6.0.weight', 'deconv1.0.weight', 'deconv3.0.bias',
          'pred_mask1.weight', 'pred_mask6.bias']
    mpd = dict(mnet.named_parameters())
    loss = sum((x * _wts(x.shape, 70 + i, device)).sum() for i, x in enumerate(ms))
    _check_grads(g, 'mask_g_', mn, mpd, torch.autograd.grad(loss, [mpd[n] for n in mn]), 5e-4)


def case_flow_golden(device):
    """Back2Future module + cost volume + feature warp vs fixtures from the reference net (stub correlation:
    the third-party op is the one parity-unpinned boundary, oracle/nets.py)."""
    g = golden('nets_small')
    tgt, refs = synth.frames(1, 64, 64, seed=42)
    tgt, refs = tgt.to(device), [r.to(device) for r in refs]
    fnet = _load(CM.Back2Future(nlevels=6), ON.flow_params(), device)
    fnet.train()
    ff, fb, occ = fnet(tgt, refs[1:3])
    for i in range(6):
        assert_close(ff[i], g[f'flow_fwd{i}'], 2e-4, f'flow_fwd{i}')
        assert_close(fb[i], g[f'flow_bwd{i}'], 2e-4, f'flow_bwd{i}')
    assert_close(occ[0][:, :, ::4, ::4], g['flow_occ0'], 2e-4, 'occ0')
    assert_close(occ[5], g['flow_occ5'], 2e-4, 'occ5')
    fn = ['conv1a.0.weight', 'conv1b.2.bias', 'conv6c.0.weight', 'decoder_fwd6.0.weight',
          'decoder_bwd2.10.weight', 'decoder_fwd2.0.weight', 'decoder_bwd4.4.bias']
    fpd = dict(fnet.named_parameters())
    lossf = sum((x * _wts(x.shape, 80 + i, device)).sum() + (y * _wts(x.shape, 80 + i, device)).sum() * 0.5
                for i, (x, y) in enumerate(zip(ff, fb)))
    _check_grads(g, 'flow_g_', fn, fpd, torch.autograd.grad(lossf, [fpd[n] for n in fn]), 1e-3)
    fnet.eval()
    with torch.no_grad():
        e = fnet(tgt, refs[1:3])
        assert_close(e[0][:, :, ::2, ::2], g['flow_eval_fwd'], 2e-4, 'flow eval')
    # cost volume / feature warp in isolation against the oracle restatement
    gen = torch.Generator().manual_seed(3)
    f1 = torch.randn(2, 12, 9, 13, generator=gen).to(device).requires_grad_(True)
    f2 = torch.randn(2, 12, 9, 13, generator=gen).to(device).requires_grad_(True)
    for rev, idx in ((False, ON.IDX_FWD), (True, ON.IDX_BWD)):
        a_ = cnn.corr81(f1, f2, rev)
        b_ = ON.correlate(f1, f2).index_select(1, torch.tensor(idx, device=device))
        assert_close(a_, b_, TOL, 'corr81')
        wt = _wts(a_.shape, 9, device)
        for x_, y_, nm in zip(torch.autograd.grad((a_ * wt).sum(), [f1, f2]), torch.autograd.grad((b_ * wt).sum(), [f1, f2]), ('df1', 'df2')):
            assert_close(x_, y_, TOL, 'corr81 ' + nm)
    flo = (torch.randn(2, 2, 9, 13, generator=gen) * 2).to(device).requires_grad_(True)
    a_, b_ = cnn.feat_warp(f1, flo), ON.b2f_warp(f1, flo)
    assert_close(a_, b_, TOL, 'feat_warp')
    wt = _wts(a_.shape, 10, device)
    for x_, y_, nm in zip(torch.autograd.grad((a_ * wt).sum(), [f1, flo]), torch.autograd.grad((b_ * wt).sum(), [f1, flo]), ('dx', 'dflow')):
        assert_close(x_, y_, TOL, 'feat_warp ' + nm)


def smoke_case(device):
    case_conv_shapes(device)


NET_CASES = [case_conv_shapes, case_bn_upsample, case_disp_pose_golden, case_mask_golden, case_flow_golden, case_alt_pose_nets]
