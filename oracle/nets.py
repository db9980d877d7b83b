"""Oracle: the hot-path CNNs as *functional* fp32 forwards over a state_dict.
TEST INFRASTRUCTURE.

Key names and shapes equal the reference modules' ``state_dict()`` (checkpoint
contract, reference utils.py:55-63), so the same dict drives the reference module,
this oracle and the CUDA product.

* DispResNet6 : reference models/DispResNet6.py:97-194
* PoseNetB6   : reference models/PoseNetB6.py:24-83
* MaskNet6    : reference models/MaskNet6.py:19-123
* Back2Future : reference models/back2future.py:51-321
* FlowNetC6   : reference models/FlowNetC6.py:32-164 (+ submodules.py:5-39); the flow net of --flownet FlowNetC6

PARITY UNPINNED at one boundary: ``spatial_correlation_sample`` restates the published
behaviour of the third-party ``spatial_correlation_sampler`` (PyPI spatial-correlation-sampler,
version un-pinned in reference requirements.txt:13, upstream
ClementPinard/Pytorch-Correlation-extension; source absent from the reference repository):
out[b,ph,pw,y,x] = sum_c in1[b,c,y,x] * in2[b,c,y+d(ph-P//2),x+d(pw-P//2)] (zero outside), with
kernel_size=1, stride=1, padding=0; the first patch index is the vertical displacement.
Back2Future calls it with patch_size P=9, dilation_patch d=1, FlowNetC6 with P=21, d=2.  It is
anchored only by the reference's call sites and Back2Future's permutation tables
(back2future.py:15-25,56-59, FlowNetC6.py:18-30).
"""
import math
import numpy as np
import torch
import torch.nn.functional as F

# ----------------------------------------------------------------------------- specs
DISP_CONV_PLANES = [32, 64, 128, 256, 512, 512, 512]
DISP_UPCONV_PLANES = [512, 512, 256, 128, 64, 32, 16]
POSE_PLANES = [16, 32, 64, 128, 256, 256, 256, 256]
MASK_UPCONV_PLANES = [256, 256, 128, 64, 32, 16]
B2F_FEAT = [(3, 16), (16, 32), (32, 64), (64, 96), (96, 128), (128, 192)]
B2F_DEC_IN = {6: 162, 5: 292, 4: 260, 3: 228, 2: 196}
B2F_DEC_PLANES = [128, 128, 96, 64, 32, 2]


def _xavier(shape, gen, fan_in, fan_out):
    a = math.sqrt(6.0 / (fan_in + fan_out))
    return (torch.rand(shape, generator=gen) * 2 - 1) * a


def _conv_p(p, name, cin, cout, k, gen, bias=True, transposed=False, bias_uniform=False):
    rf = k * k
    if transposed:
        shape = (cin, cout, k, k)      # torch ConvTranspose2d weight layout
        fan_in, fan_out = cout * rf, cin * rf
    else:
        shape = (cout, cin, k, k)
        fan_in, fan_out = cin * rf, cout * rf
    p[name + '.weight'] = _xavier(shape, gen, fan_in, fan_out)
    if bias:
        p[name + '.bias'] = torch.rand(cout, generator=gen) if bias_uniform else torch.zeros(cout)


def _bn_p(p, name, c):
    p[name + '.weight'] = torch.ones(c)
    p[name + '.bias'] = torch.zeros(c)
    p[name + '.running_mean'] = torch.zeros(c)
    p[name + '.running_var'] = torch.ones(c)
    p[name + '.num_batches_tracked'] = torch.tensor(0, dtype=torch.long)


def _basic_layer_p(p, name, inplanes, planes, blocks, stride, gen):
    for b in range(blocks):
        cin = inplanes if b == 0 else planes
        _conv_p(p, f'{name}.{b}.conv1', cin, planes, 3, gen, bias=False)
        _conv_p(p, f'{name}.{b}.conv2', planes, planes, 3, gen, bias=False)
        if b == 0 and (stride != 1 or inplanes != planes):
            _conv_p(p, f'{name}.{b}.downsample.0', inplanes, planes, 1, gen, bias=False)
            _bn_p(p, f'{name}.{b}.downsample.1', planes)


def disp_params(seed=0):
    """Xavier-uniform weights / zero bias like DispResNet6.init_weights (DispResNet6.py:138-143)."""
    g = torch.Generator().manual_seed(seed)
    p = {}
    cp, up = DISP_CONV_PLANES, DISP_UPCONV_PLANES
    _conv_p(p, 'conv1.0', 3, cp[0], 7, g)
    _conv_p(p, 'conv1.2', cp[0], cp[0], 7, g)
    for i in range(1, 7):
        _basic_layer_p(p, f'conv{i + 1}', cp[i - 1], cp[i], 2, 2, g)
    ins = [cp[6]] + up[:6]
    for j, n in enumerate(range(7, 0, -1)):
        _conv_p(p, f'upconv{n}.0', ins[j], up[j], 3, g, transposed=True)
    iconv_in = {7: up[0] + cp[5], 6: up[1] + cp[4], 5: up[2] + cp[3], 4: up[3] + cp[2],
                3: 1 + up[4] + cp[1], 2: 1 + up[5] + cp[0], 1: 1 + up[6]}
    for j, n in enumerate(range(7, 0, -1)):
        _basic_layer_p(p, f'iconv{n}', iconv_in[n], up[j], 1, 1, g)
    for n, c in zip(range(6, 0, -1), up[1:]):
        _conv_p(p, f'predict_disp{n}.0', c, 1, 3, g)
    return p


def pose_params(nb_ref_imgs=4, seed=1):
    g = torch.Generator().manual_seed(seed)
    p = {}
    pl = POSE_PLANES
    ks = [7, 5, 3, 3, 3, 3, 3, 3]
    cin = 3 * (1 + nb_ref_imgs)
    for i in range(8):
        _conv_p(p, f'conv{i + 1}.0', cin, pl[i], ks[i], g)
        cin = pl[i]
    _conv_p(p, 'pose_pred', pl[7], 6 * nb_ref_imgs, 1, g)
    return p


def mask_params(nb_ref_imgs=4, seed=2):
    g = torch.Generator().manual_seed(seed)
    p = {}
    pl, up = POSE_PLANES, MASK_UPCONV_PLANES
    ks = [7, 5, 3, 3, 3, 3]
    cin = 3 * (1 + nb_ref_imgs)
    for i in range(6):
        _conv_p(p, f'conv{i + 1}.0', cin, pl[i], ks[i], g)
        cin = pl[i]
    dins = [pl[5], up[0] + pl[4], up[1] + pl[3], up[2] + pl[2], up[3] + pl[1], up[4] + pl[0]]
    for j, n in enumerate(range(6, 0, -1)):
        _conv_p(p, f'deconv{n}.0', dins[j], up[j], 4, g, transposed=True)
        _conv_p(p, f'pred_mask{n}', up[j], nb_ref_imgs, 3, g)
    return p


def flow_params(seed=3):
    """Back2Future.init_weights: xavier weights, U[0,1) biases (back2future.py:106-116)."""
    g = torch.Generator().manual_seed(seed)
    p = {}
    for lvl, (ci, co) in enumerate(B2F_FEAT, start=1):
        for tower in 'abc':
            _conv_p(p, f'conv{lvl}{tower}.0', ci, co, 3, g, bias_uniform=True)
            _conv_p(p, f'conv{lvl}{tower}.2', co, co, 3, g, bias_uniform=True)
    for lvl in range(6, 1, -1):
        for kind in ('fwd', 'bwd', 'occ'):
            cin = 354 if (kind == 'occ' and lvl == 6) else B2F_DEC_IN[lvl]
            for j, co in enumerate(B2F_DEC_PLANES):
                _conv_p(p, f'decoder_{kind}{lvl}.{2 * j}', cin, co, 3, g, bias_uniform=True)
                cin = co
    return p


def clone_params(p, requires_grad=False, device=None):
    out = {}
    for k, v in p.items():
        t = v.detach().clone()
        if device is not None:
            t = t.to(device)
        if requires_grad and t.is_floating_point() and 'running_' not in k:
            t.requires_grad_(True)
        out[k] = t
    return out


# ----------------------------------------------------------------------------- DispResNet6
def _bn(p, name, x, training):
    return F.batch_norm(x, p[name + '.running_mean'], p[name + '.running_var'],
                        p[name + '.weight'], p[name + '.bias'], training, 0.1, 1e-5)


def _basic_block(p, name, x, stride, training):
    out = F.relu(F.conv2d(x, p[name + '.conv1.weight'], None, stride, 1))
    out = F.conv2d(out, p[name + '.conv2.weight'], None, 1, 1)
    if (name + '.downsample.0.weight') in p:
        res = _bn(p, name + '.downsample.1',
                  F.conv2d(x, p[name + '.downsample.0.weight'], None, stride, 0), training)
    else:
        res = x
    return F.relu(out + res)


def _layer(p, name, x, blocks, stride, training):
    for b in range(blocks):
        x = _basic_block(p, f'{name}.{b}', x, stride if b == 0 else 1, training)
    return x


def _crop_like(x, ref):
    assert x.size(2) >= ref.size(2) and x.size(3) >= ref.size(3)
    return x[:, :, :ref.size(2), :ref.size(3)]


def disp_forward(p, x, training=True, alpha=10, beta=0.01):
    """Reference models/DispResNet6.py:145-194."""
    c = F.relu(F.conv2d(x, p['conv1.0.weight'], p['conv1.0.bias'], 2, 3))
    c1 = F.relu(F.conv2d(c, p['conv1.2.weight'], p['conv1.2.bias'], 1, 3))
    feats = [c1]
    for n in range(2, 8):
        feats.append(_layer(p, f'conv{n}', feats[-1], 2, 2, training))
    c1, c2, c3, c4, c5, c6, c7 = feats

    def up(n, t):
        return F.relu(F.conv_transpose2d(t, p[f'upconv{n}.0.weight'], p[f'upconv{n}.0.bias'],
                                         stride=2, padding=1, output_padding=1))

    def pred(n, t):
        return alpha * torch.sigmoid(F.conv2d(t, p[f'predict_disp{n}.0.weight'],
                                              p[f'predict_disp{n}.0.bias'], 1, 1)) + beta

    def up2(d, ref):
        return _crop_like(F.interpolate(d, scale_factor=2, mode='bilinear', align_corners=False), ref)

    i7 = _layer(p, 'iconv7', torch.cat((_crop_like(up(7, c7), c6), c6), 1), 1, 1, training)
    i6 = _layer(p, 'iconv6', torch.cat((_crop_like(up(6, i7), c5), c5), 1), 1, 1, training)
    d6 = pred(6, i6)
    i5 = _layer(p, 'iconv5', torch.cat((_crop_like(up(5, i6), c4), c4), 1), 1, 1, training)
    d5 = pred(5, i5)
    i4 = _layer(p, 'iconv4', torch.cat((_crop_like(up(4, i5), c3), c3), 1), 1, 1, training)
    d4 = pred(4, i4)
    i3 = _layer(p, 'iconv3', torch.cat((_crop_like(up(3, i4), c2), c2, up2(d4, c2)), 1), 1, 1, training)
    d3 = pred(3, i3)
    i2 = _layer(p, 'iconv2', torch.cat((_crop_like(up(2, i3), c1), c1, up2(d3, c1)), 1), 1, 1, training)
    d2 = pred(2, i2)
    i1 = _layer(p, 'iconv1', torch.cat((_crop_like(up(1, i2), x), up2(d2, x)), 1), 1, 1, training)
    d1 = pred(1, i1)
    return (d1, d2, d3, d4, d5, d6) if training else d1


# ----------------------------------------------------------------------------- PoseNetB6 / MaskNet6
def pose_forward(p, tgt, refs):
    """Reference models/PoseNetB6.py:65-83."""
    nb = p['pose_pred.weight'].size(0) // 6
    assert len(refs) == nb
    x = torch.cat([tgt] + list(refs), 1)
    ks = [7, 5, 3, 3, 3, 3, 3, 3]
    for i in range(8):
        x = F.relu(F.conv2d(x, p[f'conv{i + 1}.0.weight'], p[f'conv{i + 1}.0.bias'], 2, (ks[i] - 1) // 2))
    pose = F.conv2d(x, p['pose_pred.weight'], p['pose_pred.bias'])
    pose = pose.mean(3).mean(2)
    return 0.01 * pose.view(pose.size(0), nb, 6)


def mask_forward(p, tgt, refs, training=True):
    """Reference models/MaskNet6.py:80-123."""
    x = torch.cat([tgt] + list(refs), 1)
    ks = [7, 5, 3, 3, 3, 3]
    enc = []
    for i in range(6):
        x = F.relu(F.conv2d(x, p[f'conv{i + 1}.0.weight'], p[f'conv{i + 1}.0.bias'], 2, (ks[i] - 1) // 2))
        enc.append(x)

    def dec(n, t):
        return F.relu(F.conv_transpose2d(t, p[f'deconv{n}.0.weight'], p[f'deconv{n}.0.bias'],
                                         stride=2, padding=1))

    ups = [dec(6, enc[5])]
    for n in range(5, 0, -1):
        ups.append(dec(n, torch.cat((ups[-1], enc[n - 1]), 1)))
    masks = [torch.sigmoid(F.conv2d(ups[6 - n], p[f'pred_mask{n}.weight'], p[f'pred_mask{n}.bias'], 1, 1))
             for n in range(6, 0, -1)]
    masks = masks[::-1]                       # exp_mask1 .. exp_mask6
    return tuple(masks) if training else masks[0]


# ----------------------------------------------------------------------------- Back2Future
_IDX = list(np.array([list(range(n, -1, -9)) for n in range(80, 71, -1)]).flatten())
IDX_FWD = [int(i) for i in _IDX]              # back2future.py:56-58
IDX_BWD = [int(i) for i in reversed(_IDX)]    # back2future.py:59


def spatial_correlation_sample(in1, in2, patch=9, dilation=1):
    """Restated third-party op (see module docstring): [B,C,H,W]x2 -> [B,patch,patch,H,W]."""
    B, C, H, W = in1.shape
    r = (patch // 2) * dilation
    pad = F.pad(in2, (r, r, r, r))
    rows = []
    for ph in range(patch):
        y = ph * dilation
        rows.append(torch.stack([(in1 * pad[:, :, y:y + H, pw * dilation:pw * dilation + W]).sum(1) for pw in range(patch)], 1))
    return torch.stack(rows, 1)


def correlate(in1, in2):
    """Reference models/back2future.py:15-25."""
    out = spatial_correlation_sample(in1, in2)
    b, ph, pw, h, w = out.size()
    return out.view(b, ph * pw, h, w) / in1.size(1)


def b2f_normalize(im):
    """Reference models/back2future.py:118-132."""
    im = im * 0.5 + 0.5
    mean = im.new_tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
    std = im.new_tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    return (im - mean) / std


def b2f_warp(x, flo):
    """Feature warp, border padding; the ones-mask is computed then discarded in the
    reference (``return output#*mask``).  Reference models/back2future.py:287-321."""
    B, C, H, W = x.size()
    xx = torch.arange(0, W, dtype=x.dtype, device=x.device).view(1, 1, 1, W).expand(B, 1, H, W)
    yy = torch.arange(0, H, dtype=x.dtype, device=x.device).view(1, 1, H, 1).expand(B, 1, H, W)
    vx = 2.0 * (xx + flo[:, 0:1]) / max(W - 1, 1) - 1.0
    vy = 2.0 * (yy + flo[:, 1:2]) / max(H - 1, 1) - 1.0
    grid = torch.cat((vx, vy), 1).permute(0, 2, 3, 1)
    return F.grid_sample(x, grid, mode='bilinear', padding_mode='border', align_corners=False)


def _feat_block(p, name, x):
    x = F.leaky_relu(F.conv2d(x, p[name + '.0.weight'], p[name + '.0.bias'], 2, 1), 0.2)
    return F.leaky_relu(F.conv2d(x, p[name + '.2.weight'], p[name + '.2.bias'], 1, 1), 0.2)


def _dec_block(p, name, x):
    for j in range(6):
        x = F.conv2d(x, p[f'{name}.{2 * j}.weight'], p[f'{name}.{2 * j}.bias'], 1, 1)
        if j < 5:
            x = F.leaky_relu(x, 0.2)
    return x


def _up2(t):
    return F.interpolate(t, scale_factor=2, mode='bilinear', align_corners=False)


def flow_forward(p, im_tar, im_refs, nlevels=6, training=True, with_occ=True):
    """Reference models/back2future.py:134-285.  im_refs = [I-, I+]."""
    ims = [b2f_normalize(im) for im in [im_tar] + list(im_refs)]
    fa, fb, fc = [ims[0]], [ims[2]], [ims[1]]          # a: target, b: I+ , c: I-
    for lvl in range(1, 7):
        fa.append(_feat_block(p, f'conv{lvl}a', fa[-1]))
        fb.append(_feat_block(p, f'conv{lvl}b', fb[-1]))
        fc.append(_feat_block(p, f'conv{lvl}c', fc[-1]))
    idx_f = torch.tensor(IDX_FWD, device=im_tar.device)
    idx_b = torch.tensor(IDX_BWD, device=im_tar.device)
    scale = {5: 0.625, 4: 1.25, 3: 2.5, 2: 5.0}

    flows_f, flows_b, occs = {}, {}, {}
    fup_f = fup_b = None
    for lvl in range(6, 1, -1):
        if lvl == 6:
            b_feat, c_feat = fb[6], fc[6]
        else:
            b_feat = b2f_warp(fb[lvl], scale[lvl] * fup_f)
            c_feat = b2f_warp(fc[lvl], -scale[lvl] * fup_f)
        corr = torch.cat((correlate(fa[lvl], b_feat).index_select(1, idx_f),
                          correlate(fa[lvl], c_feat).index_select(1, idx_b)), 1)
        if lvl == 6:
            in_f = in_b = corr
            in_o = torch.cat((corr, fa[6]), 1)
        else:
            in_f = torch.cat((corr, fa[lvl], fup_f), 1)
            in_b = torch.cat((corr, fa[lvl], fup_b), 1)
            in_o = in_f
        flows_f[lvl] = _dec_block(p, f'decoder_fwd{lvl}', in_f)
        flows_b[lvl] = _dec_block(p, f'decoder_bwd{lvl}', in_b)
        if with_occ:
            occs[lvl] = F.softmax(_dec_block(p, f'decoder_occ{lvl}', in_o), dim=1)
        fup_f, fup_b = _up2(flows_f[lvl]), _up2(flows_b[lvl])
        flows_f[(lvl, 'up')], flows_b[(lvl, 'up')] = fup_f, fup_b

    mult = {2: 20.0, 3: 10.0, 4: 5.0, 5: 2.5, 6: 1.25}
    ff = [mult[l] * _up2(flows_f[(l, 'up')]) for l in range(2, 7)]
    fbw = [-mult[l] * _up2(flows_b[(l, 'up')]) for l in range(2, 7)]
    oc = [F.interpolate(occs[l], scale_factor=4, mode='nearest') for l in range(2, 7)] if with_occ else None
    if not training:
        return ff[0], fbw[0], (oc[0] if with_occ else None)
    if nlevels == 6:
        ff.append(0.625 * flows_f[(6, 'up')])
        fbw.append(-0.625 * flows_b[(6, 'up')])
        if with_occ:
            oc.append(F.interpolate(occs[6], scale_factor=2, mode='nearest'))
    return ff, fbw, oc


# ----------------------------------------------------------------------------- FlowNetC6
C6_SLOPE = 0.1
C6_NPARAMS = 39276490
# (name, in, out, kernel, stride) of the conv blocks (Conv2d + bias + LeakyReLU 0.1), registration order
C6_CONVS = [('conv1', 3, 64, 7, 2), ('conv2', 64, 128, 5, 2), ('conv3', 128, 256, 5, 2), ('conv_redir', 256, 32, 1, 1),
            ('conv3_1', 473, 256, 3, 1), ('conv4', 256, 512, 3, 2), ('conv4_1', 512, 512, 3, 1), ('conv5', 512, 512, 3, 2),
            ('conv5_1', 512, 512, 3, 1), ('conv6', 512, 1024, 3, 2), ('conv6_1', 1024, 1024, 3, 1)]
C6_DECONVS = [(5, 1024, 512), (4, 1026, 256), (3, 770, 128), (2, 386, 64), (1, 194, 32)]   # ConvT k4 s2 p1 + LeakyReLU
C6_PREDICT_IN = {6: 1024, 5: 1026, 4: 770, 3: 386, 2: 194, 1: 98}                          # 3x3 -> 2, no activation


def flownetc6_correlate(in1, in2):
    """Reference models/FlowNetC6.py:18-30: [B,441,H,W], divided by C (no activation)."""
    out = spatial_correlation_sample(in1, in2, patch=21, dilation=2)
    b, ph, pw, h, w = out.size()
    return out.view(b, ph * pw, h, w) / in1.size(1)


def flownetc6_forward(p, x1, x2, training=True, div_flow=20):
    """Train mode: (flow1, ..., flow6), each div_flow * bilinear x2 of the head (full_res=True); eval mode: flow1."""
    spec = {name: (k, s) for name, _, _, k, s in C6_CONVS}

    def conv(name, x):
        k, s = spec[name]
        return F.leaky_relu(F.conv2d(x, p[name + '.0.weight'], p[name + '.0.bias'], s, (k - 1) // 2), C6_SLOPE)

    def tower(x):
        c1 = conv('conv1', x)
        c2 = conv('conv2', c1)
        return c1, c2, conv('conv3', c2)

    c1a, c2a, c3a = tower(x1)
    c3b = tower(x2)[2]
    corr = F.leaky_relu(flownetc6_correlate(c3a, c3b), C6_SLOPE)
    c3_1 = conv('conv3_1', torch.cat((conv('conv_redir', c3a), corr), 1))
    c4 = conv('conv4_1', conv('conv4', c3_1))
    c5 = conv('conv5_1', conv('conv5', c4))
    c6 = conv('conv6_1', conv('conv6', c5))
    skips = {5: c5, 4: c4, 3: c3_1, 2: c2a, 1: c1a}
    pred = lambda n, t: F.conv2d(t, p['predict_flow%d.weight' % n], p['predict_flow%d.bias' % n], 1, 1)      # noqa: E731
    flows = {6: pred(6, c6)}
    feat = c6
    for n in range(5, 0, -1):
        dec = F.leaky_relu(F.conv_transpose2d(feat, p['deconv%d.0.weight' % n], p['deconv%d.0.bias' % n], stride=2, padding=1),
                           C6_SLOPE)
        up = F.conv_transpose2d(flows[n + 1], p['upsampled_flow%d_to_%d.weight' % (n + 1, n)],
                                p['upsampled_flow%d_to_%d.bias' % (n + 1, n)], stride=2, padding=1)
        feat = torch.cat((skips[n], dec, up), 1)
        flows[n] = pred(n, feat)
    outs = [div_flow * F.interpolate(flows[n], scale_factor=2, mode='bilinear', align_corners=False) for n in range(1, 7)]
    return tuple(outs) if training else outs[0]


# ----------------------------------------------------------------------------- the flow net of a step
def flow_pair(p, tgt, refs, flownet='Back2Future'):
    """(flow_fwd, flow_bwd) of the training step, train mode (reference train.py:462-466): Back2Future sees both
    neighbours in one call (no occlusion decoders), FlowNetC6 is called once per direction."""
    if flownet == 'Back2Future':
        ff, fb, _ = flow_forward(p, tgt, refs[1:3], training=True, with_occ=False)
        return ff, fb
    if flownet == 'FlowNetC6':
        return list(flownetc6_forward(p, tgt, refs[2])), list(flownetc6_forward(p, tgt, refs[1]))
    raise ValueError('unknown flow net %r' % (flownet,))


def flow_eval(p, tgt, refs, flownet='Back2Future'):
    """flow_fwd of the flow evaluation, eval mode (reference test_flow.py:122-125)."""
    if flownet == 'Back2Future':
        return flow_forward(p, tgt, refs[1:3], training=False)[0]
    if flownet == 'FlowNetC6':
        return flownetc6_forward(p, tgt, refs[2], training=False)
    raise ValueError('unknown flow net %r' % (flownet,))
