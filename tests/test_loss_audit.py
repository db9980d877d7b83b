"""The loss audit's checker (tests/loss_audit.py), without a GPU.

The audit's own fp32 evaluation of the photometric formulas, and the fp32 oracle for the smoothness and BCE terms,
stand in for the kernels: given the same vo map they must pass every bound.  Each of ten typical kernel defects applied
to an otherwise correct result must be flagged on the output it corrupts, and the correct result must not be.  The
wrappers must restore everything on exit.  Then the audit runs on the CPU simulator build of the loss kernels: the cfg3
loss layer at b2 64x128 with 4 levels, and a sweep over the template paths the step never takes."""
import pytest
import torch
from tests import loss_audit as LA
from tests.util import sim_lib      # noqa: F401  (module fixture: the simulator library)
from cc_b200 import synth, _lib, loss_functions as CL, inverse_warp as CW, pyramid as CP
import torch.nn.functional as F
from oracle import losses as OL, geometry as OG, ssim as OSSIM

pytestmark = pytest.mark.usefixtures('sim_lib')

f32 = torch.float32


# ---- fp32 stand-ins and mutations ---------------------------------------------------------------------------------------
def _photo_call(mode, B=2, H=64, W=128, NL=4, seed=77, wssim=0.997, masks=True):
    s = synth.sample(B, H, W, seed=seed, nlevels=NL)
    sizes = [(H >> l, W >> l) for l in range(NL)]
    lv = lambda im: [torch.nn.functional.avg_pool2d(im, 1 << l) if l else im for l in range(NL)]     # noqa: E731
    R = 4 if mode == 'rigid' else 2
    refs = s['refs'] if mode == 'rigid' else s['refs'][1:3]
    cfg = dict(mode=_lib.PHOTO_RIGID if mode == 'rigid' else _lib.PHOTO_FLOW, L=NL, R=R, B=B, H=H, W=W, sizes=sizes,
               has_mask=masks, rot=_lib.ROT_EULER, pad=_lib.PAD_ZEROS, wssim=wssim, qch=0.5, lambda_oob=0.0,
               K=s['K'], Kinv=s['Kinv'], tgt=lv(s['tgt']), refs=[lv(r) for r in refs])
    if mode == 'rigid':
        tensors = [s['pose']] + s['depth'] + ([m for m in s['emask']] if masks else [])
    else:
        tensors = [f for l in range(NL) for f in (s['flow_bwd'][l], s['flow_fwd'][l])] + \
            ([1 - m[:, 1:3] for m in s['emask']] if masks else [])
    return LA.PhotoCall(cfg, tensors)


def _photo_standin(pc, mut=None, go=0.7):
    """fp32 evaluation of the kernels' formulas (optionally with a defect) -> the outputs a kernel call returns."""
    fwd, _ = LA.photo_forward(pc, f32, mut=mut)
    vo, dm, gm, scal = fwd['vo'], fwd['dmaps'], fwd['gmask'], fwd['scal']
    v, _ = LA.photo_backward(pc, fwd, go, vo, dm, scal, dt=f32, mut=mut)
    if pc.mode == 'rigid':
        grads = [v['d_pose']] + [c[0] for c in v['d_depth']]
    else:
        grads = [v['d_flow'][l][i][0] for l in range(pc.L) for i in range(pc.R)]
    grads = grads + (list(v['d_mask']) if pc.has_mask else [])
    return dict(vo=vo, dm=dm, gm=gm, scal=scal, loss=fwd['loss'], grads=grads, go=go)


def _photo_eval(pc, out):
    fc, st = LA.photo_fwd_checks(pc, out['vo'], out['dm'], out['gm'], out['scal'], out['loss'])
    bc, _ = LA.photo_bwd_checks(pc, st, torch.tensor(out['go']), out['vo'], out['dm'], out['scal'], out['grads'])
    fam = 'photo_' + pc.mode
    res, _, bad = LA.evaluate(fam, fc + bc)
    return res, bad


@pytest.fixture(scope='module')
def rigid():
    pc = _photo_call('rigid')
    return pc, _photo_eval(pc, _photo_standin(pc))


@pytest.fixture(scope='module')
def flow():
    pc = _photo_call('flow')
    return pc, _photo_eval(pc, _photo_standin(pc))


def _flagged(pc, mut, what):
    res, bad = _photo_eval(pc, _photo_standin(pc, mut))
    return {w: any(b.startswith(w + ' ') for b in bad) for w in what}, res


def test_photo_standins_pass(rigid, flow):
    for pc, (res, bad) in (rigid, flow):
        assert not bad, (pc.mode, bad)
        assert res['vo'][0] == 0


def _separable_ssim(img1, img2, window_size=13):
    """oracle.ssim with its 13x13 window applied as the kernels apply it: the fp32 1-D taps, a row pass then a column
    pass.  The oracle's 2-D window is the fp32 outer product of the same taps, whose roundings are a definition
    difference of up to ~u per tap, not a kernel error; everything else in the oracle stays as it is."""
    C = img1.size(1)
    g = OSSIM.gaussian(window_size, 1.5).to(img1)
    blur = lambda x: F.conv2d(F.conv2d(x, g.view(1, 1, 1, -1).expand(C, 1, 1, window_size).contiguous(), padding=(0, 6), groups=C),   # noqa: E731
                              g.view(1, 1, -1, 1).expand(C, 1, window_size, 1).contiguous(), padding=(6, 0), groups=C)
    mu1, mu2 = blur(img1), blur(img2)
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1, s2, s12 = blur(img1 * img1) - mu1_sq, blur(img2 * img2) - mu2_sq, blur(img1 * img2) - mu12
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    return ((2 * mu12 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2))


@pytest.mark.parametrize('mode', ['rigid', 'flow'])
def test_photo_oracle_standin_passes(mode, monkeypatch):
    """The independent fp32 oracle (oracle/losses.py: its own warp, pyramid, valid and occlusion masks, autograd
    backward) through the audit's checks.  Its vo map, built from the oracle's own masks, must agree with the audit's
    re-derivation of the kernel's gates (|Xn| <= 1, the (0, 3) / (1, 2) occlusion pairs with the unscaled cameras, the
    flow-mode validity); its loss, and its gradients of depth, pose, masks and flows, must pass every bound.  The
    oracle does not form dmaps, gmask or the scal rows, so the backward is checked from the fp64 ones."""
    monkeypatch.setattr(OL, 'ssim', _separable_ssim)
    B, H, W, NL, go = 2, 64, 128, 4, 0.7
    s = synth.sample(B, H, W, seed=77, nlevels=NL)
    pc = _photo_call(mode, B, H, W, NL)
    pool = lambda im, h, w: F.adaptive_avg_pool2d(im, (h, w))         # noqa: E731
    pc.tgt = [pool(s['tgt'], h, w) for h, w in pc.sizes]
    refs = s['refs'] if mode == 'rigid' else s['refs'][1:3]
    pc.refs = [[pool(r, h, w) for r in refs] for h, w in pc.sizes]
    vo = []
    if mode == 'rigid':
        depth = [t.clone().requires_grad_(True) for t in s['depth']]
        pose = s['pose'].clone().requires_grad_(True)
        em = [t.clone().requires_grad_(True) for t in s['emask']]
        loss = OL.photometric_reconstruction_loss(s['tgt'], s['refs'], s['K'], s['Kinv'], depth, em, pose, wssim=0.997)
        grads = list(torch.autograd.grad(loss * go, [pose] + depth + em))
        for l, (h, w) in enumerate(pc.sizes):
            ds = H / h
            K_s = torch.cat((s['K'][:, 0:2] / ds, s['K'][:, 2:]), 1)
            Kinv_s = torch.cat((s['Kinv'][:, :, 0:2] * ds, s['Kinv'][:, :, 2:]), 2)
            occ = OL.depth_occlusion_masks(s['depth'][l], s['pose'], s['K'], s['Kinv'])
            vo.append(torch.stack([(1 - (OG.inverse_warp(pc.refs[l][i], s['depth'][l][:, 0], s['pose'][:, i], K_s, Kinv_s) == 0)
                                    .prod(1).float()) * (1 - occ[:, i]) for i in range(4)], 1))
    else:
        ff = [t.clone().requires_grad_(True) for t in s['flow_fwd']]
        fb = [t.clone().requires_grad_(True) for t in s['flow_bwd']]
        fem = [(1 - m[:, 1:3]).clone().requires_grad_(True) for m in s['emask']]
        loss = OL.photometric_flow_loss(s['tgt'], refs, [fb, ff], fem, wssim=0.997)
        leaves = [f for l in range(NL) for f in (fb[l], ff[l])] + fem
        grads = list(torch.autograd.grad(loss * go, leaves))
        for l in range(NL):
            occ = OL.occlusion_masks(s['flow_bwd'][l], s['flow_fwd'][l])[0]
            vo.append(torch.stack([(1 - (OG.flow_warp(pc.refs[l][i], (s['flow_bwd'], s['flow_fwd'])[i][l]) == 0).prod(1).float())
                                   * (1 - occ) for i in range(2)], 1))
    fwd, b = LA.photo_forward(pc, torch.float64, vo_kernel=vo)
    fwd['b_gmask'] = b['gmask']
    fc = [('vo', torch.cat([v.flatten() for v in vo]), torch.cat([v.flatten() for v in fwd['vo']]),
           torch.full((sum(v.numel() for v in vo),), LA.TINY32, dtype=torch.float64), None),
          ('loss', loss.detach().reshape(()), fwd['loss'].reshape(()), torch.tensor(b['loss'], dtype=torch.float64), None)]
    bc, _ = LA.photo_bwd_checks(pc, fwd, torch.tensor(go), vo, fwd['dmaps'], fwd['scal'], grads)
    res, _, bad = LA.evaluate('photo_' + mode, fc + bc)
    assert not bad, (bad, res)
    assert fwd['ties']['vo'] <= LA.VO_TIE_FRAC * sum(v.numel() for v in vo)


def _dropped_tap(pc):
    t = list(pc.taps)
    t[0] = 0.0                       # the outer tap at distance 6, one side
    return t


@pytest.mark.parametrize('mut,what', [
    ('bwd_taps', ['d_depth']),
    ('fwd_taps', ['dmaps', 'loss']),
    ('halo_col', ['d_depth']),
    ('occ_swap', ['vo']),
    ('tile_pose', ['d_pose']),
    ('gmask_no_ssim', ['gmask', 'd_mask']),
    ('oob_level', ['scal', 'loss']),
])
def test_rigid_mutation_flagged(rigid, mut, what):
    pc, (res0, bad0) = rigid
    arg = dict(bwd_taps=_dropped_tap(pc), fwd_taps=_dropped_tap(pc), halo_col=64, occ_swap=True, tile_pose=(0, 1, 1),
               gmask_no_ssim=True, oob_level=1)[mut]
    flagged, res = _flagged(pc, {mut: arg}, what)
    assert all(flagged.values()), (mut, flagged, {w: res[w] for w in what})
    assert not any(b.startswith(w + ' ') for b in bad0 for w in what)


def test_flow_scale_flagged(flow):
    pc, (res0, bad0) = flow
    flagged, res = _flagged(pc, {'flow_scale_w': True}, ['d_flow'])
    assert flagged['d_flow'], res['d_flow']
    assert not bad0


def test_smooth_row_wrap_flagged():
    """The edge weight of the last column read across the row end: (y, w - 1) against (y + 1, 0)."""
    s = synth.sample(2, 64, 128, seed=77, nlevels=4)
    imgs = [torch.nn.functional.avg_pool2d(s['tgt'], 1 << l) if l else s['tgt'] for l in range(4)]
    preds = s['depth']
    loss = OL.edge_aware_smoothness_loss(s['tgt'], preds)
    ok = LA.smooth_checks(_lib.SMOOTH_EDGE, preds, imgs, loss)
    assert not LA.evaluate('smooth', ok)[2]
    p, im = preds[0], imgs[0]
    B, C, h, w = p.shape
    wrap = torch.exp(-(im[:, :, :-1, -1] - im[:, :, 1:, 0]).abs().mean(1))
    bad = loss + ((p[:, 0, :-1, -1] - p[:, 0, 1:, 0]).abs() * wrap).sum() / (B * C * h * (w - 1))
    res, _, fails = LA.evaluate('smooth', LA.smooth_checks(_lib.SMOOTH_EDGE, preds, imgs, bad))
    assert any(f.startswith('loss ') for f in fails), res
    # the backward: oracle autograd passes, second-order too
    for kind, fn in ((_lib.SMOOTH_EDGE, lambda q: OL.edge_aware_smoothness_loss(s['tgt'], q)), (_lib.SMOOTH_SECOND, OL.smooth_loss)):
        q = [t.clone().requires_grad_(True) for t in preds]
        ls = fn(q)
        g = torch.autograd.grad(ls * 0.3, q)
        res, _, fails = LA.evaluate('smooth', LA.smooth_checks(kind, preds, imgs, ls.detach()) +
                                       LA.smooth_checks(kind, preds, imgs, None, go=torch.tensor(0.3), grads=g))
        assert not fails, (kind, fails)


def test_bce_eps_dropped_flagged():
    s = synth.sample(2, 64, 128, seed=77, nlevels=3)
    masks = [m.clone() for m in s['emask']]
    masks[0][0, 1, 3, 5:9] = torch.tensor([1e-9, 3e-9, 0.0, 2e-8])          # masks near 0
    tg = [(torch.rand(2, 1, m.shape[2], m.shape[3], generator=torch.Generator().manual_seed(l)) > 0.5).float()
          for l, m in enumerate(masks)]
    cen = [torch.rand(2, 2, m.shape[2], m.shape[3], generator=torch.Generator().manual_seed(9 + l)) * 0.02 for l, m in enumerate(masks)]
    cfg = dict(kind=_lib.BCE_CONSENSUS, thresh=0.01, wbce=0.5, census_bwd=cen, census_fwd=cen, target_bwd=tg, target_fwd=tg)
    q = [m.clone().requires_grad_(True) for m in masks]
    loss = OL.consensus_depth_flow_mask(q, cen, cen, tg, tg, THRESH=0.01, wbce=0.5)
    g = torch.autograd.grad(loss * 0.3, q)
    res, _, fails = LA.evaluate('bce', LA.bce_checks(cfg, masks, loss=loss.detach()) +
                                   LA.bce_checks(cfg, masks, go=torch.tensor(0.3), grads=g))
    assert not fails, fails
    bad = [t.clone() for t in g]
    m0 = masks[0]
    n = m0.numel()
    # the same gradient without the epsilon of log(m + 1e-8) where the target is 1
    sel = (0, 1, 3, slice(5, 9))
    th = ((cen[0][:, 0:1] < 0.01) & (cen[0][:, 1:2] < 0.01)).float()
    tb = 1 - (1 - th) * (1 - tg[0])
    tgt4 = torch.cat([tb, tb, tb, tb], 1)
    mv = m0[sel]
    bad[0][sel] = -(0.3 / n) * (0.5 * tgt4[sel] / mv.clamp_min(1e-30) - 0.5 * (1 - tgt4[sel]) / (1 - mv))
    res, _, fails = LA.evaluate('bce', LA.bce_checks(cfg, masks, go=torch.tensor(0.3), grads=bad))
    assert any(f.startswith('d_mask ') for f in fails), res


def test_audit_restores_functions():
    """The wrappers are in place inside the context only, and are removed on exit - also when the body raises and when
    the audit itself raises because a call is over its bound."""
    def state():
        return ([(getattr(CL, c).__dict__['forward'], getattr(CL, c).__dict__['backward']) for c in ('_PhotoLoss', '_SmoothLoss', '_BceLoss')],
                CW._Pose2Flow.__dict__['forward'], CL.consensus_exp_masks, CP.levels_for)
    before = state()
    with pytest.raises(RuntimeError, match='body'):
        with LA.LossAudit(report=False):
            assert state() != before
            raise RuntimeError('body')
    assert state() == before
    saved = LA.R_OUT[('bce', 'loss')]
    try:
        LA.R_OUT[('bce', 'loss')] = -1.0                            # every BCE call now misses its bound
        m = [torch.rand(1, 4, 8, 8, generator=torch.Generator().manual_seed(3)).clamp(0.1, 0.9).requires_grad_(True)]
        with pytest.raises(AssertionError, match='loss-layer calls over their bound'):
            with LA.LossAudit(report=False):
                CL.explainability_loss(m).backward()
    finally:
        LA.R_OUT[('bce', 'loss')] = saved
    assert state() == before


# ---- the simulator build -----------------------------------------------------------------------------------------------
def _audited(tag, **kw):
    with LA.LossAudit(tag=tag) as audit:
        LA.cfg3_losses(torch.device('cpu'), **kw)
    return audit


def test_audit_simulator_cfg3():
    """Every call of the cfg3 loss layer at b2 64x128, 4 levels, audited forward and backward."""
    audit = _audited('sim_cfg3')
    n = {}
    for r in audit.rows:
        n[(r['op'], r['phase'])] = n.get((r['op'], r['phase']), 0) + 1
    assert n == {('photo_rigid', 'fwd'): 1, ('photo_rigid', 'bwd'): 1, ('photo_flow', 'fwd'): 1, ('photo_flow', 'bwd'): 1,
                 ('smooth', 'fwd'): 4, ('smooth', 'bwd'): 4, ('bce', 'fwd'): 2, ('bce', 'bwd'): 2, ('consensus', 'fwd'): 1,
                 ('pose2flow', 'fwd'): 8, ('pyramid', 'fwd'): n.get(('pyramid', 'fwd'), 0)}, n
    assert n[('pyramid', 'fwd')] >= 10


@pytest.mark.parametrize('opts', LA.SWEEP, ids=lambda o: '-'.join('%s=%s' % kv for kv in o.items()))
def test_audit_simulator_options(opts):
    """The template paths the step never takes: SSIM compiled out, the powf path, the oob term, border padding, quaternion
    poses, no masks, and an odd geometry with partial tiles in both directions at every level (21x34 at the coarsest)."""
    o = dict(opts)
    kw = {k: o.pop(k) for k in ('H', 'W', 'NL') if k in o}
    audit = _audited('sim_' + '_'.join(map(str, opts.values())), opts=o, **kw)
    fams = {r['op'] for r in audit.rows}
    assert {'photo_rigid', 'photo_flow'} <= fams
