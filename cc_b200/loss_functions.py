"""Drop-in for the reference's ``loss_functions`` module (loss_functions.py), backed by libccb200.

Every name ``train.py:23-26`` imports exists here with the same signature.  The multi-scale
photometric / SSIM / smoothness / consensus losses each run as ONE fused sm_90a launch over all
pyramid levels (csrc/photo.cu, csrc/smooth_bce.cu) with hand-derived backward kernels, instead of
the reference's ~30 k ATen calls per step (SURVEY.md 3.1).

Differences a maintainer should know:
  * the reference's NaN ``assert(... .item() == 1)`` host syncs (loss_functions.py:60,105,115) are
    not replicated - nothing here synchronises the host;
  * pyramid levels must be exact 2^l reductions of the frame (true for every net in the reference).
"""
import torch
from torch import nn
from . import _lib, pyramid
from .inverse_warp import inverse_warp, flow_warp, pose2flow   # noqa: F401  (re-exported like the reference)
from .ssim import ssim, taps13                                  # noqa: F401

epsilon = 1e-8
_ROT = {'euler': _lib.ROT_EULER, 'quat': _lib.ROT_QUAT}
_PAD = {'zeros': _lib.PAD_ZEROS, 'border': _lib.PAD_BORDER}


def _set_levels(arr, tensors, name):
    for l, t in enumerate(tensors):
        arr[l] = _lib.ptr(t, '%s[%d]' % (name, l))


# =================================================================================================
# fused photometric losses
# =================================================================================================
class _PhotoLoss(torch.autograd.Function):
    """inputs after cfg:  rigid: pose, depth[L], (mask[L])     flow: flow[L*R] (level-major), (mask[L])"""

    @staticmethod
    def forward(ctx, cfg, *tensors):
        mode, L, R, B = cfg['mode'], cfg['L'], cfg['R'], cfg['B']
        sizes = cfg['sizes']
        dev = cfg['tgt'][0].device
        d = _lib.PhotoDesc()
        d.mode, d.B, d.R, d.H, d.W, d.nlevels = mode, B, R, cfg['H'], cfg['W'], L
        for l, (h, w) in enumerate(sizes):
            d.h[l], d.w[l] = h, w
        d.has_mask, d.has_occ = int(cfg['has_mask']), 1
        d.rotation_mode, d.padding_mode = cfg.get('rot', 0), cfg.get('pad', 0)
        d.wssim, d.qch, d.lambda_oob, d.wrig = cfg['wssim'], cfg['qch'], cfg['lambda_oob'], 0.0
        d.one_minus_wssim = 1 - cfg['wssim']
        for k, v in enumerate(taps13()):
            d.taps[k] = v
        keep = []
        _set_levels(d.tgt, cfg['tgt'], 'tgt')
        for l in range(L):
            for i in range(R):
                d.ref[l][i] = _lib.ptr(cfg['refs'][i][l], 'ref')
        ts = [_lib.f32(t) for t in tensors]
        keep += ts
        if mode == _lib.PHOTO_RIGID:
            pose, depth = ts[0], ts[1:1 + L]
            masks = ts[1 + L:1 + 2 * L] if cfg['has_mask'] else None
            K, Kinv = _lib.f32(cfg['K']), _lib.f32(cfg['Kinv'])
            keep += [K, Kinv]
            d.pose, d.K, d.Kinv = _lib.ptr(pose, 'pose'), _lib.ptr(K, 'K'), _lib.ptr(Kinv, 'Kinv')
            _set_levels(d.depth, depth, 'depth')
        else:
            flows = ts[:L * R]
            masks = ts[L * R:L * R + L] if cfg['has_mask'] else None
            for l in range(L):
                for i in range(R):
                    d.flow[l][i] = _lib.ptr(flows[l * R + i], 'flow')
        if masks is not None:
            _set_levels(d.mask, masks, 'mask')
        # saved-for-backward maps only where a backward will read them: none for a value-only call, no gmask when the
        # mask needs no gradient (the loss value is the same either way)
        save, mask_grad = cfg.get('save', True), cfg.get('mask_grad', cfg['has_mask'])
        use_ssim = cfg['wssim'] != 0
        dm = [torch.empty(B, R, 9, h, w, device=dev) for (h, w) in sizes] if (use_ssim and save) else []
        vo = [torch.empty(B, R, h, w, device=dev) for (h, w) in sizes] if save else []
        gm = [torch.empty(B, R, h, w, device=dev) for (h, w) in sizes] if (mask_grad and save) else []
        if dm:
            _set_levels(d.dmaps, dm, 'dmaps')
        _set_levels(d.vo, vo, 'vo')
        if gm:
            _set_levels(d.gmask, gm, 'gmask')
        scal = torch.empty(L * R * 4, device=dev)
        part, d.partials_floats = _lib.workspace('ccb_photo_partials_floats', d, like=scal)
        loss = torch.empty(1, device=dev)
        d.scal, d.partials, d.loss = _lib.ptr(scal), _lib.ptr(part), _lib.ptr(loss)
        _lib.call('ccb_photo_loss_fwd', d, loss)
        ctx.desc, ctx.cfg = d, cfg
        ctx.keep = keep + dm + vo + gm + [scal, loss] + list(cfg['tgt']) + [t for r in cfg['refs'] for t in r]
        ctx.n_in = len(tensors)
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        d, cfg = ctx.desc, ctx.cfg
        mode, L, R, B = cfg['mode'], cfg['L'], cfg['R'], cfg['B']
        sizes = cfg['sizes']
        dev = cfg['tgt'][0].device
        g = _lib.f32(g).reshape(1)
        d.grad_out = _lib.ptr(g, 'grad_out')
        grads = []
        if mode == _lib.PHOTO_RIGID:
            d_pose = torch.empty(B, R, 6, device=dev)
            d_depth = [torch.empty(B, 1, h, w, device=dev) for (h, w) in sizes]
            part, d.pose_partials_floats = _lib.workspace('ccb_photo_pose_partials_floats', d, like=d_pose)
            d.d_pose, d.pose_partials = _lib.ptr(d_pose), _lib.ptr(part)
            _set_levels(d.d_depth, d_depth, 'd_depth')
            grads = [d_pose] + d_depth
        else:
            d_flow = [torch.empty(B, 2, h, w, device=dev) for (h, w) in sizes for _ in range(R)]
            for l in range(L):
                for i in range(R):
                    d.d_flow[l][i] = _lib.ptr(d_flow[l * R + i])
            grads = d_flow
        if cfg['has_mask'] and cfg.get('mask_grad', True):
            d_mask = [torch.empty(B, R, h, w, device=dev) for (h, w) in sizes]
            _set_levels(d.d_mask, d_mask, 'd_mask')
            grads = grads + d_mask
        elif cfg['has_mask']:
            grads = grads + [None] * L
        _lib.call('ccb_photo_loss_bwd', d, g)
        return (None,) + tuple(grads)


def _photo_apply(cfg, args, masks):
    """_PhotoLoss on `args`, told whether autograd will call its backward (grad mode on and an input that requires a
    gradient) and whether the masks need a gradient (a fixed MaskNet's output does not)."""
    grad = torch.is_grad_enabled()
    cfg['save'] = grad and any(t.requires_grad for t in args)
    cfg['mask_grad'] = cfg['save'] and cfg['has_mask'] and any(m.requires_grad for m in masks)
    return _PhotoLoss.apply(cfg, *args)


def _level_sizes(preds):
    return [(int(p.size(2)), int(p.size(3))) for p in preds]


def photometric_reconstruction_loss(tgt_img, ref_imgs, intrinsics, intrinsics_inv, depth, explainability_mask, pose,
                                    rotation_mode='euler', padding_mode='zeros', lambda_oob=0, qch=0.5, wssim=0.5):
    """Multi-scale rigid photometric loss.  Reference loss_functions.py:80-128."""
    if type(explainability_mask) not in [tuple, list]:
        explainability_mask = [explainability_mask]
    if type(depth) not in [list, tuple]:
        depth = [depth]
    pairs = list(zip(depth, explainability_mask))       # zip truncation is reference behaviour (:119-125)
    depth = [p[0] for p in pairs]
    masks = [p[1] for p in pairs]
    assert(pose.size(1) == len(ref_imgs))
    for dd, m in pairs:
        assert(m is None or dd.size()[2:] == m.size()[2:])
    has_mask = masks[0] is not None
    if any((m is not None) != has_mask for m in masks):
        raise NotImplementedError('cc_b200: explainability masks must be given for all levels or for none')
    sizes = _level_sizes(depth)
    cfg = dict(mode=_lib.PHOTO_RIGID, L=len(depth), R=len(ref_imgs), B=int(tgt_img.size(0)),
               H=int(tgt_img.size(2)), W=int(tgt_img.size(3)), sizes=sizes, has_mask=has_mask,
               rot=_ROT[rotation_mode], pad=_PAD[padding_mode], wssim=float(wssim), qch=float(qch),
               lambda_oob=float(lambda_oob), K=intrinsics, Kinv=intrinsics_inv,
               tgt=pyramid.levels_for(tgt_img, sizes), refs=[pyramid.levels_for(r, sizes) for r in ref_imgs])
    args = [pose] + list(depth) + (list(masks) if has_mask else [])
    return _photo_apply(cfg, args, masks if has_mask else [])


def photometric_flow_loss(tgt_img, ref_imgs, flows, explainability_mask, lambda_oob=0, qch=0.5, wssim=0.5):
    """Multi-scale flow photometric loss; flows = [flow_bwd_levels, flow_fwd_levels].
    Reference loss_functions.py:27-77."""
    if type(flows[0]) not in [tuple, list]:
        if explainability_mask is not None:
            explainability_mask = [explainability_mask]
        flows = [[uv] for uv in flows]
    L, R = len(flows[0]), len(flows)
    assert(R == len(ref_imgs))
    masks = [explainability_mask[i] for i in range(L)]
    for i in range(L):
        assert(masks[i] is None or flows[0][i].size()[2:] == masks[i].size()[2:])
    has_mask = masks[0] is not None
    if any((m is not None) != has_mask for m in masks):
        raise NotImplementedError('cc_b200: explainability masks must be given for all levels or for none')
    sizes = _level_sizes(flows[0])
    cfg = dict(mode=_lib.PHOTO_FLOW, L=L, R=R, B=int(tgt_img.size(0)), H=int(tgt_img.size(2)), W=int(tgt_img.size(3)),
               sizes=sizes, has_mask=has_mask, wssim=float(wssim), qch=float(qch), lambda_oob=float(lambda_oob),
               tgt=pyramid.levels_for(tgt_img, sizes), refs=[pyramid.levels_for(r, sizes) for r in ref_imgs])
    args = [flows[i][l] for l in range(L) for i in range(R)] + (list(masks) if has_mask else [])
    return _photo_apply(cfg, args, masks if has_mask else [])


def consensus_exp_masks(cam_flows_fwd, cam_flows_bwd, flows_fwd, flows_bwd, tgt_img, ref_img_fwd, ref_img_bwd,
                        wssim, wrig, ws=0.1):
    """0/1 consensus targets per level, no gradient.  Reference loss_functions.py:160-202."""
    L = len(cam_flows_fwd)
    sizes = _level_sizes(cam_flows_fwd)
    B = int(tgt_img.size(0))
    dev = tgt_img.device
    d = _lib.PhotoDesc()
    d.mode, d.B, d.R, d.H, d.W, d.nlevels = _lib.PHOTO_CONSENSUS, B, 3, int(tgt_img.size(2)), int(tgt_img.size(3)), L
    for l, (h, w) in enumerate(sizes):
        d.h[l], d.w[l] = h, w
    d.wssim, d.qch, d.lambda_oob, d.wrig = float(wssim), 0.5, 0.0, float(wrig)
    d.one_minus_wssim = 1 - float(wssim)
    for k, v in enumerate(taps13()):
        d.taps[k] = v
    tgt = pyramid.levels_for(tgt_img, sizes)
    rf, rb = pyramid.levels_for(ref_img_fwd, sizes), pyramid.levels_for(ref_img_bwd, sizes)
    fl = [[_lib.f32(cam_flows_fwd[l]), _lib.f32(cam_flows_bwd[l]), _lib.f32(flows_fwd[l])] for l in range(L)]
    out = [torch.empty(B, 1, h, w, device=dev) for (h, w) in sizes]
    _set_levels(d.tgt, tgt, 'tgt')
    _set_levels(d.target, out, 'target')
    for l in range(L):
        for i, r in enumerate((rf[l], rb[l], rf[l])):
            d.ref[l][i] = _lib.ptr(r, 'ref')
            d.flow[l][i] = _lib.ptr(fl[l][i], 'flow')
    _lib.call('ccb_consensus_targets', d, tgt_img)
    return out


# =================================================================================================
# smoothness
# =================================================================================================
class _SmoothLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cfg, *preds):
        ps = [_lib.f32(p) for p in preds]
        L = len(ps)
        B, Cc = int(ps[0].size(0)), int(ps[0].size(1))
        dev = ps[0].device
        d = _lib.SmoothDesc()
        d.kind, d.B, d.C, d.nlevels = cfg['kind'], B, Cc, L
        for l, p in enumerate(ps):
            assert p.size(0) == B and p.size(1) == Cc
            d.h[l], d.w[l] = int(p.size(2)), int(p.size(3))
        _set_levels(d.pred, ps, 'pred')
        if cfg['kind'] == _lib.SMOOTH_EDGE:
            _set_levels(d.img, cfg['img'], 'img')
        part, d.partials_floats = _lib.workspace('ccb_smooth_partials_floats', d, like=ps[0])
        loss = torch.empty(1, device=dev)
        d.partials, d.loss = _lib.ptr(part), _lib.ptr(loss)
        _lib.call('ccb_smooth_fwd', d, loss)
        ctx.desc, ctx.keep = d, ps + list(cfg.get('img', []))
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        d = ctx.desc
        g = _lib.f32(g).reshape(1)
        ps = ctx.keep[:d.nlevels]
        dp = [torch.empty_like(p) for p in ps]
        d.grad_out = _lib.ptr(g)
        _set_levels(d.d_pred, dp, 'd_pred')
        _lib.call('ccb_smooth_bwd', d, g)
        return (None,) + tuple(dp)


def edge_aware_smoothness_loss(img, pred_disp):
    """Reference loss_functions.py:287-319."""
    if type(pred_disp) not in [tuple, list]:
        pred_disp = [pred_disp]
    cfg = dict(kind=_lib.SMOOTH_EDGE, img=pyramid.levels_for(img, _level_sizes(pred_disp)))
    return _SmoothLoss.apply(cfg, *pred_disp)


def smooth_loss(pred_disp):
    """Reference loss_functions.py:323-341."""
    if type(pred_disp) not in [tuple, list]:
        pred_disp = [pred_disp]
    return _SmoothLoss.apply(dict(kind=_lib.SMOOTH_SECOND), *pred_disp)


# =================================================================================================
# mask cross-entropies
# =================================================================================================
class _BceLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cfg, *masks):
        ms = [_lib.f32(m) for m in masks]
        L = len(ms)
        B, Cc = int(ms[0].size(0)), int(ms[0].size(1))
        dev = ms[0].device
        d = _lib.BceDesc()
        d.kind, d.B, d.C, d.nlevels = cfg['kind'], B, Cc, L
        d.thresh, d.wbce = cfg.get('thresh', 0.0), cfg.get('wbce', 0.0)
        for l, m in enumerate(ms):
            d.h[l], d.w[l] = int(m.size(2)), int(m.size(3))
        _set_levels(d.mask, ms, 'mask')
        keep = list(ms)
        if cfg['kind'] == _lib.BCE_CONSENSUS:
            for name in ('census_bwd', 'census_fwd', 'target_bwd', 'target_fwd'):
                ts = [_lib.f32(t) for t in cfg[name]]
                keep += ts
                _set_levels(getattr(d, name), ts, name)
        part, d.partials_floats = _lib.workspace('ccb_bce_partials_floats', d, like=ms[0])
        loss = torch.empty(1, device=dev)
        d.partials, d.loss = _lib.ptr(part), _lib.ptr(loss)
        _lib.call('ccb_bce_fwd', d, loss)
        ctx.desc, ctx.keep = d, keep
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        d = ctx.desc
        g = _lib.f32(g).reshape(1)
        ms = ctx.keep[:d.nlevels]
        dm = [torch.empty_like(m) for m in ms]
        d.grad_out = _lib.ptr(g)
        _set_levels(d.d_mask, dm, 'd_mask')
        _lib.call('ccb_bce_bwd', d, g)
        return (None,) + tuple(dm)


def explainability_loss(mask):
    """BCE(mask, 1) summed over levels.  Reference loss_functions.py:148-155."""
    if type(mask) not in [tuple, list]:
        mask = [mask]
    return _BceLoss.apply(dict(kind=_lib.BCE_ONES), *mask)


def consensus_depth_flow_mask(explainability_mask, census_mask_bwd, census_mask_fwd, exp_masks_bwd_target,
                              exp_masks_fwd_target, THRESH, wbce):
    """Reference loss_functions.py:221-250 (+ weighted_binary_cross_entropy :252-261)."""
    assert(len(explainability_mask) == len(census_mask_bwd))
    assert(len(explainability_mask) == len(census_mask_fwd))
    cfg = dict(kind=_lib.BCE_CONSENSUS, thresh=float(THRESH), wbce=float(wbce), census_bwd=census_mask_bwd,
               census_fwd=census_mask_fwd, target_bwd=exp_masks_bwd_target, target_fwd=exp_masks_fwd_target)
    return _BceLoss.apply(cfg, *explainability_mask)


# =================================================================================================
# small helpers the reference exports (host-side torch compositions; not on the fused path)
# =================================================================================================
def spatial_normalize(disp):
    """Reference loss_functions.py:13-16."""
    _mean = disp.mean(dim=1, keepdim=True).mean(dim=2, keepdim=True).mean(dim=3, keepdim=True)
    return disp / _mean


def robust_l1(x, q=0.5, eps=1e-2):
    """Reference loss_functions.py:18-21."""
    return torch.pow((x.pow(2) + eps), q).mean()


def robust_l1_per_pix(x, q=0.5, eps=1e-2):
    """Reference loss_functions.py:23-25."""
    return torch.pow((x.pow(2) + eps), q)


def occlusion_masks(flow_bw, flow_fw):
    """Reference loss_functions.py:343-352 (fused inside the photometric kernels; exported for parity)."""
    mag_sq = flow_fw.pow(2).sum(dim=1) + flow_bw.pow(2).sum(dim=1)
    flow_diff = flow_fw + flow_bw
    occ = flow_diff.sum(dim=1) > 0.08 * mag_sq + 1.0
    return occ.type_as(flow_bw), occ.type_as(flow_fw)


def depth_occlusion_masks(depth, pose, intrinsics, intrinsics_inv):
    """Reference loss_functions.py:132-137 (full-resolution intrinsics at every level, SURVEY F4)."""
    flow_cam = [pose2flow(depth.squeeze(), pose[:, i], intrinsics, intrinsics_inv) for i in range(pose.size(1))]
    masks1, masks2 = occlusion_masks(flow_cam[1], flow_cam[2])
    masks0, masks3 = occlusion_masks(flow_cam[0], flow_cam[3])
    return torch.stack((masks0, masks1, masks2, masks3), dim=1)


def gaussian_explainability_loss(mask):
    """Reference loss_functions.py:139-145."""
    if type(mask) not in [tuple, list]:
        mask = [mask]
    loss = 0
    for mask_scaled in mask:
        loss += torch.exp(-torch.mean((mask_scaled - 0.5).pow(2)) / 0.15)
    return loss


def logical_or(a, b):
    """Reference loss_functions.py:157-158."""
    return 1 - (1 - a) * (1 - b)


def compute_joint_mask_for_depth(explainability_mask, rigidity_mask_bwd, rigidity_mask_fwd, THRESH):
    """Reference loss_functions.py:204-219."""
    joint_masks = []
    for i in range(len(explainability_mask)):
        e = explainability_mask[i]
        rf = (rigidity_mask_fwd[i] > THRESH).type_as(e)
        rb = (rigidity_mask_bwd[i] > THRESH).type_as(e)
        ej = (1 - (1 - e[:, 1]) * (1 - e[:, 2]).unsqueeze(1) > 0.5).type_as(e)
        jf = logical_or(rf, ej).detach()
        jb = logical_or(rb, ej).detach()
        joint_masks.append(torch.cat((jb, jb, jf, jf), dim=1))
    return joint_masks


def weighted_binary_cross_entropy(output, target, weights=None):
    """Reference loss_functions.py:252-261."""
    if weights is not None:
        assert len(weights) == 2
        loss = weights[1] * (target * torch.log(output + epsilon)) + \
            weights[0] * ((1 - target) * torch.log(1 - output + epsilon))
    else:
        loss = target * torch.log(output + epsilon) + (1 - target) * torch.log(1 - output + epsilon)
    return torch.neg(torch.mean(loss))


# ---- validation metrics (reference loss_functions.py:355-467; SURVEY 8f "next" N2) -----------------
# Fused masked reductions (csrc/io_ops.cu): one pass over the ground-truth grid, deterministic two-stage sums,
# no intermediate up-sampled tensors.  Same names / arguments / python-float results as the reference, so
# validate_flow_with_gt / validate_depth_with_gt (train.py:588-777) call them unchanged.
def _flow_metrics(gt, pred_a, pred_b=None, mask=None, thresh=0.5, tau=(3, 0.05), want_map=False):
    gt, pred_a = _lib.f32(gt), _lib.f32(pred_a)
    B, nc, Hg, Wg = gt.shape
    hp, wp = int(pred_a.shape[2]), int(pred_a.shape[3])
    hm = wm = 0
    if mask is not None:
        pred_b, mask = _lib.f32(pred_b), _lib.f32(mask)
        assert pred_b.shape == pred_a.shape and mask.shape[1] == 1
        hm, wm = int(mask.shape[2]), int(mask.shape[3])
    work, nbytes = _lib.workspace('ccb_flow_metrics_workspace_bytes', B, Hg, Wg, like=gt)
    out = torch.empty(4, device=gt.device)
    emap = torch.empty(B, Hg, Wg, device=gt.device) if want_map else None
    _lib.call('ccb_flow_metrics', gt, pred_a, pred_b, mask, B, int(nc), int(Hg), int(Wg), hp, wp, hm, wm, float(thresh),
              float(tau[0]), float(tau[1]), emap, work, nbytes, out, gt)
    return out, emap


def flow_diff(gt, pred):
    """Per-pixel end-point error map.  Reference loss_functions.py:355-365."""
    return _flow_metrics(gt, pred, want_map=True)[1]


def compute_epe(gt, pred):
    """Average EPE (masked by gt[:,2] when present) as a python float.  Reference :368-387."""
    return _flow_metrics(gt, pred)[0][0].item()


def outlier_err(gt, pred, tau=[3, 0.05]):
    """KITTI Fl outlier ratio.  Reference :389-407."""
    assert gt.size(1) == 3
    return _flow_metrics(gt, pred, tau=tau)[0][3].item()


def compute_all_epes(gt, rigid_pred, non_rigid_pred, rigidity_mask, THRESH=0.5):
    """[all, rigid, non-rigid EPE, outliers] with the flows composited by the rigidity mask.  Reference :409-427."""
    out = _flow_metrics(gt, rigid_pred, non_rigid_pred, rigidity_mask, thresh=THRESH)[0]
    return out.tolist()


def compute_errors(gt, pred, crop=True):
    """Depth metrics [abs_diff, abs_rel, sq_rel, a1, a2, a3] with median scaling and the Garg crop.
    Reference :430-467 (returns 0-dim tensors like the reference; the per-sample medians are found by a
    radix select on the device)."""
    gt, pred = _lib.f32(gt), _lib.f32(pred)
    B, H, W = gt.shape
    work, nbytes = _lib.workspace('ccb_depth_errors_workspace_bytes', B, H, W, like=gt)
    out = torch.empty(6, device=gt.device)
    _lib.call('ccb_depth_errors', gt, pred, B, H, W, int(bool(crop)), work, nbytes, out, gt)
    return [out[i] for i in range(6)]
