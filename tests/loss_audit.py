"""Audit of the fused loss layer against fp64, element by element, on the inputs a real run hands it.

`LossAudit` is a context manager built like tests/layer_audit.LayerAudit.  While it is active it wraps the forward and
backward of cc_b200.loss_functions._PhotoLoss, _SmoothLoss and _BceLoss, the forward of inverse_warp._Pose2Flow, and the
module attributes loss_functions.consensus_exp_masks and pyramid.levels_for (the step reaches both through the module).
After each real call it recomputes the op in fp64 from that call's own fp32 inputs - the pyramid levels the kernel was
given, depth, pose, K, K^-1, flows, masks, grad_out and the fp32 SSIM taps (ssim.taps13(), applied separably, 13 + 13
taps, as the kernels apply them) - and checks every output element against the bound derived below.  The photometric
forward is also checked on the intermediates its backward consumes: vo = valid (1 - occ), the gamma dS maps `dmaps`,
`gmask`, the per-(level, ref) `scal` rows (omw oob / n, oob, sum valid, loss term) and the loss.  The backward takes
the kernel's own vo, dmaps and scal as its inputs, so a failure names the half that is wrong.  The audit is read-only
(fp64 copies only; tests/test_gpu_fullsize.py holds the audited step bit-identical to an unaudited one).  At exit it
prints one table per family and raises an AssertionError listing every call over its bound; with $CCB_PARITY_REPORT_DIR
set, the rows go to loss_audit_<tag>.json.  Families: photo_rigid, photo_flow, smooth, bce, consensus, pose2flow,
pyramid.

Error model (u = 2^-24; |.| elementwise; every bound gets TINY32)
-----------------------------------------------------------------
Discrete decisions.  The fp64 reference takes the kernel's decisions where rounding can decide them, and checks that
rounding is the only thing that did:
  * vo is compared with the fp64 valid * (1 - occ) first.  An element may differ only where the fp64 margin of the
    deciding comparison lies within its rounding band: the zeros-padding rewrite |Xn| > 1 (band e_Xn below), the
    flow-mode validity -1 < ix < w (band e_ix), the occlusion test s > 0.08 |f|^2 + 1 (band: sum over the four flow
    components of |1 - 0.16 f_k| e_f + 6u (|s| + 0.08 |f|^2 + 1)), and, in zeros padding, the Z clamp at 1e-3 (band: the bound e_Z on the unclamped Z).  The number of
    such ties is reported; every other element must match exactly.  The reference then uses the kernel's gate at the
    ties (it takes valid = occ-free = 1 where the kernel's vo is 1, else flips the gate whose margin is in the band).
    An image value of exactly 0 inside the frame would also clear `valid`; the frames never hold one.
  * Consensus targets: tests/kernel_cases.check_consensus_targets against the oracle's sides, with fp64 sides.
  * BCE census comparisons and the abs kinks of the smoothness terms are decided on the same fp32 values in both
    places (the first differences of fp32 inputs are exact; the second differences are formed in fp32 as the kernel
    forms them), so the signs match exactly; sign(0) = 0 as in torch.

Sample coordinates.  The projection chain of geom.cuh (project, then make_samp) is a fixed sequence of fp32 operations.
With r = K^-1 [x y 1] (two roundings of |K^-1| [|x| |y| 1]: e_r = 2u |K^-1| [|x| |y| 1]), c = d r (e_c = |d| e_r +
u |c|), [X Y Z] = P [c; 1] with P = K_s [R|t] formed in fp32 from sinf / cosf (12u of |K_s| |T|) and four roundings:
  e_X = |P| e_c + 16u (|K_s| |T|) [|c|; 1],   e_q = (e_X + |X / Z| e_Z) / Z + u |X / Z|   (q = X / Z)
  e_Xn = 2 e_q / (w - 1) + 3u (2 |q| / (w - 1) + 1),   e_ix = w / 2 e_Xn + 3u (|ix| + w / 2 (|Xn| + 1))
and for the flow coordinates (flow_coords) e_Xn = 4u (|x + u| / (w - 1) + 1).  A bilinear sample is continuous in the
coordinate but its derivatives jump where the coordinate crosses an integer (or a border clamp).  Where the fp64
coordinate lies within e_ix of one, either one-sided fp64 value is accepted: the per-pixel outputs (d_depth, d_flow)
are checked against the nearer of the four (x, y) one-sided combinations, and the pose gradient, which sums every
pixel of every level, adds sum |jump| over the tied pixels of its terms to its bound.  This is stronger than the layer
audit, which drops tie elements.

Elementwise steps.  Bilinear value: 8u sum w |corner| + e_ix |d/dix| + e_iy |d/diy|; its derivative d/dix: 4u of its
magnitude + e_iy |v11 - v10 - v01 + v00|.  rl1 = (x^2 + 0.01)^q: a rsqrtf (<= 2 ulp) or powf (q != 0.5, <= 4 ulp)
plus the argument's two roundings: 5u |rl1| (rsqrtf) / 8u |rl1| (powf); rl1_d: 6u / 12u of |rl1_d|.  Both take the
propagated error of their argument, |d rl1/dx| e_x.
SSIM (ssim_tile.cuh).  Each moment m_k (mu1, E[x^2], mu2, E[y^2], E[xy]) is a 13-tap row pass then a 13-tap column
pass of fp32 FMAs: 26u blur(|v|), plus u for a squared / product operand, plus blur(propagated warped-value error).
sigma^2 = E[x^2] - mu^2 cancels in flat regions, so the error of S is propagated to first order in fp64,
e_S = sum_k |dS/dm_k| e_k (+ 2u (|E| + |mu mu|) per subtraction and 10u |S| for the final products and the <= 2 ulp
reciprocal).  dmaps = gamma dS/dm_j: sum_k |d^2 S / dm_j dm_k| e_k + 10u of its terms.  The backward blur of the
kernel's own dmaps: 26u blur(|dmaps|).
The loss scalars add the root-sum-square of their terms' elementwise bounds to the chain term: the roundings of
different pixels have independent signs (the random-sign model of the layer audit); the reduction term stays worst case.
Chains.  d_flow, d_mask and d_depth are elementwise chains: each product / sum adds u of its magnitude and each input
error is carried by the partial derivative (project_bwd: g0 = gXn 2 / ((w - 1) Z), g2 = -(g0 X + g1 Y) / Z, d_depth =
sum_k g_k (P_k . r), summed over the refs).  d_mask = c_l gmask is checked against the fp64 gmask (so a wrong gmask
fails in both halves).
Reductions.  The rounding of a sum's own chain is bounded by the worst case u * (depth of its chain) * sum |t|.  Chain
depths: photometric partials PXT (5) per thread x 3 channels, block_sum 10 (two warp trees), photo_fwd_finalize
ceil(tiles / 32) per lane + 5; smoothness / BCE: C per thread, block_sum 10, finalize ceil(blocks / 256) + 10, the
levels.  For the smoothness and BCE values (non-negative terms, elementwise bounds summed linearly) and the scal rows
this makes the bound a proof: R = 1.  The photometric loss adds the root-sum-square of its terms' elementwise bounds
instead of their sum (the roundings of different pixels have independent signs): that is the random-sign model of the
layer audit, not a proof, and its R is measured.
The pose gradient sums ~h w terms of both signs per (b, ref) and level, so a worst-case bound would be loose by the
cancellation.  It uses the random-sign model throughout: u sqrt(K) ||t||_2 for the reduction (K = h w), and the
root-sum-square over the pixels of the per-pixel chain bounds and of the tie jumps; then pose_grad_from_dP (K_s^T and
the rotation derivative, formed in fp32: 12u of |J|^T |dP|, and the sum over levels).  Its R is measured.

R and detectability.  r = |kernel - fp64| / s is held to R_OUT per output.  One dropped pixel of a loss sum (K = 3 B h
w ~ 2.6e6 terms at 256x832) moves it by ~1 / K of itself: below u D R at D ~ 30, so a single pixel is not detected
there - said plainly.  A dropped 64x20 tile is 1280 pixels of a level-0 sum, ~5e-4 of it at 256x832, far above
u D R ~ 2e-6.  The pose gradient sums about 2.1e5 level-0 terms per (b, ref) at 256x832: one pixel is again below its
bound; for one dropped tile the audit reports the r d_pose would have had (tile_drop_r: a middle level-0 tile of sample
0 removed, the least r over the refs), which tests/fullsize_cases.loss_audit_step requires above R.  On the H100 it is
3.9 against R = 1.  At 64x128 test_loss_audit's test_rigid_mutation_flagged[tile_pose] drops one.
Every checked output must also meet rel_err <= 1e-4 (tests/util.rel_err), the bar of BASELINE.json, except the two
capped where DMAPS_REL_CAP and the pose2flow cap say, whose conditioning is explained there.  The share of vo elements
decided at a rounding tie must stay under VO_TIE_FRAC.

R values: the measured worst r per family is in R_MEASURED (H100) and R_MEASURED_SIM (CPU simulator build)."""
import json
import math
import os
import statistics
import torch
import torch.nn.functional as F
from cc_b200 import _lib, synth, loss_functions as CL, inverse_warp as CW, pyramid as CP
from cc_b200.inverse_warp import pose2flow
from cc_b200.train_step import HP
from cc_b200.ssim import taps13
from tests import layer_audit as LA

U, TINY32 = LA.U, LA.TINY32
f64 = torch.float64
f32 = LA.f32
NT_PXT, BLOCK_TREE, WARP_TREE, TW, TH = 5, 10, 5, 64, 20       # ssim_tile.cuh / ccb_common.cuh block_sum
PNT = 256                                                       # smooth_bce.cu
C1, C2 = f32(0.0001), f32(0.0009)

# r bound per checked output, R_OUT[(family, output)].  The bounds of the smoothness and BCE values and gradients, the
# scal rows, vo, the pyramid and pose2flow are worst-case (R = 1 is a proof).  The others rest on first-order
# propagation (dmaps, gmask, d_depth, d_flow, d_mask) or on the random-sign model (the photometric loss and d_pose); their
# R is set from the measured worst r (R_MEASURED) with a margin of about 3.
R_OUT = {('photo_rigid', 'vo'): 1.0, ('photo_rigid', 'dmaps'): 0.2, ('photo_rigid', 'gmask'): 0.2, ('photo_rigid', 'scal'): 1.0,
         ('photo_rigid', 'loss'): 0.1, ('photo_rigid', 'd_pose'): 1.0, ('photo_rigid', 'd_depth'): 0.1, ('photo_rigid', 'd_mask'): 0.5,
         ('photo_flow', 'vo'): 1.0, ('photo_flow', 'dmaps'): 0.3, ('photo_flow', 'gmask'): 0.5, ('photo_flow', 'scal'): 1.0,
         ('photo_flow', 'loss'): 0.1, ('photo_flow', 'd_flow'): 1.0, ('photo_flow', 'd_mask'): 0.5,
         ('smooth', 'loss'): 1.0, ('smooth', 'd_pred'): 1.0, ('bce', 'loss'): 1.0, ('bce', 'd_mask'): 1.0,
         ('pose2flow', 'flow'): 1.0, ('pyramid', 'level'): 1.0}
# Worst r per output: on an H100 80GB HBM3 (700 W power limit, 2026-10-15) over every loss-layer call of the second cfg3
# step at b4 256x832 (the step is bit-reproducible) and of test_gpu_parity's option sweep; on the CPU simulator build over
# test_loss_audit's runs.  At 256x832 one dropped level-0 tile scores d_pose r = 3.9 (R = 1).
R_MEASURED = {('photo_rigid', 'dmaps'): 0.054, ('photo_rigid', 'gmask'): 0.060, ('photo_rigid', 'scal'): 0.484,
              ('photo_rigid', 'loss'): 0.024, ('photo_rigid', 'd_pose'): 0.339, ('photo_rigid', 'd_depth'): 0.021,
              ('photo_rigid', 'd_mask'): 0.148, ('photo_flow', 'dmaps'): 0.092, ('photo_flow', 'gmask'): 0.137,
              ('photo_flow', 'scal'): 0.496, ('photo_flow', 'loss'): 0.023, ('photo_flow', 'd_flow'): 0.283,
              ('photo_flow', 'd_mask'): 0.136, ('smooth', 'loss'): 0.041, ('smooth', 'd_pred'): 0.279, ('bce', 'loss'): 0.066,
              ('bce', 'd_mask'): 0.456, ('pose2flow', 'flow'): 0.101, ('pyramid', 'level'): 0.961}
R_MEASURED_SIM = {('photo_rigid', 'dmaps'): 0.063, ('photo_rigid', 'gmask'): 0.060, ('photo_rigid', 'scal'): 0.452,
                  ('photo_rigid', 'loss'): 0.024, ('photo_rigid', 'd_pose'): 0.328, ('photo_rigid', 'd_depth'): 0.021,
                  ('photo_rigid', 'd_mask'): 0.131, ('photo_flow', 'dmaps'): 0.090, ('photo_flow', 'gmask'): 0.137,
                  ('photo_flow', 'scal'): 0.496, ('photo_flow', 'loss'): 0.033, ('photo_flow', 'd_flow'): 0.202,
                  ('photo_flow', 'd_mask'): 0.136, ('smooth', 'loss'): 0.041, ('smooth', 'd_pred'): 0.258, ('bce', 'loss'): 0.038,
                  ('bce', 'd_mask'): 0.456, ('pose2flow', 'flow'): 0.091, ('pyramid', 'level'): 0.904}
R = {fam: max(v for (f, _), v in R_OUT.items() if f == fam) for fam in {f for f, _ in R_OUT}}
R['consensus'] = 1.0
# The max-abs rel_err bar of 1e-4 is replaced by a cap where the output's conditioning puts fp32 above it; both outputs
# must still meet their per-element bound.  pose2flow's flow is a coordinate (up to w - 1 pixels) minus the pixel
# index: a few-pixel flow carries the rounding of the coordinate, about 8u (w - 1) pixels, so its cap is
# max(1e-4, 8u (w - 1) / max |flow|) (H100, 256x832: 2.2e-4 at w = 832).  dmaps = gamma dS / dm carry the
# sigma^2 = E[x^2] - mu^2 cancellation of flat regions; on frames at least 416 wide their cap is 3e-4 (H100, 256x832:
# 1.6e-4), below that the 1e-4 bar holds (CPU simulator, 64x128: 1.5e-5).
DMAPS_REL_CAP, DMAPS_CAP_MIN_W = 3e-4, 416
VO_TIE_FRAC = 1e-4          # vo may differ from fp64 at rounding ties on at most this share of its elements
FAMILIES = ('photo_rigid', 'photo_flow', 'smooth', 'bce', 'consensus', 'pose2flow', 'pyramid')


def _d(t):
    return t.detach().to(f64)


def _sum_depth(nblk, lanes=32):
    return -(-nblk // lanes)


def blur(x, taps):
    """Separable 13-tap window (zero padding): the row pass, then the column pass, in x's dtype."""
    sh = x.shape
    t = torch.tensor(taps, dtype=x.dtype, device=x.device)
    y = x.reshape(-1, 1, sh[-2], sh[-1])
    y = F.conv2d(y, t.view(1, 1, 1, 13), padding=(0, 6))
    y = F.conv2d(y, t.view(1, 1, 13, 1), padding=(6, 0))
    return y.view(sh)


# ---------------------------------------------------------------------------------------------------------------------
# Geometry (geom.cuh) in any dtype, with the fp64 error bounds of the fp32 chain.
def rot_mat(ang, rot):
    return (CW.euler2mat if rot == _lib.ROT_EULER else CW.quat2mat)(ang)


def cams(pose, K, Kinv, ds, rot):
    """pose [B, R, 6] -> (K_s^-1 [B, 3, 3], K_s [B, 3, 3], T [B, R, 3, 4], P [B, R, 3, 4]); ds = H / h."""
    B, Rr = pose.shape[:2]
    dt = pose.dtype
    K, Kinv = K.to(dt), Kinv.to(dt)
    Ks = torch.cat([K[:, :2] / ds, K[:, 2:]], 1) if ds != 1 else K
    Ki = torch.cat([Kinv[:, :, :2] * ds, Kinv[:, :, 2:]], 2) if ds != 1 else Kinv
    Rm = rot_mat(pose.reshape(B * Rr, 6)[:, 3:], rot).view(B, Rr, 3, 3)
    T = torch.cat([Rm, pose[..., :3].unsqueeze(-1)], -1)
    return Ki, Ks, T, Ks.unsqueeze(1) @ T


def _grid(B, h, w, dt, dev):
    ys = torch.arange(h, dtype=dt, device=dev).view(1, h, 1).expand(B, h, w)
    xs = torch.arange(w, dtype=dt, device=dev).view(1, 1, w).expand(B, h, w)
    return xs, ys


def _mv(M, v0, v1, v2, v3=None):
    """Per-sample 3-row matrix [B, 3, k] times per-pixel vectors -> three [B, h, w] rows."""
    out = []
    for k in range(3):
        s = M[:, k, 0].view(-1, 1, 1) * v0 + M[:, k, 1].view(-1, 1, 1) * v1 + M[:, k, 2].view(-1, 1, 1) * v2
        if v3 is not None:
            s = s + M[:, k, 3].view(-1, 1, 1) * v3
        out.append(s)
    return out


def project(Ki, P, dep, w, h, Pabs=None):
    """geom.cuh project (no rewrite) for one ref: dict of r, c, X, Y, Zr, Z, q, Xn, Yn; with Pabs (= |K_s| |T|, fp64)
    also the error bounds e_X, e_Y, e_Z, e_Xn, e_Yn."""
    B = dep.shape[0]
    xs, ys = _grid(B, h, w, dep.dtype, dep.device)
    one = torch.ones_like(xs)
    r = _mv(Ki, xs, ys, one)
    c = [rk * dep for rk in r]
    X, Y, Zr = _mv(P, c[0], c[1], c[2], one)
    Z = Zr.clamp_min(1e-3)
    qx, qy = X / Z, Y / Z
    p = dict(r=r, c=c, X=X, Y=Y, Zr=Zr, Z=Z, qx=qx, qy=qy, zcl=~(Zr >= 1e-3),
             Xn=2 * qx / (w - 1) - 1, Yn=2 * qy / (h - 1) - 1)
    if Pabs is not None:
        rabs = _mv(Ki.abs(), xs.abs(), ys.abs(), one)
        e_r = [2 * U * t for t in rabs]
        e_c = [dep.abs() * er + U * ck.abs() for er, ck in zip(e_r, c)]
        cabs = [ck.abs() for ck in c]
        mag = _mv(Pabs, cabs[0], cabs[1], cabs[2], one)
        prop = _mv(torch.cat([P.abs()[:, :, :3], torch.zeros_like(P[:, :, :1])], 2), e_c[0], e_c[1], e_c[2], one)
        e = [pp + 16 * U * m for pp, m in zip(prop, mag)]
        e_Z = torch.where(p['zcl'], torch.zeros_like(Z), e[2])
        for k, (ek, q, n1) in enumerate(((e[0], qx, w - 1), (e[1], qy, h - 1))):
            eq = (ek + q.abs() * e_Z) / Z + U * q.abs()
            p['e_Xn' if k == 0 else 'e_Yn'] = 2 * eq / n1 + 3 * U * (2 * q.abs() / n1 + 1)
        p.update(e_X=e[0], e_Y=e[1], e_Z=e_Z, e_Zr=e[2], e_r=e_r, e_c=e_c)
    return p


def flow_coords(fl, w, h):
    B = fl.shape[0]
    xs, ys = _grid(B, h, w, fl.dtype, fl.device)
    ax, ay = xs + fl[:, 0], ys + fl[:, 1]
    Xn, Yn = 2 * (ax / (w - 1) - 0.5), 2 * (ay / (h - 1) - 0.5)
    return Xn, Yn, 4 * U * (ax.abs() / (w - 1) + 1), 4 * U * (ay.abs() / (h - 1) + 1)


def to_pix(Xn, n, e_Xn=None):
    """make_samp: ix = (Xn + 1) n / 2 - 1/2 and its error bound."""
    i = (Xn + 1) * (0.5 * n) - 0.5
    if e_Xn is None:
        return i, None
    return i, 0.5 * n * e_Xn + 3 * U * (i.abs() + 0.5 * n * (Xn.abs() + 1))


def coords_to_flow(Xn, Yn, w, h):
    B = Xn.shape[0]
    xs, ys = _grid(B, h, w, Xn.dtype, Xn.device)
    return (w - 1) * (Xn * 0.5 + 0.5) - xs, (h - 1) * (Yn * 0.5 + 0.5) - ys


def occ_free(ubw, vbw, ufw, vfw, e=None):
    """1 - occ_mask (loss_functions.py:343-352) and, with e (bound on each flow component's error), the margin's band."""
    mag = (ufw * ufw + vfw * vfw) + (ubw * ubw + vbw * vbw)
    s = (ufw + ubw) + (vfw + vbw)
    th = 0.08 * mag + 1.0
    om = (~(s > th)).to(ubw.dtype)
    if e is None:
        return om, None
    band = sum((1 + 0.16 * t.abs()) * et for t, et in zip((ubw, vbw, ufw, vfw), e)) + \
        6 * U * ((ufw.abs() + ubw.abs() + vfw.abs() + vbw.abs()) + 0.08 * mag + 1)
    return om, (s - th).abs() <= band


class Axis:
    """One sample coordinate of make_samp: the cell and the d coordinate / d Xn factor, as the kernel takes them from
    the fp32 coordinate (side 0), or the one-sided choices left (-1) / right (+1) of the integer the fp64 coordinate
    ties with (only at tie elements)."""

    def __init__(self, i, e, n, border):
        self.i, self.n, self.border = i, n, border
        k = i.round()
        lo, hi = (0, n - 1) if border else (-1, n)
        self.k = k
        self.tie = ((i - k).abs() <= e) & (k >= lo) & (k <= hi) if e is not None else torch.zeros_like(i, dtype=torch.bool)

    def take(self, side):
        i, n = self.i, self.n
        if self.border:
            g = torch.where((i >= 0) & (i <= n - 1), 0.5 * n, 0.0).to(i.dtype)
            ic = i.clamp(0, n - 1)
        else:
            g = torch.full_like(i, 0.5 * n)
            ic = i.clamp(-4, n + 4)
        x0 = ic.floor()
        if side:
            k = self.k
            x0 = torch.where(self.tie, k - 1 if side < 0 else k, x0)
            if self.border:
                inside = ((k >= 1) & (k <= n - 1)) if side < 0 else ((k >= 0) & (k <= n - 2))
                g = torch.where(self.tie, torch.where(inside, 0.5 * n, 0.0).to(i.dtype), g)
        return x0, ic - x0, g


def bilinear(img, x0, wx1, y0, wy1):
    """img [B, C, h, w]; cell (x0, y0) with weights -> value, d/dix, d/diy, the cross term and sum w |corner|."""
    B, C, h, w = img.shape
    x0, y0 = x0.long(), y0.long()
    flat = img.reshape(B, C, h * w)
    cs = []
    for dy in (0, 1):
        for dx in (0, 1):
            xx, yy = x0 + dx, y0 + dy
            ok = (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
            idx = torch.where(ok, yy * w + xx, 0).view(B, 1, -1).expand(B, C, -1)
            cs.append(torch.gather(flat, 2, idx).view(B, C, *x0.shape[1:]) * ok.unsqueeze(1))
    wx1, wy1 = wx1.unsqueeze(1), wy1.unsqueeze(1)
    wx0, wy0 = 1 - wx1, 1 - wy1
    v = cs[0] * (wy0 * wx0) + cs[1] * (wy0 * wx1) + cs[2] * (wy1 * wx0) + cs[3] * (wy1 * wx1)
    ddx = (cs[1] - cs[0]) * wy0 + (cs[3] - cs[2]) * wy1
    ddy = (cs[2] - cs[0]) * wx0 + (cs[3] - cs[1]) * wx1
    cross = (cs[3] - cs[2] - cs[1] + cs[0]).abs()
    mag = cs[0].abs() * (wy0 * wx0).abs() + cs[1].abs() * (wy0 * wx1).abs() + cs[2].abs() * (wy1 * wx0).abs() + \
        cs[3].abs() * (wy1 * wx1).abs()
    dmag = ((cs[1].abs() + cs[0].abs()) * wy0.abs() + (cs[3].abs() + cs[2].abs()) * wy1.abs())
    dmagy = ((cs[2].abs() + cs[0].abs()) * wx0.abs() + (cs[3].abs() + cs[1].abs()) * wx1.abs())
    return v, ddx, ddy, cross, mag, dmag, dmagy


def rl1(x, q):
    a = x * x + 0.01
    return a.sqrt() if q == 0.5 else a.pow(q)


def rl1_d(x, q):
    a = x * x + 0.01
    return x / a.sqrt() if q == 0.5 else 2 * q * x * a.pow(q - 1)


def rl1_dd(x, q):
    """|d rl1_d / dx|"""
    a = x * x + 0.01
    return (0.01 / a.pow(1.5)) if q == 0.5 else (2 * q * a.pow(q - 1) * (1 + 2 * (q - 1) * x * x / a)).abs()


def ssim_fn(mu1, exx, mu2, eyy, exy):
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    A1, A2 = 2 * mu12 + C1, 2 * (exy - mu12) + C2
    B1, B2 = mu1_sq + mu2_sq + C1, (exx - mu1_sq) + (eyy - mu2_sq) + C2
    return (A1 * A2) / (B1 * B2)


# ---------------------------------------------------------------------------------------------------------------------
# The photometric loss (photo.cu).
class PhotoCall:
    """Everything one _PhotoLoss call computes from: fp32 tensors as the kernel got them plus the kernel arguments."""

    def __init__(self, cfg, tensors):
        self.mode = 'rigid' if cfg['mode'] == _lib.PHOTO_RIGID else 'flow'
        self.L, self.R, self.B, self.H, self.W = cfg['L'], cfg['R'], cfg['B'], cfg['H'], cfg['W']
        self.sizes = list(cfg['sizes'])
        self.has_mask = bool(cfg['has_mask'])
        self.rot, self.border = cfg.get('rot', 0), cfg.get('pad', 0) == _lib.PAD_BORDER
        self.wssim, self.qch, self.lam = f32(cfg['wssim']), f32(cfg['qch']), f32(cfg['lambda_oob'])
        self.omw = f32(1 - cfg['wssim'])
        self.ssim = cfg['wssim'] != 0
        self.taps = list(taps13())
        self.tgt = [t.detach() for t in cfg['tgt']]
        self.refs = [[cfg['refs'][i][l].detach() for i in range(self.R)] for l in range(self.L)]
        ts = [t.detach().float() for t in tensors]
        L, Rr = self.L, self.R
        if self.mode == 'rigid':
            self.pose, self.depth = ts[0], ts[1:1 + L]
            self.masks = ts[1 + L:1 + 2 * L] if self.has_mask else None
            self.K, self.Kinv = cfg['K'].detach().float(), cfg['Kinv'].detach().float()
        else:
            self.flows = [[ts[l * Rr + i] for i in range(Rr)] for l in range(L)]
            self.masks = ts[L * Rr:L * Rr + L] if self.has_mask else None

    def tiles(self, l):
        h, w = self.sizes[l]
        return -(-w // TW) * -(-h // TH)


def _coords(pc, l, i, dt, bounds, occ_cams=False, cache=None):
    """Sample coordinates of ref i at level l: (Xn, Yn, e_Xn, e_Yn, proj or None); the rigid ones with the level-scaled
    camera (occ_cams: the unscaled one of the occlusion masks)."""
    h, w = pc.sizes[l]
    if pc.mode == 'flow':
        fl = pc.flows[l][i].to(dt)
        Xn, Yn, ex, ey = flow_coords(fl, w, h)
        return Xn, Yn, (ex if bounds else None), (ey if bounds else None), None
    ds = 1.0 if occ_cams else f32(pc.H) / f32(h)
    key = (l, ds, dt)
    if cache is not None and key in cache:
        Ki, Ks, T, P = cache[key]
    else:
        Ki, Ks, T, P = cams(pc.pose.to(dt), pc.K, pc.Kinv, ds, pc.rot)
        if cache is not None:
            cache[key] = (Ki, Ks, T, P)
    Pabs = (Ks.abs().unsqueeze(1) @ T.abs())[:, i] if bounds else None
    p = project(Ki, P[:, i], pc.depth[l][:, 0].to(dt), w, h, Pabs)
    p['i'] = i
    return p['Xn'], p['Yn'], p.get('e_Xn'), p.get('e_Yn'), p


def photo_forward(pc, dt=f64, vo_kernel=None, mut=None):
    """The forward of photo.cu in dtype dt.  With dt = fp64 and the kernel's vo map, also the bounds, the gates the
    kernel took and the tie counts.  mut: deliberate defects for the audit's own tests (fwd_taps, occ_swap, oob_level,
    gmask_no_ssim)."""
    mut = mut or {}
    bounds = dt == f64
    L, Rr, B = pc.L, pc.R, pc.B
    taps = mut.get('fwd_taps', pc.taps)
    dev = pc.tgt[0].device
    out = dict(vo=[], dmaps=[], gmask=[], scal=torch.zeros(L, Rr, 4, dtype=dt, device=dev), state=[], ties=dict(vo=0, coord=0))
    b_out = dict(vo=[], dmaps=[], gmask=[], scal=torch.zeros(L, Rr, 4, dtype=f64))
    vo_bad = []
    cache = {}
    Lsum, Lsum_e = 0.0, 0.0
    for l in range(L):
        h, w = pc.sizes[l]
        npx = B * h * w
        tg = pc.tgt[l].to(dt)
        # ---- occlusion (1 - occ) per ref, with its band
        if pc.mode == 'rigid':
            fl, efl = [], []
            for k in range(Rr):
                Xn, Yn, ex, ey, p = _coords(pc, l, k, dt, bounds, occ_cams=True, cache=cache)
                u_, v_ = coords_to_flow(Xn, Yn, w, h)
                fl.append((u_, v_))
                if bounds:
                    xs, ys = _grid(B, h, w, f64, dev)
                    efl.append(((w - 1) / 2 * ex + 3 * U * (u_.abs() + xs + (w - 1)),
                                (h - 1) / 2 * ey + 3 * U * (v_.abs() + ys + (h - 1))))
            pairs = [(0, Rr - 1), (1, Rr - 2)]
            if mut.get('occ_swap'):
                pairs = [(1, Rr - 2), (0, Rr - 1)]
            oms = []
            for a, b2 in pairs:
                oms.append(occ_free(fl[a][0], fl[a][1], fl[b2][0], fl[b2][1],
                                    (efl[a][0], efl[a][1], efl[b2][0], efl[b2][1]) if bounds else None))
            om_of = [oms[0] if (i == 0 or i == Rr - 1) else oms[1] for i in range(Rr)]
        else:
            fb, ff = pc.flows[l][0].to(dt), pc.flows[l][1].to(dt)
            o = occ_free(fb[:, 0], fb[:, 1], ff[:, 0], ff[:, 1], (0, 0, 0, 0) if bounds else None)
            om_of = [o] * Rr
        vo_l, dm_l, gm_l, st_l = [], [], [], []
        bvo, bdm, bgm = [], [], []
        for i in range(Rr):
            ref = pc.refs[l][i].to(dt)
            Xn, Yn, ex, ey, p = _coords(pc, l, i, dt, bounds, cache=cache)
            ix, e_ix = to_pix(Xn, w, ex)
            iy, e_iy = to_pix(Yn, h, ey)
            om, om_tie = om_of[i]
            # ---- valid: the rewrite |Xn| > 1 (rigid, zeros padding) or a corner inside the frame (flow)
            if pc.mode == 'rigid':
                if pc.border:
                    valid = torch.ones_like(Xn)
                    v_tie = torch.zeros_like(Xn, dtype=torch.bool)
                else:
                    valid = ((Xn.abs() <= 1) & (Yn.abs() <= 1)).to(dt)
                    v_tie = (((Xn.abs() - 1).abs() <= ex) | ((Yn.abs() - 1).abs() <= ey) |
                             ((p['Zr'] - 1e-3).abs() <= p['e_Zr'])) if bounds else None
            else:
                valid = ((ix > -1) & (ix < w) & (iy > -1) & (iy < h)).to(dt)
                v_tie = (((ix + 1).abs() <= e_ix) | ((ix - w).abs() <= e_ix) | ((iy + 1).abs() <= e_iy) |
                         ((iy - h).abs() <= e_iy)) if bounds else None
            vo64 = valid * om
            if vo_kernel is not None:
                vk = vo_kernel[l][:, i].to(dt)
                mis = vk != vo64
                tie = v_tie | (om_tie if om_tie is not None else torch.zeros_like(v_tie))
                vo_bad.append(int((mis & ~tie).sum()))
                out['ties']['vo'] += int(mis.sum())
                up, down = mis & tie & (vk == 1), mis & tie & (vk == 0)
                one, zero = torch.ones_like(valid), torch.zeros_like(valid)
                valid = torch.where(up, one, torch.where(down & v_tie, zero, valid))
                om = torch.where(up, one, torch.where(down & ~v_tie, zero, om))
            if pc.mode == 'rigid' and not pc.border:
                rew = valid == 0
                ix = torch.where(rew, torch.full_like(ix, 1.5 * w - 0.5), ix)
                iy = torch.where(rew, torch.full_like(iy, 1.5 * h - 0.5), iy)
            ax_, ay_ = Axis(ix, e_ix, w, pc.border), Axis(iy, e_iy, h, pc.border)
            x0, wx1, gmx = ax_.take(0)
            y0, wy1, gmy = ay_.take(0)
            wv, ddx, ddy, cross, vmag, dmag, dmagy = bilinear(ref, x0, wx1, y0, wy1)
            mk = pc.masks[l][:, i].to(dt) if pc.has_mask else torch.ones_like(valid)
            M = (valid * om).unsqueeze(1)
            e = (tg - wv) * M
            df = e * mk.unsqueeze(1)
            r1 = rl1(df, pc.qch)
            if pc.ssim:
                xv, yv = tg, wv
                mom = [blur(xv, taps), blur(xv * xv, taps), blur(yv, taps), blur(yv * yv, taps), blur(xv * yv, taps)]
                if bounds:
                    mom = [m.detach().requires_grad_(True) for m in mom]
                    with torch.enable_grad():
                        S = ssim_fn(*mom)
                        dS = torch.autograd.grad(S.sum(), mom, create_graph=True)
                    S = S.detach()
                else:
                    S = ssim_fn(*mom)
                    dS = None
                gam = -(valid * om * mk).unsqueeze(1)
                if dS is not None:
                    dmaps = torch.stack([gam * dS[2].detach(), gam * dS[3].detach(), gam * dS[4].detach()], 2)
                else:
                    mu1, exx, mu2, eyy, exy = mom
                    A1, A2 = 2 * mu1 * mu2 + C1, 2 * (exy - mu1 * mu2) + C2
                    B1, B2 = mu1 * mu1 + mu2 * mu2 + C1, (exx - mu1 * mu1) + (eyy - mu2 * mu2) + C2
                    inv = 1 / (B1 * B2)
                    dmaps = torch.stack([gam * (2 * mu1 * (A2 - A1) * inv - S * 2 * mu2 * (B2 - B1) * inv),
                                         gam * (-S / B2), gam * (2 * A1 * inv)], 2)
            else:
                S = torch.zeros_like(wv)
            sl = (1 - S * valid.unsqueeze(1)) * om.unsqueeze(1)
            gm = (rl1_d(df, pc.qch) * e + (0 if mut.get('gmask_no_ssim') else pc.wssim) * sl).sum(1)
            vo_l.append(valid * om)
            gm_l.append(gm)
            if pc.ssim:
                dm_l.append(dmaps.reshape(B, 9, h, w))
            v0, v1 = r1.sum(), (sl * mk.unsqueeze(1)).sum()
            v2, v3 = valid.sum(), rl1(1 - valid, pc.qch).sum()
            st = dict(valid=valid, om=om, ix=ix, iy=iy, e_ix=e_ix, e_iy=e_iy, proj=p, sl=sl)
            # ---- bounds
            if bounds:
                e_wv = 8 * U * vmag + e_ix.unsqueeze(1) * ddx.abs() + e_iy.unsqueeze(1) * ddy.abs() + \
                    (e_ix * e_iy).unsqueeze(1) * cross
                st.update(e_wv=e_wv, wv=wv)
                out['ties']['coord'] += int((ax_.tie | ay_.tie).sum())
                mkc = mk.unsqueeze(1)
                e_df = e_wv * M * mkc
                c_rl, c_rd = (5, 6) if pc.qch == 0.5 else (8, 12)
                e_r1 = c_rl * U * r1 + (df / (df * df + 0.01).sqrt()).abs() * e_df if pc.qch == 0.5 else \
                    c_rl * U * r1 + (2 * pc.qch * df * (df * df + 0.01).pow(pc.qch - 1)).abs() * e_df
                e_S = torch.zeros_like(wv)
                if pc.ssim:
                    av, aw, ex_ = tg.abs(), wv.abs(), e_wv
                    m = [t.detach() for t in mom]
                    em = [26 * U * blur(av, taps), 27 * U * blur(av * av, taps),
                          26 * U * blur(aw, taps) + blur(ex_, taps),
                          27 * U * blur(aw * aw, taps) + blur(2 * aw * ex_, taps),
                          27 * U * blur(av * aw, taps) + blur(av * ex_, taps)]
                    em[1] = em[1] + 2 * U * (m[1].abs() + m[0] * m[0])
                    em[3] = em[3] + 2 * U * (m[3].abs() + m[2] * m[2])
                    em[4] = em[4] + 2 * U * (m[4].abs() + (m[0] * m[2]).abs())
                    e_S = sum(g.detach().abs() * ek for g, ek in zip(dS, em)) + 10 * U * S.abs()
                    bd = []
                    for j in (2, 3, 4):
                        with torch.enable_grad():
                            H2 = torch.autograd.grad(dS[j].sum(), mom, retain_graph=True, allow_unused=True)
                        hb = sum((hk.abs() * ek) if hk is not None else 0 for hk, ek in zip(H2, em))
                        bd.append(gam.abs() * (hb + 10 * U * _dS_mag(m, S, j)))
                    bdm.append(torch.stack(bd, 2).reshape(B, 9, h, w) + TINY32)
                    del dS
                st['e_S'] = e_S
                vom = (valid * om).unsqueeze(1)
                rd = rl1_d(df, pc.qch)
                e_rd = c_rd * U * rd.abs() + rl1_dd(df, pc.qch) * e_df
                e_gm = (e_rd * e.abs() + rd.abs() * e_wv * M + pc.wssim * vom * e_S).sum(1) + \
                    4 * U * (rd.abs() * e.abs() + pc.wssim * sl.abs()).sum(1)
                st['e_gm'] = e_gm
                bgm.append(e_gm + TINY32)
                nblk = pc.tiles(l) * B
                D = 3 * NT_PXT + BLOCK_TREE + _sum_depth(nblk) + WARP_TREE
                ev0 = D * U * r1.sum() + _rss(e_r1)
                ev1 = (D + 2) * U * (sl * mkc).abs().sum() + _rss(e_S * vom * mkc)
                ev3 = D * U * rl1(1 - valid, pc.qch).sum() + 5 * U * rl1(1 - valid, pc.qch).sum()
                st['ev'] = (ev0, ev1, ev3)
            st_l.append(st)
            # ---- scal row
            n = 3.0 * npx
            lv = l
            if mut.get('oob_level') is not None and l == mut['oob_level']:
                lv = l - 1
            v2o = v2 if lv == l else out['state'][lv][i]['v2']
            st['v2'] = v2
            oob = npx / v2o if lv == l else (B * pc.sizes[lv][0] * pc.sizes[lv][1]) / v2o
            Lli = pc.omw * oob * (v0 / n + pc.wssim * (v1 / n)) + pc.lam * (v3 / npx)
            out['scal'][l, i] = torch.stack([pc.omw * oob / n, oob, v2, Lli])
            Lsum = Lsum + Lli
            if bounds:
                ev0, ev1, ev3 = st['ev']
                a0 = abs(pc.omw * float(oob) / n)
                eL = a0 * (float(ev0) + pc.wssim * float(ev1)) + pc.lam * float(ev3) / npx + \
                    6 * U * (a0 * (float(v0) + pc.wssim * abs(float(v1))) + pc.lam * float(v3) / npx)
                b_out['scal'][l, i] = torch.tensor([4 * U * pc.omw * float(oob) / n, 2 * U * float(oob), 0.0, eL]) + TINY32
                Lsum_e = Lsum_e + eL + abs(float(Lli)) * U * (L * Rr)
        out['vo'].append(torch.stack(vo_l, 1))
        out['gmask'].append(torch.stack(gm_l, 1) if pc.has_mask else None)
        out['dmaps'].append(torch.stack(dm_l, 1) if pc.ssim else None)
        out['state'].append(st_l)
        if bounds:
            b_out['gmask'].append(torch.stack(bgm, 1) if pc.has_mask else None)
            b_out['dmaps'].append(torch.stack(bdm, 1) if pc.ssim else None)
    out['loss'] = Lsum
    out['vo_bad'] = vo_bad
    if bounds:
        b_out['loss'] = Lsum_e + TINY32
    return out, (b_out if bounds else None)


def _rss(e):
    """Root-sum-square of per-element error bounds: the elementwise roundings of different pixels have independent
    signs, so their sum grows like the 2-norm (the reduction's own rounding keeps its worst-case term)."""
    return (e * e).sum().sqrt()


def _rss2(t):
    """Root-sum-square over the pixels of a [B, h, w] map -> [B]."""
    return (t * t).sum((1, 2)).sqrt()


def _dS_mag(m, S, j):
    """Magnitude of the terms ssim_point forms for dS / dm_j (its rounding scale)."""
    mu1, exx, mu2, eyy, exy = m
    A1, A2 = 2 * mu1 * mu2 + C1, 2 * (exy - mu1 * mu2) + C2
    B1, B2 = mu1 * mu1 + mu2 * mu2 + C1, (exx - mu1 * mu1) + (eyy - mu2 * mu2) + C2
    inv = 1 / (B1 * B2)
    if j == 2:
        return (2 * mu1 * inv).abs() * (A2.abs() + A1.abs()) + (S * 2 * mu2 * inv).abs() * (B2.abs() + B1.abs())
    if j == 3:
        return (S / B2).abs()
    return (2 * A1 * inv).abs()


def pose_jac(pc, l, dt=f64):
    """P(pose) of level l and the Jacobian |dP / dpose| [B, R, 12, 6]."""
    h, w = pc.sizes[l]
    ds = f32(pc.H) / f32(h)
    pose = pc.pose.to(dt)

    def fn(p):
        return cams(p, pc.K, pc.Kinv, ds, pc.rot)[3]
    J = torch.autograd.functional.jacobian(fn, pose)            # [B, R, 3, 4, B, R, 6]
    B, Rr = pose.shape[:2]
    J = J.reshape(B, Rr, 12, B, Rr, 6)
    idx_b = torch.arange(B)
    idx_r = torch.arange(Rr)
    return J[idx_b[:, None], idx_r[None, :], :, idx_b[:, None], idx_r[None, :], :]      # [B, R, 12, 6]


def photo_backward(pc, fwd, go, vo_k, dmaps_k, scal_k, dt=f64, mut=None):
    """The backward of photo.cu in dtype dt from the kernel's own vo, dmaps and scal (fwd: photo_forward's state of the
    same call).  Returns (values, bounds): values d_depth [L] + d_pose, or d_flow [L][R]; d_mask [L] (from fwd's
    gmask).  Bounds only for fp64; with them, the per-pixel outputs carry the four one-sided (x, y) combinations, of
    which the checks take the nearest at each element (`nearest`).  mut: bwd_taps, halo_col, tile_pose, flow_scale_w."""
    mut = mut or {}
    bounds = dt == f64
    L, Rr, B = pc.L, pc.R, pc.B
    taps = mut.get('bwd_taps', pc.taps)
    go = float(go)
    vals = dict(d_depth=[], d_flow=[], d_mask=[], variants=[])
    bnds = dict(d_depth=[], d_flow=[], d_mask=[])
    dev = pc.tgt[0].device
    dP_tot = torch.zeros(B, Rr, 6, dtype=dt, device=dev)
    e_pose = torch.zeros(B, Rr, 6, dtype=f64, device=dev)
    ties = 0
    for l in range(L):
        h, w = pc.sizes[l]
        tg = pc.tgt[l].to(dt)
        gd = []
        dflow_l, dflow_b = [], []
        dPl = torch.zeros(B, Rr, 12, dtype=dt, device=dev)
        e_dPl = torch.zeros(B, Rr, 12, dtype=f64, device=dev)
        if l == 0:
            tile_dP = torch.zeros(Rr, 12, dtype=dt, device=dev)
        dmask_l, dmask_b = [], []
        for i in range(Rr):
            st = fwd['state'][l][i]
            c_l = go * float(scal_k[l, i, 0])
            c_s = c_l * pc.wssim
            M = vo_k[l][:, i].to(dt).unsqueeze(1)
            mk = pc.masks[l][:, i].to(dt).unsqueeze(1) if pc.has_mask else torch.ones_like(M)
            M = M * mk
            if pc.ssim:
                dm = dmaps_k[l][:, i].to(dt).reshape(B, 3, 3, h, w)
                bl = blur(dm, taps)
                if mut.get('halo_col') is not None and l == 0:
                    X = mut['halo_col']
                    cut = dm.clone()
                    cut[..., :X] = 0
                    bl[..., X] = blur(cut, taps)[..., X]
                e_bl = 26 * U * blur(dm.abs(), taps) if bounds else None
            ref = pc.refs[l][i].to(dt)
            ax_ = Axis(st['ix'].to(dt), st['e_ix'], w, pc.border)
            ay_ = Axis(st['iy'].to(dt), st['e_iy'], h, pc.border)
            sides = [(0, 0)] + ([(-1, -1), (-1, 1), (1, -1), (1, 1)] if bounds else [])
            res = []
            for sx, sy in sides:
                x0, wx1, gmx = ax_.take(sx)
                y0, wy1, gmy = ay_.take(sy)
                wv, ddx, ddy, cross, vmag, dmag, dmagy = bilinear(ref, x0, wx1, y0, wy1)
                df = (tg - wv) * M
                gw = -c_l * rl1_d(df, pc.qch) * M
                if pc.ssim:
                    gw = gw + c_s * (bl[:, :, 0] + 2 * wv * bl[:, :, 1] + tg * bl[:, :, 2])
                gix, giy = (gw * ddx).sum(1), (gw * ddy).sum(1)
                gXn, gYn = gix * gmx, giy * gmy
                res.append(dict(gXn=gXn, gYn=gYn, gw=gw, wv=wv, ddx=ddx, ddy=ddy, cross=cross, dmag=dmag, dmagy=dmagy,
                                gmx=gmx, gmy=gmy, df=df))
            base = res[0]
            tie = ax_.tie | ay_.tie
            ties += int(tie.sum()) if bounds else 0
            if bounds:
                e_wv = st['e_wv']
                e_dx = 4 * U * base['dmag'] + st['e_iy'].unsqueeze(1) * base['cross']
                e_dy = 4 * U * base['dmagy'] + st['e_ix'].unsqueeze(1) * base['cross']
                c_rd = 6 if pc.qch == 0.5 else 12
                rd = rl1_d(base['df'], pc.qch)
                e_gw = abs(c_l) * M * (c_rd * U * rd.abs() + rl1_dd(base['df'], pc.qch) * e_wv * M) + \
                    7 * U * abs(c_l) * (rd * M).abs()
                if pc.ssim:
                    e_gw = e_gw + abs(c_s) * (e_bl[:, :, 0] + 2 * base['wv'].abs() * e_bl[:, :, 1] + 2 * bl[:, :, 1].abs() * e_wv +
                                              tg.abs() * e_bl[:, :, 2]) + \
                        6 * U * abs(c_s) * (bl[:, :, 0].abs() + 2 * (base['wv'] * bl[:, :, 1]).abs() + (tg * bl[:, :, 2]).abs())
                gw = base['gw']
                e_gix = (e_gw * base['ddx'].abs() + gw.abs() * e_dx).sum(1) + 3 * U * (gw * base['ddx']).abs().sum(1)
                e_giy = (e_gw * base['ddy'].abs() + gw.abs() * e_dy).sum(1) + 3 * U * (gw * base['ddy']).abs().sum(1)
                e_gXn = base['gmx'] * e_gix + U * base['gXn'].abs()
                e_gYn = base['gmy'] * e_giy + U * base['gYn'].abs()
            if pc.mode == 'flow':
                sw = (2.0 / w, 2.0 / h) if mut.get('flow_scale_w') else (2.0 / (w - 1), 2.0 / (h - 1))
                cand = [torch.stack([r_['gXn'] * sw[0], r_['gYn'] * sw[1]], 1) for r_ in res]
                dflow_l.append(cand)
                if bounds:
                    dflow_b.append(torch.stack([sw[0] * e_gXn, sw[1] * e_gYn], 1) + 2 * U * cand[0].abs() + TINY32)
            else:
                p = st['proj']
                P = cams(pc.pose.to(dt), pc.K, pc.Kinv, f32(pc.H) / f32(h), pc.rot)[3][:, i]
                Z, X, Y = p['Z'], p['X'], p['Y']
                d_k = _mv(P, p['r'][0], p['r'][1], p['r'][2])
                cand_dd, cand_t = [], []
                for r_ in res:
                    g0 = r_['gXn'] * (2 / (w - 1)) / Z
                    g1 = r_['gYn'] * (2 / (h - 1)) / Z
                    g2 = torch.where(p['zcl'], torch.zeros_like(Z), -(g0 * X + g1 * Y) / Z)
                    cand_dd.append(g0 * d_k[0] + g1 * d_k[1] + g2 * d_k[2])
                    cand_t.append([g * cj for g in (g0, g1, g2) for cj in (p['c'][0], p['c'][1], p['c'][2], torch.ones_like(Z))])
                t = cand_t[0]
                if mut.get('tile_pose') is not None and l == 0:
                    b_, ty, tx = mut['tile_pose']
                    t = [tt.clone() for tt in t]
                    for tt in t:
                        tt[b_, ty * TH:(ty + 1) * TH, tx * TW:(tx + 1) * TW] = 0
                dPl[:, i] = torch.stack([tt.sum((1, 2)) for tt in t], 1)
                vals['variants'].append((l, i, cand_dd))
                if bounds:
                    ax2, ay2 = 2 / (w - 1), 2 / (h - 1)
                    g0 = base['gXn'] * ax2 / Z
                    g1 = base['gYn'] * ay2 / Z
                    g2 = torch.where(p['zcl'], torch.zeros_like(Z), -(g0 * X + g1 * Y) / Z)
                    rz = p['e_Z'] / Z
                    e_g0 = ax2 / Z * e_gXn + (4 * U + rz) * g0.abs()
                    e_g1 = ay2 / Z * e_gYn + (4 * U + rz) * g1.abs()
                    e_g2 = torch.where(p['zcl'], torch.zeros_like(Z),
                                       (e_g0 * X.abs() + g0.abs() * p['e_X'] + e_g1 * Y.abs() + g1.abs() * p['e_Y']) / Z +
                                       g2.abs() * rz + 4 * U * (g0 * X).abs().add((g1 * Y).abs()) / Z)
                    rabs = [rr.abs() for rr in p['r']]
                    Pabs_i = P.abs()
                    dmag_ = _mv(Pabs_i, rabs[0], rabs[1], rabs[2])
                    e_dk = [ _mv(Pabs_i, p['e_r'][0], p['e_r'][1], p['e_r'][2])[k] + 16 * U * dmag_[k] for k in range(3)]
                    gs, egs = (g0, g1, g2), (e_g0, e_g1, e_g2)
                    e_dd = sum(eg * dk.abs() + g.abs() * ed for g, eg, dk, ed in zip(gs, egs, d_k, e_dk)) + \
                        3 * U * sum((g * dk).abs() for g, dk in zip(gs, d_k))
                    gd.append((cand_dd, e_dd, tie))
                    ones = torch.ones_like(Z)
                    e_t = [eg * cj.abs() + g.abs() * ecj + U * (g * cj).abs()
                           for g, eg in zip(gs, egs) for cj, ecj in zip(list(p['c']) + [ones], list(p['e_c']) + [torch.zeros_like(Z)])]
                    # random-sign model over the pixels: rss of the per-pixel chain bounds and of the tie jumps, and
                    # u sqrt(K) ||t||_2 for the reduction itself (K = h w pixels per (b, ref) at this level)
                    jump = [torch.stack([(cand_t[s_][k] - cand_t[0][k]).abs() for s_ in range(1, 5)]).amax(0) * tie
                            for k in range(12)]
                    e_dPl[:, i] = torch.stack([_rss2(et) + _rss2(jk) + U * math.sqrt(h * w) * _rss2(tt)
                                               for et, jk, tt in zip(e_t, jump, cand_t[0])], 1)
                    if l == 0:
                        # the contribution of one 64x20 tile of sample 0 (a middle tile): how far one dropped tile
                        # moves d_pose, reported against the bound at the call's real proportions
                        ty, tx = (h // TH) // 2, (w // TW) // 2
                        tile_dP[i] = torch.stack([tt[0, ty * TH:(ty + 1) * TH, tx * TW:(tx + 1) * TW].sum() for tt in cand_t[0]])
                else:
                    gd.append((cand_dd, None, None))
            if pc.has_mask:
                gm64 = fwd['gmask'][l][:, i].to(dt)
                dmask_l.append(c_l * gm64)
                if bounds:
                    dmask_b.append(abs(c_l) * fwd['b_gmask'][l][:, i] + 2 * U * (c_l * gm64).abs() + TINY32)
        if pc.mode == 'flow':
            vals['d_flow'].append(dflow_l)
            bnds['d_flow'].append(dflow_b)
        else:
            # d_depth: sum over the refs (sequential fp32 adds in the kernel)
            cands = [sum(c_[0][s_] for c_ in gd) for s_ in range(len(gd[0][0]))]
            vals['d_depth'].append([c_.unsqueeze(1) for c_ in cands])
            if bounds:
                e_dd = sum(c_[1] for c_ in gd) + 3 * U * sum(c_[0][0].abs() for c_ in gd)
                bnds['d_depth'].append(e_dd.unsqueeze(1) + TINY32)
            # pose: dP -> d pose through the level's camera
            J = pose_jac(pc, l, dt)
            dP_tot = dP_tot + torch.einsum('brkj,brk->brj', J, dPl)
            if bounds:
                Ja = J.abs()
                e_pose = e_pose + torch.einsum('brkj,brk->brj', Ja, e_dPl) + (12 + L) * U * torch.einsum('brkj,brk->brj', Ja, dPl.abs())
            if l == 0 and bounds:
                vals['tile_dpose'] = torch.einsum('rkj,rk->rj', J[0], tile_dP)
        if pc.has_mask:
            vals['d_mask'].append(torch.stack(dmask_l, 1))
            if bounds:
                bnds['d_mask'].append(torch.stack(dmask_b, 1))
    if pc.mode == 'rigid':
        vals['d_pose'] = dP_tot
        bnds['d_pose'] = e_pose + TINY32
    vals['ties'] = ties
    return vals, (bnds if bounds else None)


def nearest(got, cands):
    """Per element, the candidate closest to got (the one-sided fp64 values at the tie elements)."""
    g = _d(got)
    best = cands[0]
    bd = (g - best).abs()
    for c in cands[1:]:
        d = (g - c).abs()
        best = torch.where(d < bd, c, best)
        bd = torch.minimum(bd, d)
    return best


def photo_fwd_checks(pc, vo, dmaps, gmask, scal, loss):
    """checks of one photometric forward from the kernel's (or a stand-in's) outputs; returns (checks, fwd state)."""
    fwd, b = photo_forward(pc, f64, vo_kernel=vo)
    checks = []
    for l in range(pc.L):
        exact = fwd['vo'][l]
        checks.append(('vo', vo[l], exact, torch.full_like(exact, TINY32), None))
        if pc.ssim:
            checks.append(('dmaps', dmaps[l], fwd['dmaps'][l], b['dmaps'][l], None))
        if pc.has_mask:
            checks.append(('gmask', gmask[l], fwd['gmask'][l], b['gmask'][l], None))
    checks.append(('scal', scal.view(pc.L, pc.R, 4), fwd['scal'], b['scal'], None))
    checks.append(('loss', loss.reshape(()), fwd['loss'].reshape(()), torch.tensor(b['loss'], dtype=f64), None))
    fwd['b_gmask'] = b['gmask']
    return _merge(checks), fwd


def _merge(checks):
    """Same-named checks of several levels -> one check each (flattened), so a call reports one r per output."""
    out, order = {}, []
    for what, got, ref, s, tie in checks:
        if what not in out:
            out[what] = ([], [], [])
            order.append(what)
        out[what][0].append(_d(got).reshape(-1).cpu())
        out[what][1].append(ref.detach().to(f64).reshape(-1).cpu())
        out[what][2].append(s.detach().to(f64).reshape(-1).cpu() if torch.is_tensor(s) else torch.full_like(out[what][1][-1], s))
    return [(w_, torch.cat(out[w_][0]), torch.cat(out[w_][1]), torch.cat(out[w_][2]), None) for w_ in order]


def photo_bwd_checks(pc, fwd, go, vo, dmaps, scal, grads):
    """grads: what the backward returned after the None of cfg (rigid: d_pose, d_depth[L], d_mask[L]; flow:
    d_flow[L*R] level-major, d_mask[L])."""
    v, b = photo_backward(pc, fwd, go, vo, dmaps, scal.view(pc.L, pc.R, 4))
    L, Rr = pc.L, pc.R
    extra = {}
    checks = []
    if pc.mode == 'rigid':
        d_pose, d_depth = grads[0], grads[1:1 + L]
        rest = grads[1 + L:]
        checks.append(('d_pose', d_pose, v['d_pose'], b['d_pose'], None))
        # r of d_pose[0] if one middle tile of level 0 had been dropped: the least r over the refs
        drop = (_d(d_pose)[0] - v['tile_dpose'] - v['d_pose'][0]).abs() / b['d_pose'][0]
        extra = dict(tile_drop_r=float(drop.amax(1).amin()))
        for l in range(L):
            checks.append(('d_depth', d_depth[l], nearest(d_depth[l], v['d_depth'][l]), b['d_depth'][l], None))
    else:
        d_flow = grads[:L * Rr]
        rest = grads[L * Rr:]
        for l in range(L):
            for i in range(Rr):
                got = d_flow[l * Rr + i]
                checks.append(('d_flow', got, nearest(got, v['d_flow'][l][i]), b['d_flow'][l][i], None))
    if pc.has_mask:
        for l in range(L):
            checks.append(('d_mask', rest[l], v['d_mask'][l], b['d_mask'][l], None))
    extra['coord_ties'] = v['ties']
    return _merge(checks), extra


# ---------------------------------------------------------------------------------------------------------------------
# Smoothness (smooth_bce.cu)
def _sgn(x):
    return torch.sign(x)


def smooth_checks(kind, preds, imgs, loss, go=None, grads=None):
    """Forward (loss) or backward (grads) checks of one _SmoothLoss call against fp64.  The abs kinks are decided on
    the fp32 values the kernel forms, so their signs match exactly."""
    L = len(preds)
    total, e_total = 0.0, 0.0
    checks = []
    lw = 1.0
    for l, p32 in enumerate(preds):
        p = _d(p32)
        B, C, h, w = p.shape
        nblk = B * -(-(h * w) // PNT)
        D = C + BLOCK_TREE + _sum_depth(nblk, 256) + BLOCK_TREE + L
        if kind == _lib.SMOOTH_EDGE:
            # edge_w: three abs differences, two adds, / 3, expf (<= 2 ulp): wx within wx (4u s / 3 + 4u)
            im = _d(imgs[l])
            sx = (im[:, :, :-1] - im[:, :, 1:]).abs().sum(1, keepdim=True)
            sy = (im[:, :, :, :-1] - im[:, :, :, 1:]).abs().sum(1, keepdim=True)
            wx, wy = torch.exp(-(sx / 3)), torch.exp(-(sy / 3))
            ewx, ewy = wx * (4 * U * sx / 3 + 4 * U), wy * (4 * U * sy / 3 + 4 * U)
            dx, dy = p[:, :, :-1] - p[:, :, 1:], p[:, :, :, :-1] - p[:, :, :, 1:]
            n0, n1 = B * C * (h - 1) * w, B * C * h * (w - 1)
            if grads is None:
                s0, s1 = (dx.abs() * wx).sum(), (dy.abs() * wy).sum()
                e0 = D * U * s0 + (dx.abs() * (ewx + 2 * U * wx)).sum()
                e1 = D * U * s1 + (dy.abs() * (ewy + 2 * U * wy)).sum()
                total = total + s0 / n0 + s1 / n1
                e_total = e_total + e0 / n0 + e1 / n1 + 3 * U * (s0 / n0 + s1 / n1)
            else:
                # d = go * sum of <= 4 signed weights w / n: each weight's error, its division, four adds
                sgx = _sgn((p32[:, :, :-1] - p32[:, :, 1:]).double())
                sgy = _sgn((p32[:, :, :, :-1] - p32[:, :, :, 1:]).double())
                g, m = torch.zeros_like(p), torch.zeros_like(p)
                tx, ty = sgx * wx / n0, sgy * wy / n1
                mx, my = sgx.abs() * (ewx + 6 * U * wx) / n0, sgy.abs() * (ewy + 6 * U * wy) / n1
                g[:, :, :-1] += tx
                g[:, :, 1:] -= tx
                g[..., :-1] += ty
                g[..., 1:] -= ty
                m[:, :, :-1] += mx
                m[:, :, 1:] += mx
                m[..., :-1] += my
                m[..., 1:] += my
                ref = float(go) * g
                checks.append(('d_pred', grads[l], ref, abs(float(go)) * m + 2 * U * ref.abs() + TINY32, None))
        else:
            def d2(a, b, c):
                return (a - b) - (b - c)
            q = p32
            terms = [d2(q[..., 2:], q[..., 1:-1], q[..., :-2]),
                     (q[:, :, 1:, 1:] - q[:, :, 1:, :-1]) - (q[:, :, :-1, 1:] - q[:, :, :-1, :-1]),
                     (q[:, :, 1:, 1:] - q[:, :, :-1, 1:]) - (q[:, :, 1:, :-1] - q[:, :, :-1, :-1]),
                     d2(q[:, :, 2:], q[:, :, 1:-1], q[:, :, :-2])]
            pd = p
            ex = [d2(pd[..., 2:], pd[..., 1:-1], pd[..., :-2]),
                  (pd[:, :, 1:, 1:] - pd[:, :, 1:, :-1]) - (pd[:, :, :-1, 1:] - pd[:, :, :-1, :-1]),
                  (pd[:, :, 1:, 1:] - pd[:, :, :-1, 1:]) - (pd[:, :, 1:, :-1] - pd[:, :, :-1, :-1]),
                  d2(pd[:, :, 2:], pd[:, :, 1:-1], pd[:, :, :-2])]
            ns = [B * C * h * (w - 2), B * C * (h - 1) * (w - 1), B * C * (h - 1) * (w - 1), B * C * (h - 2) * w]
            lwf = f32(lw)
            if grads is None:
                # fp32 second difference: 3 roundings of |a| + 2|b| + |c|
                mags = [ (pd[..., 2:].abs() + 2 * pd[..., 1:-1].abs() + pd[..., :-2].abs()),
                         pd[:, :, 1:, 1:].abs() + pd[:, :, 1:, :-1].abs() + pd[:, :, :-1, 1:].abs() + pd[:, :, :-1, :-1].abs(),
                         pd[:, :, 1:, 1:].abs() + pd[:, :, 1:, :-1].abs() + pd[:, :, :-1, 1:].abs() + pd[:, :, :-1, :-1].abs(),
                         (pd[:, :, 2:].abs() + 2 * pd[:, :, 1:-1].abs() + pd[:, :, :-2].abs())]
                Ls, es = 0.0, 0.0
                for t, n, mg in zip(ex, ns, mags):
                    s_ = t.abs().sum()
                    Ls = Ls + s_ / n
                    es = es + (D * U * s_ + 3 * U * mg.sum()) / n + 2 * U * s_ / n
                total = total + Ls * lwf
                e_total = e_total + es * lwf + 5 * U * Ls * lwf
            else:
                sg = [_sgn(t.double()) for t in terms]
                g = torch.zeros_like(p)
                m = torch.zeros_like(p)
                # dx2 (along w) and dy2 (along h): coefficients +1, -2, +1 at offsets 0, 1, 2
                for t, n, ax in ((sg[0], ns[0], -1), (sg[3], ns[3], -2)):
                    size = p.shape[ax]
                    for off, c in ((0, 1.0), (1, -2.0), (2, 1.0)):
                        idx = [slice(None)] * 4
                        idx[ax] = slice(off, size - 2 + off)
                        g[tuple(idx)] += c * t / n
                        m[tuple(idx)] += abs(c) * t.abs() / n
                for t, n in ((sg[1], ns[1]), (sg[2], ns[2])):
                    for (oy, ox, c) in ((1, 1, 1.0), (1, 0, -1.0), (0, 1, -1.0), (0, 0, 1.0)):
                        g[:, :, oy:h - 1 + oy, ox:w - 1 + ox] += c * t / n
                        m[:, :, oy:h - 1 + oy, ox:w - 1 + ox] += t.abs() / n
                ref = float(go) * lwf * g
                s = abs(float(go) * lwf) * 16 * U * m + 2 * U * ref.abs() + TINY32
                checks.append(('d_pred', grads[l], ref, s, None))
            lw /= 2.3
    if grads is None:
        checks.append(('loss', loss.reshape(()), torch.as_tensor(total, dtype=f64), torch.as_tensor(e_total + TINY32, dtype=f64), None))
    return _merge(checks)


# ---------------------------------------------------------------------------------------------------------------------
# BCE (smooth_bce.cu)
def bce_checks(cfg, masks, loss=None, go=None, grads=None):
    """Forward (loss) or backward (grads) checks of one _BceLoss call against fp64."""
    kind = cfg['kind']
    eps = 1e-8
    L = len(masks)
    checks = []
    total, e_total = 0.0, 0.0
    for l, m32 in enumerate(masks):
        m = _d(m32)
        B, C, h, w = m.shape
        n = B * C * h * w
        nblk = B * -(-(h * w) // PNT)
        D = C + BLOCK_TREE + _sum_depth(nblk, 256) + BLOCK_TREE + L
        if kind == _lib.BCE_ONES:
            t = -torch.log(m).clamp_min(-100)
            if grads is None:
                s_ = t.sum()
                total = total + s_ / n
                e_total = e_total + (D * U * s_ + (2 * U * t.abs() + U).sum()) / n + 2 * U * s_ / n
            else:
                gn = float(go) / n
                ref = gn * (m - 1) / torch.clamp_min((1 - m) * m, 1e-12)
                checks.append(('d_mask', grads[l], ref, 6 * U * ref.abs() + TINY32, None))
        else:
            th = f32(cfg['thresh'])
            cf, cb = cfg['census_fwd'][l].float(), cfg['census_bwd'][l].float()
            f = ((cf[:, 0:1] < th) & (cf[:, 1:2] < th)).double()
            bw = ((cb[:, 0:1] < th) & (cb[:, 1:2] < th)).double()
            f = 1 - (1 - f) * (1 - _d(cfg['target_fwd'][l]))
            bw = 1 - (1 - bw) * (1 - _d(cfg['target_bwd'][l]))
            tt = torch.cat([bw, bw, f, f], 1)
            w0, w1 = f32(cfg['wbce']), f32(1 - f32(cfg['wbce']))
            a, b = m + eps, (1 - m) + eps
            if grads is None:
                t = w1 * (tt * torch.log(a)) + w0 * ((1 - tt) * torch.log(b))
                s_ = t.sum()
                mag = (w1 * tt * torch.log(a).abs() + w0 * (1 - tt) * torch.log(b).abs())
                total = total - s_ / n
                e_total = e_total + (D * U * mag.sum() + (4 * U * mag + 3 * U * (w1 * tt + w0 * (1 - tt))).sum()) / n + 2 * U * mag.sum() / n
            else:
                gn = float(go) / n
                ref = -gn * (w1 * tt / a - w0 * (1 - tt) / b)
                mag = abs(gn) * (w1 * tt / a + w0 * (1 - tt) / b)
                checks.append(('d_mask', grads[l], ref, 6 * U * mag + TINY32, None))
    if grads is None:
        checks.append(('loss', loss.reshape(()), torch.as_tensor(total, dtype=f64), torch.as_tensor(e_total + TINY32, dtype=f64), None))
    return _merge(checks)


# ---------------------------------------------------------------------------------------------------------------------
def pose2flow_checks(depth, pose, K, Kinv, rot, out):
    """pose2flow forward (warp_ops.cu rigid_fwd_kernel<true>: unscaled camera, no rewrite)."""
    B, h, w = depth.shape
    Ki, Ks, T, P = cams(_d(pose).view(B, 1, 6), _d(K), _d(Kinv), 1.0, rot)
    p = project(Ki, P[:, 0], _d(depth), w, h, (Ks.abs().unsqueeze(1) @ T.abs())[:, 0])
    u_, v_ = coords_to_flow(p['Xn'], p['Yn'], w, h)
    xs, ys = _grid(B, h, w, f64, depth.device)
    ref = torch.stack([u_, v_], 1)
    s = torch.stack([(w - 1) / 2 * p['e_Xn'] + 3 * U * (u_.abs() + xs + (w - 1)),
                     (h - 1) / 2 * p['e_Yn'] + 3 * U * (v_.abs() + ys + (h - 1))], 1) + TINY32
    cap = max(LA.REL_BAR, 8 * U * (max(w, h) - 1) / max(float(ref.abs().max()), 1e-30))
    return [('flow', out, ref, s, None)], {'flow': cap}


def pyramid_checks(img, sizes, levels):
    """levels_for: level l the exact 2^l box mean; the kernel's 2x2 means of 2x2 means round 2 adds per stage of sums
    of |x| (the 0.25 is exact)."""
    x = _d(img)
    H = x.shape[2]
    checks = []
    for (h, w), got in zip(sizes, levels):
        k = H // h
        stages = int(round(math.log2(k)))
        if stages == 0:
            checks.append(('level', got, x, torch.full_like(x, TINY32), None))
            continue
        ref = F.avg_pool2d(x, k)
        s = 2 * stages * U * F.avg_pool2d(x.abs(), k) + TINY32
        checks.append(('level', got, ref, s, None))
    return _merge(checks)


def evaluate(fam, checks, rel_cap=None):
    """layer_audit.evaluate of each check against its own R_OUT; rel_cap: {output: cap} replacing the 1e-4 bar."""
    res, bad = {}, []
    for chk in checks:
        r1, _, b1 = LA.evaluate(fam, [chk], {fam: R_OUT[(fam, chk[0])]})
        res.update(r1)
        cap = (rel_cap or {}).get(chk[0])
        bad += [b for b in b1 if not (cap is not None and ' rel_err ' in b and res[chk[0]][1] <= cap)]
    return res, max([v[0] for v in res.values()] or [0.0]), bad


# ---------------------------------------------------------------------------------------------------------------------
def cfg3_losses(device, B=2, H=64, W=128, NL=4, seed=77, hp=HP, opts=None):
    """loss_cfg3's loss layer (train_step.loss_cfg3 without the nets) on synthetic network outputs; backward of the
    weighted sum.  opts: rot, pad, wssim, qch, lam, masks."""
    s = synth.sample(B, H, W, seed=seed, nlevels=NL)
    dv = lambda x: [t.to(device) for t in x] if isinstance(x, list) else x.to(device)      # noqa: E731
    o = dict(rot='euler', pad='zeros', wssim=hp['wssim'], qch=hp['qch'], lam=hp['lambda_oob'], masks=True)
    o.update(opts or {})
    tgt, refs, K, Kinv = dv(s['tgt']), dv(s['refs']), dv(s['K']), dv(s['Kinv'])
    depth = [t.requires_grad_(True) for t in dv(s['depth'])]
    pose = dv(s['pose']).requires_grad_(True)
    emask = [t.requires_grad_(True) for t in dv(s['emask'])]
    ff = [t.requires_grad_(True) for t in dv(s['flow_fwd'])]
    fb = [t.requires_grad_(True) for t in dv(s['flow_bwd'])]
    cam_f = [pose2flow(d.squeeze(1), pose[:, 2], K, Kinv, rotation_mode=o['rot']) for d in depth]
    cam_b = [pose2flow(d.squeeze(1), pose[:, 1], K, Kinv, rotation_mode=o['rot']) for d in depth]
    tm = CL.consensus_exp_masks(cam_f, cam_b, ff, fb, tgt, refs[2], refs[1], wssim=o['wssim'], wrig=hp['wrig'], ws=hp['w3'])
    rig_f = [(a - b).abs() for a, b in zip(cam_f, ff)]
    rig_b = [(a - b).abs() for a, b in zip(cam_b, fb)]
    em = emask if o['masks'] else [None] * NL
    fem = [1 - m[:, 1:3] for m in emask] if o['masks'] else [None] * NL
    l1 = CL.photometric_reconstruction_loss(tgt, refs, K, Kinv, depth, em, pose, rotation_mode=o['rot'], padding_mode=o['pad'],
                                            lambda_oob=o['lam'], qch=o['qch'], wssim=o['wssim'])
    l2 = CL.explainability_loss(emask)
    l3 = sum(CL.edge_aware_smoothness_loss(tgt, p) for p in (depth, ff, fb, emask))
    l4 = CL.photometric_flow_loss(tgt, refs[1:3], [fb, ff], fem, lambda_oob=o['lam'], qch=o['qch'], wssim=o['wssim'])
    l5 = CL.consensus_depth_flow_mask(emask, rig_b, rig_f, tm, tm, THRESH=hp['THRESH'], wbce=hp['wbce'])
    loss = hp['w1'] * l1 + hp['w2'] * l2 + hp['w3'] * l3 + hp['w4'] * l4 + hp['w5'] * l5
    loss.backward()
    return loss

SWEEP = [dict(wssim=0.0), dict(qch=0.4), dict(lam=0.2), dict(pad='border'), dict(rot='quat'), dict(masks=False),
         dict(H=84, W=136, NL=3)]




class LossAudit:
    """with LossAudit() as audit: ... run the loss layer forward / backward ...  (see the module docstring)"""

    FNS = {'photo': (CL, '_PhotoLoss'), 'smooth': (CL, '_SmoothLoss'), 'bce': (CL, '_BceLoss')}

    def __init__(self, tag='audit', report=True, consensus=True):
        self.tag, self.report, self.consensus = tag, report, consensus
        self.rows = []
        self._saved = None

    def __enter__(self):
        self._saved = {k: (getattr(m, c).__dict__['forward'], getattr(m, c).__dict__['backward']) for k, (m, c) in self.FNS.items()}
        self._saved_p2f = CW._Pose2Flow.__dict__['forward']
        self._saved_attr = (CL.consensus_exp_masks, CP.levels_for)
        try:
            for k, (m, c) in self.FNS.items():
                f, b = self._saved[k]
                setattr(getattr(m, c), 'forward', staticmethod(self._wrap_fwd(k, f.__func__)))
                setattr(getattr(m, c), 'backward', staticmethod(self._wrap_bwd(k, b.__func__)))
            CW._Pose2Flow.forward = staticmethod(self._wrap_p2f(self._saved_p2f.__func__))
            CL.consensus_exp_masks = self._wrap_consensus(self._saved_attr[0])
            CP.levels_for = self._wrap_pyramid(self._saved_attr[1])
        except BaseException:
            self._restore()
            raise
        return self

    def __exit__(self, et, ev, tb):
        self._restore()
        if et is None:
            self.finish()
        return False

    def _restore(self):
        if self._saved is not None:
            for k, (m, c) in self.FNS.items():
                setattr(getattr(m, c), 'forward', self._saved[k][0])
                setattr(getattr(m, c), 'backward', self._saved[k][1])
            CW._Pose2Flow.forward = self._saved_p2f
            CL.consensus_exp_masks, CP.levels_for = self._saved_attr
            self._saved = None

    # ---- wrappers ---------------------------------------------------------------------------------------------------
    def _wrap_fwd(self, fam, orig):
        audit = self

        def forward(ctx, cfg, *tensors):
            out = orig(ctx, cfg, *tensors)
            with torch.no_grad():
                audit._fwd(fam, ctx, cfg, tensors, out)
            return out
        return forward

    def _wrap_bwd(self, fam, orig):
        audit = self

        def backward(ctx, g):
            grads = orig(ctx, g)
            with torch.no_grad():
                audit._bwd(fam, ctx, g, grads)
            return grads
        return backward

    def _wrap_p2f(self, orig):
        audit = self

        def forward(ctx, depth, pose, K, Kinv, rot, pad):
            out = orig(ctx, depth, pose, K, Kinv, rot, pad)
            with torch.no_grad():
                checks, cap = pose2flow_checks(depth.detach().float(), pose.detach().float(), K.detach().float(),
                                               Kinv.detach().float(), rot, out)
                audit._record('pose2flow', 'fwd', tuple(depth.shape), checks, 3, rel_cap=cap)
            return out
        return forward

    def _wrap_consensus(self, orig):
        audit = self

        def consensus_exp_masks(cam_f, cam_b, ff, fb, tgt, rf, rb, wssim, wrig, ws=0.1):
            out = orig(cam_f, cam_b, ff, fb, tgt, rf, rb, wssim, wrig, ws)
            if audit.consensus:
                with torch.no_grad():
                    audit._consensus(out, cam_f, cam_b, ff, fb, tgt, rf, rb, wssim, wrig)
            return out
        return consensus_exp_masks

    def _wrap_pyramid(self, orig):
        audit = self

        def levels_for(img, sizes):
            out = orig(img, sizes)
            with torch.no_grad():
                audit._record('pyramid', 'fwd', tuple(img.shape), pyramid_checks(img, sizes, out),
                              max((img.shape[2] // h) ** 2 for h, _ in sizes))
            return out
        return levels_for

    # ---- per-call checks ---------------------------------------------------------------------------------------------
    def _fwd(self, fam, ctx, cfg, tensors, out):
        if fam == 'photo':
            pc = PhotoCall(cfg, tensors)
            L = pc.L
            keep = ctx.keep[len(tensors) + (2 if pc.mode == 'rigid' else 0):]
            dm = keep[:L] if pc.ssim else [None] * L
            keep = keep[L if pc.ssim else 0:]
            vo, keep = keep[:L], keep[L:]
            gm = keep[:L] if pc.has_mask else [None] * L
            keep = keep[L if pc.has_mask else 0:]
            scal = keep[0]
            checks, st = photo_fwd_checks(pc, vo, dm, gm, scal, out)
            ctx._audit = (pc, st, vo, dm, scal)
            n_vo = sum(t.numel() for t in vo)
            r = self._record('photo_' + pc.mode, 'fwd', (pc.B, pc.L, pc.R) + tuple(pc.sizes[0]), checks, 3 * pc.B * max(h * w for h, w in pc.sizes),
                             dict(vo_ties=st['ties']['vo'], vo_elems=n_vo, coord_ties=st['ties']['coord'],
                                  partial_tiles=[bool(h % TH or w % TW) for h, w in pc.sizes]),
                             rel_cap={'dmaps': DMAPS_REL_CAP} if pc.W >= DMAPS_CAP_MIN_W else None)
            if sum(st['vo_bad']):
                r['bad'].append('vo: %d elements differ from fp64 away from a threshold' % sum(st['vo_bad']))
            if st['ties']['vo'] > VO_TIE_FRAC * n_vo:
                r['bad'].append('vo: %d rounding ties of %d elements (more than %g of them)' % (st['ties']['vo'], n_vo, VO_TIE_FRAC))
        elif fam == 'smooth':
            preds = [t.detach().float() for t in tensors]
            imgs = cfg.get('img')
            ctx._audit = (cfg['kind'], preds, imgs)
            self._record('smooth', 'fwd', tuple(preds[0].shape), smooth_checks(cfg['kind'], preds, imgs, out), preds[0].numel())
        else:
            masks = [t.detach().float() for t in tensors]
            ctx._audit = (cfg, masks)
            self._record('bce', 'fwd', tuple(masks[0].shape), bce_checks(cfg, masks, loss=out), masks[0].numel())

    def _bwd(self, fam, ctx, g, grads):
        if fam == 'photo':
            pc, st, vo, dm, scal = ctx._audit
            checks, extra = photo_bwd_checks(pc, st, g, vo, dm, scal, grads[1:])
            # longest reduction: the pose sum over one level's pixels per (b, ref); the flow gradient sums 3 channels
            self._record('photo_' + pc.mode, 'bwd', (pc.B, pc.L, pc.R) + tuple(pc.sizes[0]), checks,
                         max(h * w for h, w in pc.sizes) if pc.mode == 'rigid' else 3, extra)
        elif fam == 'smooth':
            kind, preds, imgs = ctx._audit
            self._record('smooth', 'bwd', tuple(preds[0].shape), smooth_checks(kind, preds, imgs, None, go=g, grads=grads[1:]), 12)
        else:
            cfg, masks = ctx._audit
            self._record('bce', 'bwd', tuple(masks[0].shape), bce_checks(cfg, masks, go=g, grads=grads[1:]), 1)

    def _consensus(self, out, cam_f, cam_b, ff, fb, tgt, rf, rb, wssim, wrig):
        from oracle import losses as OL
        from tests.kernel_cases import check_consensus_targets
        sides = OL.consensus_sides(cam_f, cam_b, ff, fb, tgt, rf, rb, wssim=wssim, wrig=wrig)
        ref = [(a <= (b + 1e-8)).float() for a, b in sides]
        dd = lambda x: [t.detach().double() for t in x]          # noqa: E731
        sides64 = OL.consensus_sides(dd(cam_f), dd(cam_b), dd(ff), dd(fb), tgt.double(), rf.double(), rb.double(),
                                     wssim=wssim, wrig=wrig)
        row = dict(op='consensus', phase='fwd', shape=list(tgt.shape), K=0, r=0.0, checks={}, bad=[])
        try:
            n_mis, n_px = check_consensus_targets(out, ref, sides, sides64=sides64)
            row.update(ties=n_mis, pixels=n_px)
        except AssertionError as e:
            row['bad'].append(str(e))
            row['r'] = float('inf')
        self.rows.append(row)

    def _record(self, fam, phase, shape, checks, K, extra=None, rel_cap=None):
        """K: the longest reduction one checked value of the call sums (1 for elementwise outputs)."""
        res, r, bad = evaluate(fam, checks, rel_cap)
        row = dict(op=fam, phase=phase, shape=list(shape), K=K, r=r,
                   checks={k: dict(r=v[0], rel=v[1], ties=v[2]) for k, v in res.items()}, bad=bad)
        row.update(extra or {})
        self.rows.append(row)
        return row

    # ---- report -------------------------------------------------------------------------------------------------------
    def summary(self):
        fams = {}
        for row in self.rows:
            fams.setdefault(row['op'], []).append(row)
        out = {}
        for fam, rows in fams.items():
            rs = [row['r'] for row in rows]
            out[fam] = dict(calls=len(rows), fwd=sum(r_['phase'] == 'fwd' for r_ in rows), bwd=sum(r_['phase'] == 'bwd' for r_ in rows),
                            r_max=max(rs), r_median=statistics.median(rs), R=R[fam],
                            ties=sum(row.get('vo_ties', 0) + row.get('coord_ties', 0) + row.get('ties', 0) for row in rows),
                            rel_max=max([c['rel'] for row in rows for c in row['checks'].values()] or [0.0]),
                            outputs={w: dict(r_max=max(row['checks'][w]['r'] for row in rows if w in row['checks']),
                                             rel_max=max(row['checks'][w]['rel'] for row in rows if w in row['checks']),
                                             R=R_OUT.get((fam, w)))
                                     for w in sorted({w for row in rows for w in row['checks']})})
            if fam == 'photo_rigid':
                drops = [row['tile_drop_r'] for row in rows if 'tile_drop_r' in row]
                if drops:
                    out[fam]['tile_drop_r'] = min(drops)
        return out

    def finish(self):
        summ = self.summary()
        if self.report:
            print('\n== loss audit %s: %d calls' % (self.tag, len(self.rows)))
            print('   %-12s %5s %5s %10s %10s %5s %8s %10s' % ('family', 'fwd', 'bwd', 'r worst', 'r median', 'R', 'ties', 'rel max'))
            for fam in FAMILIES:
                if fam in summ:
                    d = summ[fam]
                    print('   %-12s %5d %5d %10.3g %10.3g %5.3g %8d %10.2e' % (fam, d['fwd'], d['bwd'], d['r_max'], d['r_median'],
                                                                         d['R'], d['ties'], d['rel_max']))
                    for w, o in d['outputs'].items():
                        print('     %-10s %21s %10.3g %5.3g %8s %10.2e' % (w, '', o['r_max'], o['R'], '', o['rel_max']))
                    if 'tile_drop_r' in d:
                        print('     one dropped level-0 tile would score d_pose r = %.3g' % d['tile_drop_r'])
            out = os.environ.get('CCB_PARITY_REPORT_DIR')
            if out:
                os.makedirs(out, exist_ok=True)
                with open(os.path.join(out, 'loss_audit_%s.json' % self.tag), 'w') as f:
                    json.dump(dict(summary=summ, R={'%s.%s' % k: v for k, v in R_OUT.items()}, rows=self.rows), f, indent=1, default=str)
        bad = ['%s %s %s: %s' % (row['op'], row['phase'], row['shape'], '; '.join(row['bad'])) for row in self.rows if row['bad']]
        assert not bad, '%d loss-layer calls over their bound:\n  ' % len(bad) + '\n  '.join(bad[:60])
        return summ
