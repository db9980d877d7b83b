"""Per-layer audit of the CUDA kernels against fp64, element by element, on the inputs a real run hands them.

`LayerAudit` is a context manager.  While it is active, the forward and backward staticmethods of the seven autograd
Functions of cc_b200.nn (_Conv2dFn, _ConvT2dFn, _BatchNormFn, _Upsample2xFn, _Corr81Fn, _Corr441dFn, _FeatWarpFn) are
wrapped: after each real kernel call the wrapper takes the call's fp32 inputs (x, w, bias, res, upstream gradient, the saved
output / statistics), recomputes the operation in fp64 with torch, and checks every output element against the bound
derived below.  Gradients a backward wrote straight into FlatAdam's flat buffer (cc_b200.nn._grad_slot) are read from
`param._ccb_grad` right after the backward returns.  The audit is read-only: it works on fp64 copies, freed per call, and
changes no fp32 result (tests/test_gpu_fullsize.py holds the audited step bit-identical to an unaudited one).

Module names come from forward pre-hooks on the nets handed to the audit; the backward row of a call carries the name
of its forward.  Convolution rows carry the kernels the call dispatched to (ccb_debug_last_conv_kernel after every
fprop / dgrad / wgrad launch) and the plan of each launch (ccb_debug_conv_plan: the path - CUDA-core GEMM, tensor cores,
tensor-core weight gradient through padded rows - and the split-K count).  On exit the audit prints one table per op
family - calls, worst and median normalised error, kernels seen - and raises an AssertionError listing every call over
its bound.  With $CCB_PARITY_REPORT_DIR set,
the rows are written there as layer_audit_<tag>.json.

Error model (u = 2^-24, |.| elementwise, every bound gets TINY32 for products that underflow fp32)
-----------------------------------------------------------------------------------------------
Long reductions (convolution fprop / dgrad / wgrad / bias gradient, BatchNorm sums, the cost volume).  An output
element i is a sum of K_i products t_i.  Rounding the running sums of K terms of random sign leaves an error of the
order u * sqrt(K) * ||t_i||_2 - the partial sums grow like sqrt(k) times the rms term - whatever the blocking (tiles,
split-K, CTA trees only shorten the chains).  The worst case gamma_K * sum |t| is useless for detection at K ~ 10^5.
So the scale of element i is

    s_i = (u * sqrt(K) + c_t) * ||t_i||_2  +  epilogue roundings  +  TINY32

where ||t_i||_2 is computed in fp64 by the same operation on squared operands (conv(x^2, w^2), convT(dz^2, w^2),
wgrad(x^2, dz^2), sum dz^2, corr(f1^2, f2^2), ...), K is the largest number of products one element sums (Ci k^2 for
fprop, Co ceil(k/s)^2 for a stride-s data gradient, B Ho Wo for the weight and bias gradients, C or 81 for the cost
volume, C or 441 for FlowNetC6's dilated one), and c_t is the error each product carries before it is summed, a
per-term relative error of random sign:
  C_TC   = 12u  tensor-core convolutions: the 3xTF32 split keeps hi*hi + hi*lo + lo*hi, so each product is off by
                about 2^-21 = 8u of itself; plus ~4u for the fp32 rounding of the operand (dz = g * act'(y)) and product
  C_PROD =  4u  CUDA-core reductions: the product and its operand roundings
The epilogue adds EPI = 3 roundings of |acc| + |bias| + |res| (two adds and the activation input); an activation with
Lipschitz constant L (1 for ReLU / LeakyReLU / none, sigmoid'(z) for the sigmoid) scales the bound by L and adds its
own rounding (LeakyReLU's slope multiply: u |y|; sigmoid, expf + add + divide: 4u |y|).

The check is r_i = |kernel_i - fp64_i| / s_i <= R_op, R_op a constant per op family (R below).  R_op must leave one
dropped or duplicated term of typical size detectable: that term's error is ||t||_2 / sqrt(K), so r = 1 / (u K) and
R_op < 1 / (u K_max) for the largest K the audit meets (asserted at exit).  At 256x832 the weight gradient of
DispResNet6's iconv1 reduces 4 * 256 * 832 = 851968 products (1 / (u K) = 19.7), conv1's 212992 (78.8).

Where the terms of a reduction share a sign, the sqrt(K) model is optimistic: the partial sums grow linearly instead of
like sqrt(k), and a chain of n fp32 additions leaves an error of about u sqrt(n) / 3 * |sum| = u sqrt(n) / 3 * sqrt(K)
||t||_2 for equal terms, i.e. r ~ sqrt(n) / 3.  The weight and bias gradients of the heads at full resolution are such
sums (non-negative activations times an upstream gradient of one sign over most of the map): MaskNet6's pred_mask1 bias
gradient (K = 851968) measures r = 6.3 on the H100, the largest of the step, which matches chains of a few hundred
additions.  This stays below the detectability cap, so R_conv = 10 keeps a dropped term of typical size visible.

BatchNorm (N = B h w values per channel).  mean: u rms(x) + u |mean|; variance: u rms((x - mean)^2) + 2u var;
invstd = 1/sqrt(var + eps): invstd (s_var / (2 (var + eps)) + 3u).  The running statistics add 3 / 4 roundings of
their summands to momentum times those.  y and dx are elementwise given the statistics the kernel saved (they are
the backward's own inputs): y = xh gamma + beta within 4u (|xh gamma| + |beta|); dbeta = sum g and dgamma =
sum g xh are long reductions (K = N, c_t = 0 and 4u); dx = gamma invstd (g - dbeta/N - xh dgamma/N) gets the
reductions' bounds divided by N plus 6u of its three terms.

Dilated cost volume (corr441d: FlowNetC6's 21x21 displacements at dilation 2, LeakyReLU(0.1) fused).
  forward: the kernel sums the C products f1 f2 of an output in fp32, divides by C and applies the activation.  The
           activation is inverted exactly in fp64 (out / 0.1f where out <= 0: the slope multiply adds u |z|), and the
           pre-activation z is held to  s = (u sqrt(C) + C_PROD) ||t||_2 / C + 3u |z|  (K = C).
  d f1 / d f2: sums of the 441 products dz f (dz = g * leaky'(out), from the sign of the forward's own output), divided
           by C:  s = (u sqrt(441) + C_PROD) ||t||_2 / C + 2u |ref|  (K = 441).

Elementwise and short ops: a worst-case count of roundings times u sum |terms|, so R = 1 is a proof, not a fit.
  upsample2x forward: hy (hx a + lx b) + ly (hx c + lx d) rounds each term at most 4 times (its x-weight product,
                      the inner add, the y-weight product, the outer add), weights non-negative: 4u upsample(|x|)
  upsample2x backward: a sequential sum of <= 16 weighted terms plus the weight product and the multiply: 17u sum |w g|
  BatchNorm in eval mode (misc_ops.cu bn_eval_kernel), y = (x - rm) * inv * gamma + beta with inv = 1 / sqrtf(rv + eps)
                      from the call's own fp32 running statistics (family bn_eval).  inv: the add is off by u of rv + eps,
                      which the square root halves, then the square root and the divide round once each: 2.5u of inv.
                      The subtract, the multiply by inv and the multiply by gamma add u each: x^ gamma is off by at most
                      5.5u |x^ gamma| to first order; the final add rounds once more, u |y|.  The 0.5u left over covers the
                      second-order terms:  s = 6u |x^ gamma| + u |y|.  (The build keeps IEEE sqrt and divide, no
                      fast-math; a fused multiply-add only removes roundings.)

Feature warp (bilinear sample of x at (i + flow), border padding, Back2Future's normalisation).  The kernel's fp32
sample coordinate differs from the exact one by at most delta = 8u (|x + u| + W) pixels (about six roundings of
quantities of magnitude up to |x + u| + W).
  forward: delta_x max(|d out/d ix| left and right of ix) + the same for y + 6u sum |w v|
  d_x: a scatter summed in 64-bit fixed point (warp_ops.cu fx_scale): each contribution g wy wx is rounded twice in
       fp32 (2u |g w|), moves by at most |g| (delta_x + delta_y) with the coordinate, and is rounded to the fixed-point
       grid 2^-(62-e-c) with max finite |g| < 2^e, h w < 2^c: the absolute term n_i 2^(e+c-63) for the n_i
       contributions that reach element i.  The final conversion to fp32 adds u |d_x|.
  d_flow: a sum over C channels of g * d out/d ix (K = C, c_t = 4u), plus delta_y |d^2 out / d ix d iy| (the x
       derivative moves with the y weight), plus 3u |d_flow| for the scaling.  The gradient jumps where the sample
       coordinate crosses an integer, so a pixel whose fp64 coordinate lies within delta of an integer (a tie, as in
       kernel_cases.check_consensus_targets) may differ in that component; no other pixel may.

Every checked output must also meet rel_err <= 1e-4 (max |error| / max |fp64|, tests/util.rel_err), the bar of
BASELINE.json."""
import ctypes
import json
import math
import os
import statistics
import torch
import torch.nn.functional as F
from cc_b200 import nn as cnn, _lib
from oracle import nets as ON

U = 2.0 ** -24
TINY32 = 1e-44
C_TC = 12 * U
C_PROD = 4 * U
EPI = 3
REL_BAR = 1e-4

# Bound on r_i = |kernel - fp64| / s_i per op family, and the worst r measured on an H100 80GB HBM3 (700 W power limit;
# production dispatch) over all calls of the second cfg3 step at b4 256x832 (committed weight cache) with either flow net
# and of the evaluation forwards at b1 256x832 (corr441d: 3.65 in the FlowNetC6 step, 3.47 in its eval forward; bn_eval:
# 0.465), and, for the CUDA-core kernels, on the CPU simulator build over the five nets at 64x128 / 64x64 and the eval
# forwards at b1 64x128.  The runs are bit-reproducible, so these do not vary from run to run.  Caps 1 / (u K_max) at
# 256x832: 19.7 for conv / convT / bn (K = 851968), 8.7e4 for corr81, 3.8e4 for corr441d (K = 441).
R = dict(conv=10.0, convT=10.0, bn=6.0, bn_eval=1.0, upsample=1.0, corr81=6.0, corr441d=6.0, featwarp=2.0)
R_MEASURED = dict(conv=6.3, convT=5.41, bn=2.38, bn_eval=0.465, upsample=0.81, corr81=2.01, corr441d=3.65,
                  featwarp=0.37)      # H100
R_MEASURED_SIM = dict(conv=2.32, convT=2.35, bn=0.92, bn_eval=0.441, upsample=0.73, corr81=1.19, corr441d=2.42, featwarp=0.26)
FAMILIES = ('conv', 'convT', 'bn', 'bn_eval', 'upsample', 'corr81', 'corr441d', 'featwarp')
PLAN_PATHS = ('ffma', 'tc', 'tc_padded')      # ccb_debug_conv_plan's path codes

NUM_SMS, BN_CHUNK, CORR_CT, CORR_CG = 132, 8192, 16, 4      # ccb_common.cuh, misc_ops.cu, b2f_ops.cu


def f32(x):
    """A Python float as the fp32 kernel argument it becomes."""
    return float(torch.tensor(x, dtype=torch.float32))


def bn_splits(B, plane):
    """misc_ops.cu: the number of BN_CHUNK-value splits a BatchNorm channel is reduced in."""
    return (B * plane + BN_CHUNK - 1) // BN_CHUNK


def corr_chunks(B, C, h, w):
    """b2f_ops.cu corr_chunks: how many channel chunks a cost-volume launch is cut into."""
    cdiv = lambda a, b: (a + b - 1) // b      # noqa: E731
    tiles = cdiv(w, CORR_CT) * cdiv(h, CORR_CT) * B
    return max(1, min(cdiv(2 * NUM_SMS, tiles), cdiv(C, CORR_CG), 32))


def _d(t):
    return t.detach().double()


def _sq(t):
    return t * t


# ---------------------------------------------------------------------------------------------------------------------
# Per-op checks.  Each returns (checks, K_max): checks = [(what, got fp32, ref fp64, s fp64, tie mask or None)].
def _act64(z, act, slope):
    """fp64 activation, its Lipschitz factor and the rounding count of the fp32 activation."""
    if act == _lib.ACT_RELU:
        return z.clamp_min(0), 1.0, 0
    if act == _lib.ACT_LEAKY:
        return torch.where(z > 0, z, z * f32(slope)), 1.0, 1
    if act == _lib.ACT_SIGMOID:
        y = torch.sigmoid(z)
        return y, y * (1 - y), 4
    return z, 1.0, 0


def _act_bwd64(g, y, act, slope):
    """dz = g * act'(y) from the kernel's fp32 output y, as ccb_act_bwd_bias computes it; and its rounding count."""
    if act == _lib.ACT_RELU:
        return g * (y > 0), 0
    if act == _lib.ACT_LEAKY:
        return torch.where(y > 0, g, g * f32(slope)), 1
    if act == _lib.ACT_SIGMOID:
        yd = _d(y)
        return g * yd * (1 - yd), 3
    return g, 0


def _epilogue(z, s, bias, res, act, slope, y):
    mag = z.abs()
    if bias is not None:
        b = _d(bias).view(1, -1, 1, 1)
        z, mag = z + b, mag + b.abs()
    if res is not None:
        r = _d(res)
        z, mag = z + r, mag + r.abs()
    y64, L, ra = _act64(z, act, slope)
    return [('y', y, y64, L * (s + EPI * U * mag) + ra * U * y64.abs() + TINY32, None)]


def conv_fwd_checks(x, w, bias, res, stride, pad, act, slope, y):
    xd, wd = _d(x), _d(w)
    K = w.shape[1] * w.shape[2] * w.shape[3]
    z = F.conv2d(xd, wd, None, stride, pad)
    s = (U * math.sqrt(K) + C_TC) * F.conv2d(_sq(xd), _sq(wd), None, stride, pad).sqrt()
    return _epilogue(z, s, bias, res, act, slope, y), K


def conv_bwd_checks(x, w, y, g, stride, pad, act, slope, dx=None, dw=None, db=None, dres=None):
    xd, wd = _d(x), _d(w)
    dz, ra = _act_bwd64(_d(g), y, act, slope)
    B, Co, Ho, Wo = dz.shape
    k = w.shape[2]
    out, kmax = [], 0
    if dres is not None:
        out.append(('dres', dres, dz, ra * U * dz.abs() + TINY32, None))
    if dx is not None:
        K = Co * (-(-k // stride)) ** 2
        ref = torch.nn.grad.conv2d_input(x.shape, wd, dz, stride, pad)
        tn = torch.nn.grad.conv2d_input(x.shape, _sq(wd), _sq(dz), stride, pad).sqrt()
        out.append(('dx', dx, ref, (U * math.sqrt(K) + C_TC) * tn + TINY32, None))
        kmax = max(kmax, K)
    K = B * Ho * Wo
    if dw is not None:
        ref = torch.nn.grad.conv2d_weight(xd, w.shape, dz, stride, pad)
        tn = torch.nn.grad.conv2d_weight(_sq(xd), w.shape, _sq(dz), stride, pad).sqrt()
        out.append(('dw', dw, ref, (U * math.sqrt(K) + C_TC) * tn + TINY32, None))
        kmax = max(kmax, K)
    if db is not None:
        out.append(('db', db, dz.sum((0, 2, 3)), (U * math.sqrt(K) + C_PROD) * _sq(dz).sum((0, 2, 3)).sqrt() + TINY32, None))
        kmax = max(kmax, K)
    return out, kmax


def convT_fwd_checks(x, w, bias, stride, pad, out_pad, act, slope, y):
    xd, wd = _d(x), _d(w)
    K = w.shape[0] * (-(-w.shape[2] // stride)) ** 2
    z = F.conv_transpose2d(xd, wd, None, stride, pad, out_pad)
    s = (U * math.sqrt(K) + C_TC) * F.conv_transpose2d(_sq(xd), _sq(wd), None, stride, pad, out_pad).sqrt()
    return _epilogue(z, s, bias, None, act, slope, y), K


def convT_bwd_checks(x, w, y, g, stride, pad, act, slope, dx=None, dw=None, db=None):
    """ConvTranspose2d backward: dx is a conv2d of dz (fprop kernel), dw the conv weight gradient with the roles of
    activations and gradients swapped."""
    xd, wd = _d(x), _d(w)
    dz, _ = _act_bwd64(_d(g), y, act, slope)
    out, kmax = [], 0
    if dx is not None:
        K = w.shape[1] * w.shape[2] * w.shape[3]
        ref = F.conv2d(dz, wd, None, stride, pad)
        tn = F.conv2d(_sq(dz), _sq(wd), None, stride, pad).sqrt()
        out.append(('dx', dx, ref, (U * math.sqrt(K) + C_TC) * tn + TINY32, None))
        kmax = K
    if dw is not None:
        K = x.shape[0] * x.shape[2] * x.shape[3]
        ref = torch.nn.grad.conv2d_weight(dz, w.shape, xd, stride, pad)
        tn = torch.nn.grad.conv2d_weight(_sq(dz), w.shape, _sq(xd), stride, pad).sqrt()
        out.append(('dw', dw, ref, (U * math.sqrt(K) + C_TC) * tn + TINY32, None))
        kmax = max(kmax, K)
    if db is not None:
        K = dz.shape[0] * dz.shape[2] * dz.shape[3]
        out.append(('db', db, dz.sum((0, 2, 3)), (U * math.sqrt(K) + C_PROD) * _sq(dz).sum((0, 2, 3)).sqrt() + TINY32, None))
        kmax = max(kmax, K)
    return out, kmax


def bn_fwd_checks(x, gamma, beta, rm_old, rv_old, rm_new, rv_new, stats, y, eps, momentum):
    """Training-mode BatchNorm forward: saved statistics (mean, invstd) and running statistics against fp64 of x;
    y against fp64 of the elementwise apply given the saved statistics."""
    xd = _d(x)
    B, C, h, w = x.shape
    N = B * h * w
    eps, mom = f32(eps), f32(momentum)
    mean = xd.mean((0, 2, 3))
    q = _sq(xd - mean.view(1, -1, 1, 1))
    var = q.mean((0, 2, 3))
    inv = 1 / (var + eps).sqrt()
    s_mean = U * _sq(xd).mean((0, 2, 3)).sqrt() + U * mean.abs() + TINY32
    s_var = U * _sq(q).mean((0, 2, 3)).sqrt() + 2 * U * var + TINY32
    s_inv = inv * (s_var / (2 * (var + eps)) + 3 * U) + TINY32
    out = [('mean', stats[:, 0], mean, s_mean, None), ('invstd', stats[:, 1], inv, s_inv, None)]
    if rm_new is not None:
        rmo, rvo = _d(rm_old), _d(rv_old)
        unb = N / (N - 1) if N > 1 else 1.0
        out.append(('running_mean', rm_new, (1 - mom) * rmo + mom * mean,
                    mom * s_mean + 3 * U * ((1 - mom) * rmo.abs() + mom * mean.abs()) + TINY32, None))
        out.append(('running_var', rv_new, (1 - mom) * rvo + mom * var * unb,
                    mom * unb * s_var + 4 * U * ((1 - mom) * rvo.abs() + mom * unb * var) + TINY32, None))
    mk, ik = _d(stats[:, 0]).view(1, -1, 1, 1), _d(stats[:, 1]).view(1, -1, 1, 1)
    xhg = (xd - mk) * ik * _d(gamma).view(1, -1, 1, 1)
    b = _d(beta).view(1, -1, 1, 1)
    out.append(('y', y, xhg + b, 4 * U * (xhg.abs() + b.abs()) + TINY32, None))
    return out, N


def bn_eval_checks(x, gamma, beta, rm, rv, y, eps):
    """Eval-mode BatchNorm: y against fp64 of (x - rm) / sqrt(rv + eps) gamma + beta from the call's fp32 running
    statistics (module docstring: 6u |x^ gamma| + u |y|).  Elementwise: K = 1."""
    v = lambda t: _d(t).view(1, -1, 1, 1)      # noqa: E731
    xhg = (_d(x) - v(rm)) / (v(rv) + f32(eps)).sqrt() * v(gamma)
    ref = xhg + v(beta)
    return [('y', y, ref, 6 * U * xhg.abs() + U * ref.abs() + TINY32, None)], 1


def bn_bwd_checks(x, gamma, stats, g, dx=None, dgamma=None, dbeta=None):
    xd, gd = _d(x), _d(g)
    B, C, h, w = x.shape
    N = B * h * w
    mk, ik = _d(stats[:, 0]).view(1, -1, 1, 1), _d(stats[:, 1]).view(1, -1, 1, 1)
    xh = (xd - mk) * ik
    db = gd.sum((0, 2, 3))
    t = gd * xh
    dg = t.sum((0, 2, 3))
    s_db = U * math.sqrt(N) * _sq(gd).sum((0, 2, 3)).sqrt() + TINY32
    s_dg = (U * math.sqrt(N) + C_PROD) * _sq(t).sum((0, 2, 3)).sqrt() + TINY32
    out = []
    if dbeta is not None:
        out.append(('dbeta', dbeta, db, s_db, None))
    if dgamma is not None:
        out.append(('dgamma', dgamma, dg, s_dg, None))
    if dx is not None:
        gi = (_d(gamma).view(1, -1, 1, 1) * ik).abs()
        a, c = (db / N).view(1, -1, 1, 1), (dg / N).view(1, -1, 1, 1)
        ref = _d(gamma).view(1, -1, 1, 1) * ik * (gd - a - xh * c)
        s = gi * ((s_db / N).view(1, -1, 1, 1) + xh.abs() * (s_dg / N).view(1, -1, 1, 1)) + \
            6 * U * gi * (gd.abs() + a.abs() + (xh * c).abs()) + TINY32
        out.append(('dx', dx, ref, s, None))
    return out, N


def upsample_fwd_checks(x, y):
    xd = _d(x)
    up = lambda t: F.interpolate(t, scale_factor=2, mode='bilinear', align_corners=False)     # noqa: E731
    return [('y', y, up(xd), 4 * U * up(xd.abs()) + TINY32, None)], 4


def upsample_bwd_checks(g, in_shape, dx):
    gd = _d(g)
    adj = lambda t: torch.ops.aten.upsample_bilinear2d_backward(t, list(t.shape[2:]), list(in_shape), False)   # noqa: E731
    return [('dx', dx, adj(gd), 17 * U * adj(gd.abs()) + TINY32, None)], 16


def _corr_nat(f1, f2):
    """sum_c f1[c](y, x) f2[c](y + i - 4, x + j - 4) in natural displacement order k = 9 i + j (no 1/C)."""
    B, C, h, w = f1.shape
    f2p = F.pad(f2, (4, 4, 4, 4))
    return torch.stack([(f1 * f2p[:, :, i:i + h, j:j + w]).sum(1) for i in range(9) for j in range(9)], 1)


def _corr_adj(Gn, f1, f2):
    """Adjoint of _corr_nat for the natural-order gradient Gn: (d f1, d f2), no 1/C."""
    B, C, h, w = f1.shape
    f2p = F.pad(f2, (4, 4, 4, 4))
    d1 = torch.zeros_like(f1)
    d2p = torch.zeros_like(f2p)
    for k in range(81):
        i, j = divmod(k, 9)
        gk = Gn[:, k:k + 1]
        d1 += gk * f2p[:, :, i:i + h, j:j + w]
        d2p[:, :, i:i + h, j:j + w] += gk * f1
    return d1, d2p[:, :, 4:4 + h, 4:4 + w]


def _corr_idx(rev, device):
    return torch.tensor(ON.IDX_BWD if rev else ON.IDX_FWD, device=device)


def corr81_fwd_checks(f1, f2, rev, out):
    C = f1.shape[1]
    idx = _corr_idx(rev, f1.device)
    a, b = _d(f1), _d(f2)
    ref = _corr_nat(a, b)[:, idx] / C
    tn = _corr_nat(_sq(a), _sq(b))[:, idx].sqrt() / C
    return [('out', out, ref, (U * math.sqrt(C) + C_PROD) * tn + 2 * U * ref.abs() + TINY32, None)], C


def corr81_bwd_checks(f1, f2, rev, g, d1=None, d2=None):
    C = f1.shape[1]
    idx = _corr_idx(rev, f1.device)
    a, b, gd = _d(f1), _d(f2), _d(g)
    Gn = torch.empty_like(gd)
    Gn[:, idx] = gd
    r1, r2 = _corr_adj(Gn, a, b)
    t1, t2 = _corr_adj(_sq(Gn), _sq(a), _sq(b))
    out = []
    for what, got, ref, tn in (('d_f1', d1, r1, t1), ('d_f2', d2, r2, t2)):
        if got is not None:
            ref = ref / C
            out.append((what, got, ref, (U * 9 + C_PROD) * tn.sqrt() / C + 2 * U * ref.abs() + TINY32, None))
    return out, 81


# ---- FlowNetC6's dilated cost volume ---------------------------------------------------------------------------------
CORR441D_N, CORR441D_R = 21, 20          # displacements per axis, reach in pixels (10 steps of 2)
CORR441D_SLOPE32 = f32(0.1)              # the fused LeakyReLU's slope as the kernel holds it


def corr441d_sample(a, b):
    """The restated third-party correlation at FlowNetC6's call (patch 21, dilation 2) as [B,441,h,w], not divided by C."""
    B, _, h, w = a.shape
    return ON.spatial_correlation_sample(a, b, patch=CORR441D_N, dilation=2).reshape(B, CORR441D_N ** 2, h, w)


def corr441d_adjoint(G, f1, f2):
    """(sum_k G_k f2(. + d_k), sum_k G_k(. - d_k) f1(. - d_k)) over the 441 displacements d_k, no 1/C."""
    B, C, h, w = f1.shape
    N, R_ = CORR441D_N, CORR441D_R
    f2p = F.pad(f2, (R_, R_, R_, R_))
    d1 = torch.zeros_like(f1)
    d2p = torch.zeros_like(f2p)
    for i in range(N):
        for j in range(N):
            gk = G[:, N * i + j:N * i + j + 1]
            sl = (slice(None), slice(None), slice(2 * i, 2 * i + h), slice(2 * j, 2 * j + w))
            d1 += gk * f2p[sl]
            d2p[sl] += gk * f1
    return d1, d2p[:, :, R_:R_ + h, R_:R_ + w]


def corr441d_fwd_checks(f1, f2, out):
    """The pre-activation z recovered from the kernel's output against fp64 (module docstring); K = C."""
    C = f1.shape[1]
    a, b = _d(f1), _d(f2)
    z = corr441d_sample(a, b) / C
    tn = corr441d_sample(_sq(a), _sq(b)).sqrt() / C
    o = _d(out)
    zk = torch.where(o > 0, o, o / CORR441D_SLOPE32)
    return [('z', zk, z, (U * math.sqrt(C) + C_PROD) * tn + 3 * U * z.abs() + TINY32, None)], C


def corr441d_bwd_checks(f1, f2, out, g, d1=None, d2=None):
    """d f1 and d f2 against fp64 (module docstring); K = 441."""
    C = f1.shape[1]
    a, b, gd = _d(f1), _d(f2), _d(g)
    dz = torch.where(out > 0, gd, gd * CORR441D_SLOPE32)
    r1, r2 = corr441d_adjoint(dz, a, b)
    t1, t2 = corr441d_adjoint(_sq(dz), _sq(a), _sq(b))
    checks = []
    for what, got, ref, tn in (('d_f1', d1, r1, t1), ('d_f2', d2, r2, t2)):
        if got is not None:
            ref = ref / C
            checks.append((what, got, ref, (U * CORR441D_N + C_PROD) * tn.sqrt() / C + 2 * U * ref.abs() + TINY32, None))
    return checks, CORR441D_N ** 2


# ---- feature warp ---------------------------------------------------------------------------------------------------
def _warp_coords(flo, h, w):
    """fp64 sample coordinates of Model.warp (grid_sample border, align_corners=False) from the fp32 flow, before the
    border clamp, and the bound delta on the kernel's fp32 coordinate error (pixels)."""
    fl = _d(flo)
    xs = torch.arange(w, dtype=torch.float64, device=flo.device).view(1, 1, w)
    ys = torch.arange(h, dtype=torch.float64, device=flo.device).view(1, h, 1)
    ax, ay = xs + fl[:, 0], ys + fl[:, 1]
    ix = (2 * ax / max(w - 1, 1) - 1 + 1) * (0.5 * w) - 0.5
    iy = (2 * ay / max(h - 1, 1) - 1 + 1) * (0.5 * h) - 0.5
    return ix, iy, 8 * U * (ax.abs() + w), 8 * U * (ay.abs() + h)


class _Samp:
    """Bilinear sample positions at (ix, iy) after the border clamp (geom.cuh make_samp)."""

    def __init__(self, ix, iy, h, w):
        self.gx = torch.where((ix >= 0) & (ix <= w - 1), 0.5 * w, 0.0)
        self.gy = torch.where((iy >= 0) & (iy <= h - 1), 0.5 * h, 0.0)
        ix, iy = ix.clamp(0, w - 1), iy.clamp(0, h - 1)
        x0, y0 = ix.floor(), iy.floor()
        self.wx1, self.wy1 = ix - x0, iy - y0
        self.wx0, self.wy0 = 1 - self.wx1, 1 - self.wy1
        x0, y0 = x0.long(), y0.long()
        self.idx, self.ok = [], []
        for dy in (0, 1):
            for dx in (0, 1):
                ok = (x0 + dx < w) & (y0 + dy < h)
                self.ok.append(ok)
                self.idx.append(torch.where(ok, (y0 + dy) * w + x0 + dx, 0).flatten(1))     # [B, hw]
        self.w = [self.wy0 * self.wx0, self.wy0 * self.wx1, self.wy1 * self.wx0, self.wy1 * self.wx1]

    def corners(self, v):
        """v [B, C, h, w] -> the four corner values [B, C, h, w] (0 where the corner is outside)."""
        B, C, h, w = v.shape
        vf = v.reshape(B, C, h * w)
        return [torch.gather(vf, 2, i.unsqueeze(1).expand(B, C, h * w)).view(B, C, h, w) * ok.unsqueeze(1)
                for i, ok in zip(self.idx, self.ok)]

    def scatter(self, vals):
        """vals: four [B, C, h, w] contributions (one per corner) -> their sum at the corner pixels."""
        B, C, h, w = vals[0].shape
        out = torch.zeros(B, C, h * w, dtype=vals[0].dtype, device=vals[0].device)
        for v, i, ok in zip(vals, self.idx, self.ok):
            out.scatter_add_(2, i.unsqueeze(1).expand(B, C, h * w), (v * ok.unsqueeze(1)).reshape(B, C, h * w))
        return out.view(B, C, h, w)

    def dx(self, c):
        return (c[1] - c[0]) * self.wy0.unsqueeze(1) + (c[3] - c[2]) * self.wy1.unsqueeze(1)

    def dy(self, c):
        return (c[2] - c[0]) * self.wx0.unsqueeze(1) + (c[3] - c[1]) * self.wx1.unsqueeze(1)


def featwarp_fwd_checks(x, flo, out):
    B, C, h, w = x.shape
    xd = _d(x)
    ix, iy, dlx, dly = _warp_coords(flo, h, w)
    sp = _Samp(ix, iy, h, w)
    c = sp.corners(xd)
    wts = [t.unsqueeze(1) for t in sp.w]
    ref = sum(wq * cq for wq, cq in zip(wts, c))
    lx = torch.maximum(*[_Samp(ix + d * dlx, iy, h, w).dx(_Samp(ix + d * dlx, iy, h, w).corners(xd)).abs() for d in (-1, 1)])
    ly = torch.maximum(*[_Samp(ix, iy + d * dly, h, w).dy(_Samp(ix, iy + d * dly, h, w).corners(xd)).abs() for d in (-1, 1)])
    s = dlx.unsqueeze(1) * lx + dly.unsqueeze(1) * ly + 6 * U * sum(wq * cq.abs() for wq, cq in zip(wts, c)) + TINY32
    return [('out', out, ref, s, None)], 4


def fx_resolution(g, h, w):
    """warp_ops.cu fx_scale: the fixed-point grid of the image-gradient scatter is 2^-(62-e-c), max finite |g| < 2^e,
    h*w < 2^c; rounding one contribution to it is off by at most half a step, 2^(e+c-63)."""
    a = g.detach().abs()
    gmax = float(a[torch.isfinite(a)].max()) if bool(torch.isfinite(a).any()) else 0.0
    if not gmax > 0:
        return 0.0
    e = math.frexp(f32(gmax))[1]              # gmax = m 2^E, m in [0.5, 1): ilogbf(gmax) + 1 = E
    c = (h * w).bit_length()
    return 2.0 ** (e + c - 63)


def featwarp_bwd_checks(x, flo, g, dx=None, dflow=None):
    B, C, h, w = x.shape
    xd, gd = _d(x), _d(g)
    ix, iy, dlx, dly = _warp_coords(flo, h, w)
    sp = _Samp(ix, iy, h, w)
    out, extra = [], {}
    if dx is not None:
        wts = [t.unsqueeze(1) for t in sp.w]
        ref = sp.scatter([gd * wq for wq in wts])
        absum = sp.scatter([gd.abs() * wq for wq in wts])
        moved = sp.scatter([gd.abs() * (dlx + dly).unsqueeze(1)] * 4)
        n = sp.scatter([torch.ones_like(gd[:, :1])] * 4)                       # contributions per source pixel
        fx = n * fx_resolution(g, h, w)
        extra['fx_term_max'] = float(fx.max())
        out.append(('d_x', dx, ref, 2 * U * absum + moved + fx + U * ref.abs() + TINY32, None))
    if dflow is not None:
        c = sp.corners(xd)
        cross = (c[3] - c[2] - c[1] + c[0]).abs()
        res = []
        for comp, dfun, gm, ext, dl_other, coord, dl in ((0, sp.dx, sp.gx, w, dly, ix, dlx), (1, sp.dy, sp.gy, h, dlx, iy, dly)):
            t = gd * dfun(c)
            sc = gm * (2.0 / max(ext - 1, 1))
            ref = t.sum(1) * sc
            lin = ((c[1] - c[0]).abs() * sp.wy0.unsqueeze(1) + (c[3] - c[2]).abs() * sp.wy1.unsqueeze(1)) if comp == 0 else \
                ((c[2] - c[0]).abs() * sp.wx0.unsqueeze(1) + (c[3] - c[1]).abs() * sp.wx1.unsqueeze(1))
            s = sc * ((U * math.sqrt(C) + C_PROD) * _sq(t).sum(1).sqrt() + 4 * U * (gd.abs() * lin).sum(1) +
                      dl_other * (gd.abs() * cross).sum(1)) + 3 * U * ref.abs() + TINY32
            tie = (coord - coord.round()).abs() <= dl
            res.append((ref, s, tie))
        ref = torch.stack([r[0] for r in res], 1)
        s = torch.stack([r[1] for r in res], 1)
        tie = torch.stack([r[2] for r in res], 1)
        extra['ties'] = int(tie.sum())
        out.append(('d_flow', dflow, ref, s, tie))
    return out, C, extra


# ---------------------------------------------------------------------------------------------------------------------
def measure(got, ref, s, tie=None):
    """(worst r, rel_err, number of tie elements excluded): r = |got - ref| / s over the non-tie elements."""
    d = (_d(got) - ref).abs()
    r = torch.nan_to_num(d / s, nan=float('inf'))
    if tie is not None:
        r = r.masked_fill(tie, 0.0)
        d = d.masked_fill(tie, 0.0)
    rmax = float(r.max()) if r.numel() else 0.0
    rel = float(torch.nan_to_num(d, nan=float('inf')).max()) / max(float(ref.abs().max()), 1e-30) if d.numel() else 0.0
    return rmax, rel, int(tie.sum()) if tie is not None else 0


def evaluate(op, checks, R=R):
    """checks of one call -> {what: (r, rel, ties)}, worst r, and the list of failures against R[op] / REL_BAR (R: the
    bound table of the audit the call belongs to)."""
    res, bad = {}, []
    for what, got, ref, s, tie in checks:
        assert got.shape == ref.shape, (op, what, tuple(got.shape), tuple(ref.shape))
        r, rel, nt = measure(got, ref, s, tie)
        res[what] = (r, rel, nt)
        if not r <= R[op]:
            bad.append('%s r %.3g > R %.3g' % (what, r, R[op]))
        if not rel <= REL_BAR:
            bad.append('%s rel_err %.3g > %.0e' % (what, rel, REL_BAR))
    return res, max([v[0] for v in res.values()] or [0.0]), bad


def assert_conv_within_bound(kind, x, w, stride, pad, bias=None, res=None, out_pad=0, act=None, slope=0.0, y=None, g=None,
                             dx=None, dw=None, db=None, dres=None, what=''):
    """One convolution (kind 'conv') or ConvTranspose2d (kind 'convT') call held element by element to the audit's
    bound: the forward output y with its bias / residual / activation epilogue, and, given the upstream gradient g of y,
    the gradients dx, dw, db (and dres) that were computed - the checks conv_fwd_checks / conv_bwd_checks (convT_*)
    build, evaluated against R[kind] and REL_BAR.  act: an _lib.ACT_* code or its cc_b200.nn name (None, 'relu',
    'leaky', 'sigmoid'); the backward differentiates it at y, so y is needed with an activation.  Unlike rel_err
    against the largest |fp64| of the whole tensor, the bound scales with each element's own products: a k-stage that
    lost its tf32 lo terms stands out at r = 20-230 where rel_err still reads 3e-5 to 1e-4 (tests/test_layer_audit.py).
    Returns {check: worst r}."""
    act = act if isinstance(act, int) else cnn.ACT[act]
    checks = []
    if kind == 'conv':
        if y is not None:
            checks += conv_fwd_checks(x, w, bias, res, stride, pad, act, slope, y)[0]
        if g is not None:
            checks += conv_bwd_checks(x, w, y, g, stride, pad, act, slope, dx=dx, dw=dw, db=db, dres=dres)[0]
    else:
        assert kind == 'convT' and res is None and dres is None, kind
        if y is not None:
            checks += convT_fwd_checks(x, w, bias, stride, pad, out_pad, act, slope, y)[0]
        if g is not None:
            checks += convT_bwd_checks(x, w, y, g, stride, pad, act, slope, dx=dx, dw=dw, db=db)[0]
    assert checks, (kind, what, 'nothing to check')
    out, _, bad = evaluate(kind, checks)
    assert not bad, '%s %s over the bound (R = %.3g): %s' % (kind, what, R[kind], '; '.join(bad))
    return {k: v[0] for k, v in out.items()}


class LayerAudit:
    """with LayerAudit(nets={'disp': net, ...}) as audit: ... run forward / backward ...  (see the module docstring)"""

    FNS = {'conv': '_Conv2dFn', 'convT': '_ConvT2dFn', 'bn': '_BatchNormFn', 'upsample': '_Upsample2xFn',
           'corr81': '_Corr81Fn', 'corr441d': '_Corr441dFn', 'featwarp': '_FeatWarpFn'}

    def __init__(self, nets=None, tag='audit', report=True):
        self.nets = dict(nets or {})
        self.tag, self.report = tag, report
        self.rows = []
        self._stack, self._hooks, self._kern, self._count = [], [], [], {}
        self._saved = None

    # ---- patching -------------------------------------------------------------------------------------------------
    def __enter__(self):
        self._saved = {fam: (getattr(cnn, cls).__dict__['forward'], getattr(cnn, cls).__dict__['backward'])
                       for fam, cls in self.FNS.items()}
        self._saved_run = cnn._run
        try:
            for prefix, net in self.nets.items():
                for name, m in net.named_modules():
                    full = prefix + ('.' + name if name else '')
                    self._hooks.append(m.register_forward_pre_hook(lambda mod, a, full=full: self._stack.append(full)))
                    self._hooks.append(m.register_forward_hook(lambda mod, a, o: self._stack.pop() and None))
            cnn._run = self._run
            for fam, cls in self.FNS.items():
                f, b = self._saved[fam]
                setattr(getattr(cnn, cls), 'forward', staticmethod(self._wrap_fwd(fam, f.__func__)))
                setattr(getattr(cnn, cls), 'backward', staticmethod(self._wrap_bwd(fam, b.__func__)))
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
            for fam, cls in self.FNS.items():
                setattr(getattr(cnn, cls), 'forward', self._saved[fam][0])
                setattr(getattr(cnn, cls), 'backward', self._saved[fam][1])
            cnn._run = self._saved_run
        for h in self._hooks:
            h.remove()
        self._hooks, self._stack = [], []

    def _run(self, op, d, *args):
        self._saved_run(op, d, *args)
        k = _lib.lib().ccb_debug_last_conv_kernel()
        plan = (ctypes.c_int * 2)()
        _lib.call('ccb_debug_conv_plan', d, op, plan)
        call = ('fprop', 'dgrad', 'wgrad')[op]
        self._kern.append(('%s:%s' % ((k or b'?').decode(), call), dict(call=call, path=PLAN_PATHS[plan[0]], splits=plan[1])))

    def _name(self, fam):
        top = self._stack[-1] if self._stack else ''
        if fam in ('conv', 'convT', 'bn'):
            return top
        n = self._count.get((top, fam), 0)
        self._count[(top, fam)] = n + 1
        return '%s:%s#%d' % (top, fam, n)

    def _wrap_fwd(self, fam, orig):
        audit = self

        def forward(ctx, *args):
            k0 = len(audit._kern)
            before = (args[3].clone(), args[4].clone()) if fam == 'bn' and args[5] else None      # running stats
            kept, save = [], ctx.save_for_backward          # what the forward saves (BatchNorm: its statistics)
            ctx.save_for_backward = lambda *t: (kept.extend(t), save(*t))
            try:
                out = orig(ctx, *args)
            finally:
                del ctx.save_for_backward
            ctx._audit_name = audit._name(fam)
            with torch.no_grad():
                audit._fwd(fam, ctx, args, out, before, kept, audit._kern[k0:])
            return out
        return forward

    def _wrap_bwd(self, fam, orig):
        audit = self

        def backward(ctx, g):
            saved = ctx.saved_tensors
            k0 = len(audit._kern)
            grads = orig(ctx, g)
            with torch.no_grad():
                audit._bwd(fam, ctx, saved, g, grads, audit._kern[k0:])
            return grads
        return backward

    # ---- checks of one call ---------------------------------------------------------------------------------------
    @staticmethod
    def _param_grad(ctx, i, returned):
        """A parameter gradient the backward returned, or - written straight into the optimiser's flat buffer - the
        slot it wrote; None when it was not computed."""
        if returned is not None or not ctx.needs_input_grad[i]:
            return returned
        p = ctx.params[i - 1] if hasattr(ctx, 'params') else None
        return getattr(p, '_ccb_grad', None)

    def _fwd(self, fam, ctx, a, out, before, kept, kern):
        extra = {}
        if fam == 'conv':
            x, w, bias, res, stride, pad, act, slope = a
            checks, K = conv_fwd_checks(x, w, bias, res, stride, pad, act, slope, out)
            shape = tuple(x.shape) + (w.shape[0], w.shape[2], stride)
        elif fam == 'convT':
            x, w, bias, stride, pad, op, act, slope = a
            checks, K = convT_fwd_checks(x, w, bias, stride, pad, op, act, slope, out)
            shape = tuple(x.shape) + (w.shape[1], w.shape[2], stride)
        elif fam == 'bn':
            x, gamma, beta, rm, rv, training, eps, momentum = a
            shape = tuple(x.shape)
            if training:
                checks, K = bn_fwd_checks(x, gamma, beta, before[0], before[1], rm, rv, kept[2], out, eps, momentum)
                extra['splits'] = bn_splits(x.shape[0], x.shape[2] * x.shape[3])
            else:
                fam = 'bn_eval'
                checks, K = bn_eval_checks(x, gamma, beta, rm, rv, out, eps)
        elif fam == 'upsample':
            checks, K = upsample_fwd_checks(a[0], out)
            shape = tuple(a[0].shape)
        elif fam == 'corr81':
            f1, f2, rev = a
            checks, K = corr81_fwd_checks(f1, f2, bool(rev), out)
            shape = tuple(f1.shape)
            extra['chunks'] = corr_chunks(*f1.shape)
        elif fam == 'corr441d':
            checks, K = corr441d_fwd_checks(a[0], a[1], out)
            shape = tuple(a[0].shape)
        else:
            checks, K = featwarp_fwd_checks(a[0], a[1], out)
            shape = tuple(a[0].shape)
        self._record(fam, ctx._audit_name, 'fwd', shape, kern, checks, K, extra)

    def _bwd(self, fam, ctx, saved, g, grads, kern):
        extra = {}
        name = getattr(ctx, '_audit_name', '?')
        if fam == 'conv':
            x, w, y = saved
            stride, pad, act, slope, has_bias, has_res = ctx.cfg
            dw, db = self._param_grad(ctx, 1, grads[1]), (self._param_grad(ctx, 2, grads[2]) if has_bias else None)
            checks, K = conv_bwd_checks(x, w, y, g, stride, pad, act, slope, dx=grads[0], dw=dw, db=db,
                                        dres=grads[3] if has_res else None)
            shape = tuple(x.shape) + (w.shape[0], w.shape[2], stride)
        elif fam == 'convT':
            x, w, y = saved
            stride, pad, act, slope, has_bias, H, W = ctx.cfg
            dw, db = self._param_grad(ctx, 1, grads[1]), (self._param_grad(ctx, 2, grads[2]) if has_bias else None)
            checks, K = convT_bwd_checks(x, w, y, g, stride, pad, act, slope, dx=grads[0], dw=dw, db=db)
            shape = tuple(x.shape) + (w.shape[1], w.shape[2], stride)
        elif fam == 'bn':
            x, gamma, stats = saved
            checks, K = bn_bwd_checks(x, gamma, stats, g, dx=grads[0], dgamma=self._param_grad(ctx, 1, grads[1]),
                                      dbeta=self._param_grad(ctx, 2, grads[2]))
            shape = tuple(x.shape)
            extra['splits'] = bn_splits(x.shape[0], x.shape[2] * x.shape[3])
        elif fam == 'upsample':
            checks, K = upsample_bwd_checks(g, ctx.shape, grads)
            shape = tuple(ctx.shape)
        elif fam == 'corr81':
            f1, f2 = saved
            checks, K = corr81_bwd_checks(f1, f2, bool(ctx.rev), g, d1=grads[0], d2=grads[1])
            shape = tuple(f1.shape)
            extra['chunks'] = corr_chunks(*f1.shape)
        elif fam == 'corr441d':
            f1, f2, out = saved
            checks, K = corr441d_bwd_checks(f1, f2, out, g, d1=grads[0], d2=grads[1])
            shape = tuple(f1.shape)
        else:
            x, flo = saved
            checks, K, extra = featwarp_bwd_checks(x, flo, g, dx=grads[0], dflow=grads[1])
            shape = tuple(x.shape)
        self._record(fam, name, 'bwd', shape, kern, checks, K, extra)

    def _record(self, fam, name, phase, shape, kern, checks, K, extra):
        res, r, bad = evaluate(fam, checks)
        row = dict(op=fam, name=name, phase=phase, shape=list(shape), kernels=sorted({k for k, _ in kern}), K=K, r=r,
                   checks={k: dict(r=v[0], rel=v[1], ties=v[2]) for k, v in res.items()}, bad=bad)
        if kern:
            row['plans'] = [p for _, p in kern]
        row.update(extra)
        self.rows.append(row)

    # ---- report ---------------------------------------------------------------------------------------------------
    def summary(self):
        fams = {}
        for row in self.rows:
            fams.setdefault(row['op'], []).append(row)
        out = {}
        for fam, rows in fams.items():
            rs = [row['r'] for row in rows]
            out[fam] = dict(calls=len(rows), r_max=max(rs), r_median=statistics.median(rs), R=R[fam],
                            K_max=max(row['K'] for row in rows),
                            rel_max=max(c['rel'] for row in rows for c in row['checks'].values()),
                            kernels=sorted({k for row in rows for k in row['kernels']}))
        return out

    def finish(self):
        summ = self.summary()
        if self.report:
            print('\n== layer audit %s: %d calls' % (self.tag, len(self.rows)))
            print('   %-9s %6s %10s %10s %6s %9s %10s  kernels' % ('op', 'calls', 'r worst', 'r median', 'R', 'K max', 'rel max'))
            for fam in FAMILIES:
                if fam in summ:
                    d = summ[fam]
                    print('   %-9s %6d %10.3g %10.3g %6.3g %9d %10.2e  %s' % (fam, d['calls'], d['r_max'], d['r_median'], d['R'],
                                                                        d['K_max'], d['rel_max'], ' '.join(d['kernels'])))
            out = os.environ.get('CCB_PARITY_REPORT_DIR')
            if out:
                os.makedirs(out, exist_ok=True)
                with open(os.path.join(out, 'layer_audit_%s.json' % self.tag), 'w') as f:
                    json.dump(dict(summary=summ, R=R, rows=self.rows), f, indent=1)
        bad = ['%s %s %s %s: %s' % (row['op'], row['phase'], row['name'], row['shape'], '; '.join(row['bad']))
               for row in self.rows if row['bad']]
        for fam, d in summ.items():
            if fam != 'upsample' and not R[fam] < 1 / (U * d['K_max']):
                bad.append('%s: R %.3g does not leave one dropped term detectable at K = %d (needs R < %.3g)' % (
                    fam, R[fam], d['K_max'], 1 / (U * d['K_max'])))
        assert not bad, '%d layer calls over their bound:\n  ' % len(bad) + '\n  '.join(bad[:60])
        return summ
