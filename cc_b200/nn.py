"""Layer primitives of the four networks on the libccb200 kernels: Conv2d / ConvTranspose2d with fused
bias + residual + activation epilogues, BatchNorm2d, bilinear x2 upsampling - each a
torch.autograd.Function over hand-written forward / data-gradient / weight-gradient kernels.

Parameter names and shapes equal torch's nn.Conv2d / nn.ConvTranspose2d / nn.BatchNorm2d, so the
reference's checkpoints (utils.py:55-63) load unchanged.  No cuDNN / ATen compute on this path."""
import ctypes as C
import math
import torch
from torch import nn
from . import _lib

ACT = {None: _lib.ACT_NONE, 'none': _lib.ACT_NONE, 'relu': _lib.ACT_RELU, 'leaky': _lib.ACT_LEAKY,
       'sigmoid': _lib.ACT_SIGMOID}
CONV_IMPL = _lib.IMPL_AUTO          # tests flip this to force the FFMA or the tensor-core path

_WORK = {}
_WORK_RETIRED = []          # outgrown buffers a captured CUDA graph may still point into: kept alive, never reused
GRAPH_LIVE = False          # set by Trainer.capture(): from then on an outgrown workspace is retired, not freed


def _workspace(dev, floats):
    """One grow-only scratch buffer per device (split-K partials, prepared weights); stream-ordered reuse.
    The raw pointer is baked into captured CUDA graphs, so once a graph exists an outgrown buffer is parked in
    _WORK_RETIRED instead of going back to the caching allocator (a replay would otherwise write into freed memory)."""
    if floats <= 0:
        return None, 0
    buf = _WORK.get(dev)
    if buf is None or buf.numel() < floats:
        if buf is not None and GRAPH_LIVE:
            _WORK_RETIRED.append(buf)
        buf = torch.empty(int(floats), device=dev, dtype=torch.float32)
        _WORK[dev] = buf
    return buf, buf.numel()


WCACHE = None               # handle of the weight cache conv calls use (set by Trainer.step for its own nets only)


class WeightCache:
    """Prepared (tf32 hi|lo, kernel K order) copies of the conv weights, refreshed once per optimiser step in ONE launch
    instead of once per conv call (include/ccb200.h: ccb_wcache_*).  The first step run with the cache active RECORDS
    the layouts; commit() allocates the persistent buffer; from then on conv calls skip their preparation launch.
    Owner contract: refresh() after every change of the weights."""

    def __init__(self, device):
        self.device = device
        self.h = _lib.call('ccb_wcache_create')
        self.committed = False
        self.buf = self.table = None

    def commit(self):
        floats, tbytes = _lib.call('ccb_wcache_plan_floats', self.h), _lib.call('ccb_wcache_table_bytes', self.h)
        self.buf = torch.empty(max(int(floats), 1), device=self.device, dtype=torch.float32)
        self.table = torch.empty(int(tbytes), device=self.device, dtype=torch.uint8)
        _lib.call('ccb_wcache_commit', self.h, self.buf, floats, self.table, tbytes, self.buf)
        self.committed = True
        self.refresh()

    def refresh(self):
        if self.committed:
            _lib.call('ccb_wcache_refresh', self.h, self.buf)

    def stats(self):
        out = (C.c_longlong * 4)()
        _lib.call('ccb_wcache_stats', self.h, out)
        return dict(layouts=out[0], hits=out[1], misses=out[2], committed=bool(out[3]))

    def __del__(self):
        try:
            _lib.call('ccb_wcache_destroy', self.h)
        except Exception:
            pass


def _desc(B, Ci, Hi, Wi, Co, Ho, Wo, k, stride, pad, act, slope):
    d = _lib.ConvDesc()
    d.B, d.Ci, d.Hi, d.Wi, d.Co, d.Ho, d.Wo = B, Ci, Hi, Wi, Co, Ho, Wo
    d.kh = d.kw = k
    d.stride, d.pad, d.act, d.slope, d.impl = stride, pad, act, slope, CONV_IMPL
    d.wcache = WCACHE
    return d


_CONV_OPS = ('ccb_conv2d_fprop', 'ccb_conv2d_dgrad', 'ccb_conv2d_wgrad')


def _run(op, d, *args):
    work, wf = _workspace(args[0].device, _lib.call('ccb_conv_workspace_floats', d, op))
    _lib.call(_CONV_OPS[op], d, *args, work, wf, args[0])


def _grad_slot(param, like):
    """Where a parameter gradient is written: straight into the optimiser's flat gradient buffer when
    the parameter is registered with cc_b200.optim.FlatAdam (no AccumulateGrad add), else a new tensor.
    Returns (tensor, direct)."""
    slot = getattr(param, '_ccb_grad', None) if param is not None else None
    if slot is not None and not param._ccb_written:
        param._ccb_written = True
        return slot, True
    if slot is not None:
        param._ccb_indirect = True      # second use in one backward: this gradient reaches the flat buffer through AccumulateGrad
    return torch.empty_like(like), False


def _grad_done(*params):
    """Tell the data-parallel bucket scheduler (cc_b200.dist.GradBuckets) that the kernels writing these parameters'
    gradients have been enqueued on the current stream."""
    for p in params:
        cb = getattr(p, '_ccb_bucket', None) if p is not None else None
        if cb is not None:
            cb.note(p)


def _act_bwd_bias(g, y, act, slope, db):
    """dz = g * act'(y) and (db given) db[c] = sum dz, one pass (ccb_act_bwd_bias)."""
    if act == _lib.ACT_NONE and db is None:
        return g
    B, Cc = g.shape[0], g.shape[1]
    plane = g.numel() // (B * Cc)
    dz = torch.empty_like(g) if act != _lib.ACT_NONE else g
    work, wf = _lib.workspace('ccb_act_bwd_bias_workspace_floats', B, Cc, plane, like=g) if db is not None else (None, 0)
    _lib.call('ccb_act_bwd_bias', g, y, dz if act != _lib.ACT_NONE else None, db, B, Cc, plane, act, slope, work, wf, g)
    return dz


class _Conv2dFn(torch.autograd.Function):
    """y = act(conv2d(x, w) + bias + res)"""

    @staticmethod
    def forward(ctx, x, w, bias, res, stride, pad, act, slope):
        w_in, b_in = w, bias
        x, w = _lib.f32(x), _lib.f32(w)
        bias = _lib.f32(bias) if bias is not None else None
        res = _lib.f32(res) if res is not None else None
        B, Ci, Hi, Wi = x.shape
        Co, _, k, _ = w.shape
        Ho, Wo = (Hi + 2 * pad - k) // stride + 1, (Wi + 2 * pad - k) // stride + 1
        y = torch.empty(B, Co, Ho, Wo, device=x.device, dtype=torch.float32)
        d = _desc(B, Ci, Hi, Wi, Co, Ho, Wo, k, stride, pad, act, slope)
        _run(_lib.CONV_FPROP, d, x, w, bias, res, y)
        ctx.save_for_backward(x, w, y if act != _lib.ACT_NONE else None)
        ctx.cfg = (stride, pad, act, slope, bias is not None, res is not None)
        ctx.params = (w_in, b_in)
        return y

    @staticmethod
    def backward(ctx, g):
        x, w, y = ctx.saved_tensors
        stride, pad, act, slope, has_bias, has_res = ctx.cfg
        B, Ci, Hi, Wi = x.shape
        Co, _, k, _ = w.shape
        want_w = ctx.needs_input_grad[1] or (has_bias and ctx.needs_input_grad[2])
        db, b_direct = _grad_slot(ctx.params[1], w.new_empty(Co)) if (has_bias and want_w) else (None, False)
        dz = _act_bwd_bias(_lib.f32(g), y, act, slope, db)          # activation backward + bias gradient: one pass over g
        d = _desc(B, Ci, Hi, Wi, Co, dz.shape[2], dz.shape[3], k, stride, pad, _lib.ACT_NONE, 0.0)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            _run(_lib.CONV_DGRAD, d, dz, w, None, None, dx)
        if want_w:
            dw, w_direct = _grad_slot(ctx.params[0], w)
            _run(_lib.CONV_WGRAD, d, x, dz, dw)
            _grad_done(ctx.params[0] if w_direct else None, ctx.params[1] if b_direct else None)
            dw = None if w_direct else dw
            db = None if b_direct else db
        return dx, dw, db, (dz if has_res else None), None, None, None, None


class _ConvT2dFn(torch.autograd.Function):
    """y = act(conv_transpose2d(x, w) + bias); torch weight layout [Cin, Cout, k, k].
    Forward is the data-gradient kernel of the conv (Co=Cin, Ci=Cout) - SURVEY.md K7."""

    @staticmethod
    def forward(ctx, x, w, bias, stride, pad, out_pad, act, slope):
        w_in, b_in = w, bias
        x, w = _lib.f32(x), _lib.f32(w)
        bias = _lib.f32(bias) if bias is not None else None
        B, Cin, h, wd = x.shape
        _, Cout, k, _ = w.shape
        H = (h - 1) * stride - 2 * pad + k + out_pad
        W = (wd - 1) * stride - 2 * pad + k + out_pad
        y = torch.empty(B, Cout, H, W, device=x.device, dtype=torch.float32)
        d = _desc(B, Cout, H, W, Cin, h, wd, k, stride, pad, act, slope)
        _run(_lib.CONV_DGRAD, d, x, w, bias, None, y)
        ctx.save_for_backward(x, w, y if act != _lib.ACT_NONE else None)
        ctx.cfg = (stride, pad, act, slope, bias is not None, H, W)
        ctx.params = (w_in, b_in)
        return y

    @staticmethod
    def backward(ctx, g):
        x, w, y = ctx.saved_tensors
        stride, pad, act, slope, has_bias, H, W = ctx.cfg
        B, Cin, h, wd = x.shape
        _, Cout, k, _ = w.shape
        want_b = has_bias and ctx.needs_input_grad[2]
        db, b_direct = _grad_slot(ctx.params[1], w.new_empty(Cout)) if want_b else (None, False)
        dz = _act_bwd_bias(_lib.f32(g), y, act, slope, db)
        if want_b:
            _grad_done(ctx.params[1] if b_direct else None)
            db = None if b_direct else db
        d = _desc(B, Cout, H, W, Cin, h, wd, k, stride, pad, _lib.ACT_NONE, 0.0)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            _run(_lib.CONV_FPROP, d, dz, w, None, None, dx)
        if ctx.needs_input_grad[1]:
            dw, direct = _grad_slot(ctx.params[0], w)
            _run(_lib.CONV_WGRAD, d, dz, x, dw)              # roles swapped: activations = dz, grads = x
            _grad_done(ctx.params[0] if direct else None)
            dw = None if direct else dw
        return dx, dw, db, None, None, None, None, None


class _BatchNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, rm, rv, training, eps, momentum):
        ctx.params = (gamma, beta)
        x, gamma, beta = _lib.f32(x), _lib.f32(gamma), _lib.f32(beta)
        B, Cc, h, w = x.shape
        y = torch.empty_like(x)
        stats = torch.empty(Cc, 2, device=x.device) if training else None
        work, wf = _lib.workspace('ccb_bn_workspace_floats', B, Cc, h * w, like=x) if training else (None, 0)
        _lib.call('ccb_bn_fwd', x, gamma, beta, y, stats, rm, rv, B, Cc, h * w, eps, momentum, int(training), work, wf, x)
        ctx.save_for_backward(x, gamma, stats)
        ctx.training = training
        return y

    @staticmethod
    def backward(ctx, g):
        x, gamma, stats = ctx.saved_tensors
        if not ctx.training:
            raise NotImplementedError('cc_b200: BatchNorm backward is implemented for training mode only')
        B, Cc, h, w = x.shape
        g = _lib.f32(g)
        dx = torch.empty_like(x)
        dg, g_direct = _grad_slot(ctx.params[0], gamma)
        db, b_direct = _grad_slot(ctx.params[1], gamma)
        work, wf = _lib.workspace('ccb_bn_workspace_floats', B, Cc, h * w, like=x)
        _lib.call('ccb_bn_bwd', x, g, gamma, stats, dx, dg, db, B, Cc, h * w, work, wf, x)
        _grad_done(ctx.params[0] if g_direct else None, ctx.params[1] if b_direct else None)
        return dx, (None if g_direct else dg), (None if b_direct else db), None, None, None, None, None


class _Upsample2xFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = _lib.f32(x)
        B, Cc, h, w = x.shape
        y = torch.empty(B, Cc, 2 * h, 2 * w, device=x.device, dtype=torch.float32)
        _lib.call('ccb_upsample2x_fwd', x, y, B * Cc, h, w, x)
        ctx.shape = (B, Cc, h, w)
        return y

    @staticmethod
    def backward(ctx, g):
        B, Cc, h, w = ctx.shape
        g = _lib.f32(g)
        dx = torch.empty(B, Cc, h, w, device=g.device, dtype=torch.float32)
        _lib.call('ccb_upsample2x_bwd', g, dx, B * Cc, h, w, g)
        return dx


def conv2d(x, w, bias=None, res=None, stride=1, padding=0, act=None, slope=0.0):
    return _Conv2dFn.apply(x, w, bias, res, stride, padding, ACT[act], slope)


def conv_transpose2d(x, w, bias=None, stride=1, padding=0, output_padding=0, act=None, slope=0.0):
    return _ConvT2dFn.apply(x, w, bias, stride, padding, output_padding, ACT[act], slope)


def upsample2x(x):
    """F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=False)."""
    return _Upsample2xFn.apply(x)


# -------------------------------------------------------------------------------------------------
class Conv2d(nn.Module):
    """nn.Conv2d (square kernel) + optional fused activation; parameters named like torch's."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, bias=True, act=None, slope=0.0):
        super().__init__()
        self.in_channels, self.out_channels, self.kernel_size = in_channels, out_channels, kernel_size
        self.stride, self.padding, self.act, self.slope = stride, padding, act, slope
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels, kernel_size, kernel_size))
        self.bias = nn.Parameter(torch.empty(out_channels)) if bias else None
        self.reset_parameters()

    def reset_parameters(self):           # torch's default Conv2d init
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            bound = 1 / math.sqrt(self.in_channels * self.kernel_size ** 2)
            nn.init.uniform_(self.bias, -bound, bound)

    def forward(self, x, res=None):
        return conv2d(x, self.weight, self.bias, res, self.stride, self.padding, self.act, self.slope)


class ConvTranspose2d(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, output_padding=0, bias=True,
                 act=None, slope=0.0):
        super().__init__()
        self.in_channels, self.out_channels, self.kernel_size = in_channels, out_channels, kernel_size
        self.stride, self.padding, self.output_padding, self.act, self.slope = stride, padding, output_padding, act, slope
        self.weight = nn.Parameter(torch.empty(in_channels, out_channels, kernel_size, kernel_size))
        self.bias = nn.Parameter(torch.empty(out_channels)) if bias else None
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            bound = 1 / math.sqrt(out_channels * kernel_size ** 2)
            nn.init.uniform_(self.bias, -bound, bound)

    def forward(self, x):
        return conv_transpose2d(x, self.weight, self.bias, self.stride, self.padding, self.output_padding, self.act,
                                self.slope)


class BatchNorm2d(nn.Module):
    def __init__(self, num_features, eps=1e-5, momentum=0.1):
        super().__init__()
        self.num_features, self.eps, self.momentum = num_features, eps, momentum
        self.weight = nn.Parameter(torch.ones(num_features))
        self.bias = nn.Parameter(torch.zeros(num_features))
        self.register_buffer('running_mean', torch.zeros(num_features))
        self.register_buffer('running_var', torch.ones(num_features))
        self.register_buffer('num_batches_tracked', torch.tensor(0, dtype=torch.long))

    def forward(self, x):
        if self.training:
            self.num_batches_tracked += 1
        return _BatchNormFn.apply(x, self.weight, self.bias, self.running_mean, self.running_var, self.training,
                                  self.eps, self.momentum)


class Fused(nn.Module):
    """Parameter-free placeholder for an activation module that is fused into the preceding layer's
    epilogue; it keeps nn.Sequential indices (hence state_dict keys) identical to the reference."""

    def __init__(self, what='relu'):
        super().__init__()
        self.what = what

    def forward(self, x):
        return x

    def extra_repr(self):
        return 'fused=' + self.what


def xavier_init_(module, bias_uniform=False):
    """The reference nets' init_weights(): xavier_uniform on (transposed) conv weights, zero bias
    (Back2Future: U[0,1) bias, back2future.py:106-116)."""
    for m in module.modules():
        if isinstance(m, (Conv2d, ConvTranspose2d)):
            nn.init.xavier_uniform_(m.weight.data)
            if m.bias is not None:
                if bias_uniform:
                    nn.init.uniform_(m.bias.data)
                else:
                    m.bias.data.zero_()


# -------------------------------------------------------------------------------------------------
# Back2Future operators
class _Corr81Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, f1, f2, reversed_):
        f1, f2 = _lib.f32(f1), _lib.f32(f2)
        B, Cc, h, w = f1.shape
        out = torch.empty(B, 81, h, w, device=f1.device, dtype=torch.float32)
        work, wf = _lib.workspace('ccb_corr81_fwd_workspace_floats', B, Cc, h, w, like=f1)
        _lib.call('ccb_corr81_fwd', f1, f2, out, B, Cc, h, w, int(reversed_), work, wf, f1)
        ctx.save_for_backward(f1, f2)
        ctx.rev = int(reversed_)
        return out

    @staticmethod
    def backward(ctx, g):
        f1, f2 = ctx.saved_tensors
        B, Cc, h, w = f1.shape
        g = _lib.f32(g)
        d1 = torch.empty_like(f1) if ctx.needs_input_grad[0] else None
        d2 = torch.empty_like(f2) if ctx.needs_input_grad[1] else None
        if d1 is not None or d2 is not None:
            work, wf = _lib.workspace('ccb_corr81_bwd_workspace_floats', B, Cc, h, w, like=f1) if d2 is not None else (None, 0)
            _lib.call('ccb_corr81_bwd', f1, f2, g, d1, d2, B, Cc, h, w, ctx.rev, work, wf, f1)
        return d1, d2, None


class _Corr441dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, f1, f2):
        f1, f2 = _lib.f32(f1), _lib.f32(f2)
        if f1.shape != f2.shape or f1.dim() != 4:
            raise ValueError('cc_b200: corr441d needs two [B,C,h,w] maps of one shape, got %s and %s'
                             % (tuple(f1.shape), tuple(f2.shape)))
        B, Cc, h, w = f1.shape
        out = torch.empty(B, 441, h, w, device=f1.device, dtype=torch.float32)
        _lib.call('ccb_corr441d_fwd', f1, f2, out, B, Cc, h, w, f1)
        ctx.save_for_backward(f1, f2, out)
        return out

    @staticmethod
    def backward(ctx, g):
        f1, f2, out = ctx.saved_tensors
        B, Cc, h, w = f1.shape
        g = _lib.f32(g)
        d1 = torch.empty_like(f1) if ctx.needs_input_grad[0] else None
        d2 = torch.empty_like(f2) if ctx.needs_input_grad[1] else None
        if d1 is not None or d2 is not None:
            _lib.call('ccb_corr441d_bwd', f1, f2, out, g, d1, d2, B, Cc, h, w, f1)
        return d1, d2


class _FeatWarpFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, flo):
        x, flo = _lib.f32(x), _lib.f32(flo)
        B, Cc, h, w = x.shape
        out = torch.empty_like(x)
        _lib.call('ccb_featwarp_fwd', x, flo, B, Cc, h, w, out, x)
        ctx.save_for_backward(x, flo)
        return out

    @staticmethod
    def backward(ctx, g):
        x, flo = ctx.saved_tensors
        B, Cc, h, w = x.shape
        g = _lib.f32(g)
        dx = torch.zeros_like(x) if ctx.needs_input_grad[0] else None
        df = torch.empty_like(flo) if ctx.needs_input_grad[1] else None
        work, words = _lib.scatter_workspace(x) if dx is not None else (None, 0)
        _lib.call('ccb_featwarp_bwd', x, flo, B, Cc, h, w, g, df, dx, work, words, x)
        return dx, df


def corr81(f1, f2, reversed_=False):
    """correlate(f1, f2).index_select(1, idx_fwd | idx_bwd) of back2future.py:15-25,173-176."""
    return _Corr81Fn.apply(f1, f2, reversed_)


def corr441d(f1, f2):
    """LeakyReLU(0.1)(correlate(f1, f2)) of FlowNetC6.py:18-30,111-112: the 21x21 cost volume at dilation 2, [B,441,h,w]."""
    return _Corr441dFn.apply(f1, f2)


def feat_warp(x, flo):
    """Model.warp of back2future.py:287-321."""
    return _FeatWarpFn.apply(x, flo)
