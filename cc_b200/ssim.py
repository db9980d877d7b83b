"""Drop-in for the reference's ``ssim`` module (ssim.py): 13x13 Gaussian SSIM map, zero padded,
depthwise - computed by the separable shared-memory kernels in csrc/warp_ops.cu + ssim_tile.cuh."""
from math import exp
import torch
from . import _lib


def gaussian(window_size, sigma):
    """Reference ssim.py:9-11 (the fp32 taps handed to the kernels are built exactly like this)."""
    gauss = torch.Tensor([exp(-(x - window_size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(window_size)])
    return gauss / gauss.sum()


def create_window(window_size, channel):
    """Reference ssim.py:13-17."""
    _1D_window = gaussian(window_size, 1.5).unsqueeze(1)
    _2D_window = _1D_window.mm(_1D_window.t()).float().unsqueeze(0).unsqueeze(0)
    return _2D_window.expand(channel, 1, window_size, window_size).contiguous()


_TAPS = None


def taps13():
    global _TAPS
    if _TAPS is None:
        _TAPS = [float(v) for v in gaussian(13, 1.5)]
    return _TAPS


class _Ssim(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img1, img2):
        a, b = _lib.f32(img1), _lib.f32(img2)
        Bn, Cc, h, w = a.shape
        out = torch.empty_like(a)
        _lib.call('ccb_ssim_fwd', a, b, Bn * Cc, h, w, taps13(), out, a)
        ctx.save_for_backward(a, b)
        return out

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        Bn, Cc, h, w = a.shape
        g = _lib.f32(g)
        d1 = torch.empty_like(a) if ctx.needs_input_grad[0] else None
        d2 = torch.empty_like(b) if ctx.needs_input_grad[1] else None
        work, wf = _lib.workspace('ccb_ssim_bwd_workspace_floats', Bn * Cc, h, w, like=a)
        _lib.call('ccb_ssim_bwd', a, b, Bn * Cc, h, w, taps13(), g, d1, d2, work, wf, a)
        return d1, d2


def ssim(img1, img2, window_size=13, size_average=True):
    """SSIM *map* [B,C,H,W] (the reference's ``.mean()`` is commented out).  Reference ssim.py:68-76."""
    if window_size != 13:
        raise NotImplementedError('cc_b200.ssim: only the window the reference actually uses (13) is built')
    assert img1.size() == img2.size()
    return _Ssim.apply(img1, img2)
