"""numpy restatements of the two Pillow resamplers behind the reference's scipy.misc calls, and of NormalizeLocally
(custom_transforms.py:33-44), for checks at sizes where neither the reference nor Pillow is at hand.

  rotate_u8  = scipy.misc.imrotate(im, angle) = Image.rotate(angle, resample=BILINEAR): Pillow's affine_transform with
               bilinear_filter32RGB, fp64 without fused multiply-adds, truncated to uint8; 0 where the source point
               falls outside the image.  The six coefficients come from input_pipeline.pil_rotate_affine.
  resize_u8  = scipy.misc.imresize(im, (h, w)) = Image.resize((w, h), BILINEAR): ImagingResample's triangle filter
               widened by the scale factor on a downscale, weights in 22-bit fixed point, horizontal pass first, each
               pass rounded back to uint8; a pass whose size does not change is skipped.
Python floats and numpy's element-wise ufuncs are IEEE double without contraction, as Pillow's x86-64 build is."""
import numpy as np

PRECISION_BITS = 22


def rotate_u8(im, a):
    """im [H,W,3] uint8, a = 6 affine coefficients (output pixel centre -> input point) -> [H,W,3] uint8."""
    H, W, _ = im.shape
    a = [float(v) for v in a]
    yy, xx = np.meshgrid(np.arange(H, dtype=np.float64) + 0.5, np.arange(W, dtype=np.float64) + 0.5, indexing='ij')
    xin = a[0] * xx + a[1] * yy + a[2]
    yin = a[3] * xx + a[4] * yy + a[5]
    inside = (xin >= 0) & (xin < W) & (yin >= 0) & (yin < H)
    xin, yin = xin - 0.5, yin - 0.5
    x, y = np.floor(xin), np.floor(yin)
    dx, dy = xin - x, yin - y
    x, y = x.astype(np.int64), y.astype(np.int64)
    x0, x1, yc = np.clip(x, 0, W - 1), np.clip(x + 1, 0, W - 1), np.clip(y, 0, H - 1)
    y1ok = (y + 1 >= 0) & (y + 1 < H)
    y1 = np.clip(y + 1, 0, H - 1)
    src = im.astype(np.float64)
    out = np.zeros_like(im)
    for c in range(3):
        p = src[..., c]
        v1 = p[yc, x0] + (p[yc, x1] - p[yc, x0]) * dx
        v2 = np.where(y1ok, p[y1, x0] + (p[y1, x1] - p[y1, x0]) * dx, v1)
        v = v1 + (v2 - v1) * dy
        out[..., c] = np.where(inside, v.astype(np.uint8), 0)
    return out


def resample_coeffs(in_size, out_size):
    """Pillow precompute_coeffs + normalize_coeffs_8bpc for the bilinear filter: (xmin [out], k [out, ksize] int64)."""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 1.0 * filterscale
    ksize = int(np.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    xmins, kk = np.zeros(out_size, np.int64), np.zeros((out_size, ksize), np.int64)
    for xx in range(out_size):
        center = 0.0 + (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [max(0.0, 1.0 - abs((x + xmin - center + 0.5) * ss)) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        for x in range(xmax):
            kk[xx, x] = int(0.5 + (w[x] / ww if ww != 0.0 else w[x]) * (1 << PRECISION_BITS))
        xmins[xx] = xmin
    return xmins, kk


def _pass(im, out_size, axis):
    """One 8-bit resampling pass of im [..., n, ..., 3] along `axis`."""
    xmins, kk = resample_coeffs(im.shape[axis], out_size)
    x = np.moveaxis(im.astype(np.int64), axis, 0)
    n, ks = x.shape[0], kk.shape[1]
    idx = np.minimum(xmins[:, None] + np.arange(ks)[None, :], n - 1)          # zero weights past xmax
    acc = np.full((out_size,) + x.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    for j in range(ks):
        acc += x[idx[:, j]] * kk[:, j].reshape((out_size,) + (1,) * (x.ndim - 1))
    return np.moveaxis(np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8), 0, axis)


def resize_u8(im, h, w):
    """im [Hs,Ws,3] uint8 -> [h,w,3] uint8."""
    out = im
    if w != im.shape[1]:
        out = _pass(out, w, 1)
    if h != im.shape[0]:
        out = _pass(out, h, 0)
    return np.ascontiguousarray(out)


def normalize_locally(frames):
    """frames [F,3,H,W] (one sample's frames, fp32) -> (normalised frames, mean [3], std [3]): fp64 mean and unbiased
    std per channel over all frames, rounded to fp32, then (x - m) / s in fp32."""
    x = np.asarray(frames, np.float32)
    v = x.transpose(1, 0, 2, 3).reshape(3, -1).astype(np.float64)
    n = v.shape[1]
    mean = v.sum(1) / n
    std = np.sqrt(((v - mean[:, None]) ** 2).sum(1) / (n - 1))
    m, s = mean.astype(np.float32), std.astype(np.float32)
    with np.errstate(divide='ignore', invalid='ignore'):          # a zero std gives inf / nan, as in the reference
        out = (x - m[None, :, None, None]) / s[None, :, None, None]
    return out.astype(np.float32), m, s
