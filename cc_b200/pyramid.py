"""Image pyramid shared by every loss term of a step.

The reference re-pools the full-resolution frames with ``adaptive_avg_pool2d`` inside every loss
function at every level (15 pools per level per step: loss_functions.py:36-37,89-90,163-165,315).
Here one kernel builds all levels once per frame tensor; results are memoised for the step.

State: the C library keeps none; this Python-side memo holds at most 12 (frame tensor -> levels) entries keyed on tensor
identity + version, and `Trainer.step` clears it on entry and exit, so no reference outlives a step.  Plain callers
of the loss functions may call `clear()` themselves (stale entries are only ever evicted, never wrong: a changed
tensor has a new version)."""
import torch
from . import _lib

_CACHE = []          # [(src tensor, version, nlevels, [levels])], most recent last
_CACHE_MAX = 12


def level_sizes(H, W, nlevels):
    return [(H >> l, W >> l) for l in range(nlevels)]


def build(img, nlevels):
    """img [B,C,H,W] -> [img, level1, ...]; level l is the exact 2^l box mean."""
    img = _lib.f32(img)
    B, Cc, H, W = img.shape
    if nlevels == 1:
        return [img]
    div = 1 << (nlevels - 1)
    if H % div or W % div:
        raise NotImplementedError('cc_b200: frame size %dx%d is not divisible by %d (pyramid levels must '
                                  'be exact halvings)' % (H, W, div))
    outs = [torch.empty(B, Cc, H >> l, W >> l, device=img.device, dtype=torch.float32) for l in range(1, nlevels)]
    _lib.call('ccb_image_pyramid', img, B * Cc, H, W, nlevels, outs, img)
    return [img] + outs


def get(img, nlevels):
    """Cached pyramid of a frame tensor (keyed on tensor identity + version counter)."""
    for k, (src, ver, nl, lv) in enumerate(_CACHE):
        if src is img and ver == img._version and nl >= nlevels:
            return lv[:nlevels]
    lv = build(img, nlevels)
    _CACHE.append((img, img._version, nlevels, lv))
    if len(_CACHE) > _CACHE_MAX:
        del _CACHE[0]
    return lv


def clear():
    del _CACHE[:]


def levels_for(img, sizes):
    """Pyramid levels matching the (h,w) list of a prediction pyramid; sizes must be exact halvings
    of the frame (what the reference's nets produce at 256x832 / 128x416)."""
    H, W = img.shape[2], img.shape[3]
    idx = []
    for (h, w) in sizes:
        l = 0
        while (H >> l) > h:
            l += 1
        if (H >> l) != h or (W >> l) != w or H % (1 << l) or W % (1 << l):
            raise NotImplementedError('cc_b200: level size %dx%d is not an exact 2^l reduction of %dx%d'
                                      % (h, w, H, W))
        idx.append(l)
    pyr = get(img, max(idx) + 1)
    return [pyr[l] for l in idx]
