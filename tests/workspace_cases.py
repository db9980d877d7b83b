"""The workspace contract of include/ccb200.h, entry point by entry point: every scratch buffer comes with its size, the
library refuses a short one before it launches anything, and a larger one changes nothing.  Run on the CPU simulator
build (tests/test_workspace_contract.py) and on the H100 (tests/test_gpu_workspace_contract.py).

Each row drives the entry point through its Python caller at a small shape.  While the caller runs, the call of the
entry point is intercepted and repeated with the buffer it was given (the size its query returns), with one 8x the
size + 4096, and with one unit short; the last must raise naming the entry point and the buffer, launch nothing and
leave outputs filled with a sentinel as they were.  Then the original call proceeds."""
import collections
import ctypes as C
import re
import numpy as np
import pytest
import torch
from cc_b200 import _lib, evaluate as CE, input_pipeline as CI, inverse_warp as CW, loss_functions as CL, nn as cnn, \
    ssim as CS, synth

# entry: the C name without 'ccb_' (as ccb_last_error_string() names it); buf / size: the argument positions of the
# buffer and its size, or the descriptor field names; outs: output argument positions or descriptor fields; run: the
# Python caller at a small shape; invalid: (size query, arguments) that must give -1.
Row = collections.namedtuple('Row', 'entry buf size outs run invalid')
UNITS = {'floats': torch.float32, 'words': torch.int64, 'bytes': torch.uint8}


def _leaf(t):
    return t.clone().requires_grad_(True)


def _rand(dev, *shape, seed=0, lo=0.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(*shape, generator=g)).to(dev)


def _act_bwd_bias(dev):
    g, y = _rand(dev, 1, 3, 96, 96, seed=1, lo=-1), _rand(dev, 1, 3, 96, 96, seed=2, lo=-1)      # B * plane > 8192
    cnn._act_bwd_bias(g, y, _lib.ACT_RELU, 0.0, torch.empty(3, device=dev))


def _bn(dev):
    x = _leaf(_rand(dev, 2, 3, 5, 7, seed=3))
    y = cnn._BatchNormFn.apply(x, _leaf(_rand(dev, 3, seed=4)), _leaf(_rand(dev, 3, seed=5)), torch.zeros(3, device=dev),
                               torch.ones(3, device=dev), True, 1e-5, 0.1)
    y.backward(_rand(dev, 2, 3, 5, 7, seed=6, lo=-1))


def _corr81(dev):
    f1, f2 = _leaf(_rand(dev, 1, 64, 8, 8, seed=7)), _leaf(_rand(dev, 1, 64, 8, 8, seed=8))     # several channel chunks
    cnn.corr81(f1, f2).backward(_rand(dev, 1, 81, 8, 8, seed=9, lo=-1))


def _ssim(dev):
    a, b = _leaf(_rand(dev, 1, 3, 12, 20, seed=10)), _leaf(_rand(dev, 1, 3, 12, 20, seed=11))
    CS.ssim(a, b).sum().backward()


def _flow_warp(dev):
    img, flow = _leaf(_rand(dev, 2, 3, 10, 14, seed=12)), _leaf(_rand(dev, 2, 2, 10, 14, seed=13, lo=-2, hi=2))
    CW.flow_warp(img, flow).sum().backward()


def _featwarp(dev):
    x, flow = _leaf(_rand(dev, 1, 4, 9, 11, seed=14)), _leaf(_rand(dev, 1, 2, 9, 11, seed=15, lo=-2, hi=2))
    cnn.feat_warp(x, flow).sum().backward()


def _rigid_inputs(dev, B=1, H=16, W=32):
    K, Kinv = (t.to(dev) for t in synth.intrinsics(B, H, W))
    depth = _leaf(_rand(dev, B, 1, H, W, seed=16, lo=1, hi=5))
    return K, Kinv, depth


def _inverse_warp(dev):
    K, Kinv, depth = _rigid_inputs(dev)
    pose = _leaf(_rand(dev, 1, 6, seed=17, lo=-0.05, hi=0.05))
    CW.inverse_warp(_rand(dev, 1, 3, 16, 32, seed=18), depth[:, 0], pose, K, Kinv).sum().backward()


def _pose2flow(dev):
    K, Kinv, depth = _rigid_inputs(dev)
    pose = _leaf(_rand(dev, 1, 6, seed=19, lo=-0.05, hi=0.05))
    CW.pose2flow(depth[:, 0], pose, K, Kinv).sum().backward()


def _photo(dev):
    tgt, refs = synth.frames(1, 16, 32, seed=20)
    K, Kinv, depth = _rigid_inputs(dev)
    pose = _leaf(_rand(dev, 1, len(refs), 6, seed=21, lo=-0.05, hi=0.05))
    CL.photometric_reconstruction_loss(tgt.to(dev), [r.to(dev) for r in refs], K, Kinv, [depth], [None], pose).backward()


def _smooth(dev):
    CL.smooth_loss([_leaf(_rand(dev, 2, 1, 16, 24, seed=22)), _leaf(_rand(dev, 2, 1, 8, 12, seed=23))]).backward()


def _bce(dev):
    CL.explainability_loss([_leaf(_rand(dev, 2, 4, 16, 24, seed=24, lo=0.1, hi=0.9))]).backward()


def _flow_metrics(dev):
    gt = _rand(dev, 2, 3, 12, 20, seed=25, lo=-3, hi=3)
    gt[:, 2] = (gt[:, 2] > 0).float()
    CL.compute_all_epes(gt, _rand(dev, 2, 2, 6, 10, seed=26), _rand(dev, 2, 2, 6, 10, seed=27), _rand(dev, 2, 1, 6, 10, seed=28))


def _depth_errors(dev):
    CL.compute_errors(_rand(dev, 2, 12, 20, seed=29, lo=0.5, hi=90), _rand(dev, 2, 12, 20, seed=30, lo=0.5, hi=90))


def _mask_iou(dev):
    CE.motion_mask_counts(_rand(dev, 1, 3, 8, 12, seed=31), _rand(dev, 1, 2, 8, 12, seed=32), _rand(dev, 1, 2, 8, 12, seed=33),
                          (_rand(dev, 1, 10, 14, seed=34) > 0.5).float(), torch.full((1, 10, 14), 26.0, device=dev), 0.7,
                          want_masks=True)


def _flow_color(dev):
    CE.flow_colors(_rand(dev, 1, 2, 2, 6, 9, seed=35, lo=-4, hi=4))


def _kitti_flow_errors(dev):
    gt, pred = (np.random.RandomState(s).randint(0, 65536, (1, 6, 9, 3)).astype(np.uint16) for s in (36, 37))
    CE.kitti_flow_errors(gt, pred)          # numpy triplets: the call puts them on the library's device


def _resize_u8(dev):
    CI.resize_frames((_rand(dev, 2, 9, 13, 3, seed=38, hi=255)).to(torch.uint8), 6, 17)


def _normalize_local(dev):
    CI.normalize_local([_rand(dev, 2, 3, 7, 9, seed=39), _rand(dev, 2, 3, 7, 9, seed=40)])


_PHOTO_BAD = lambda: _lib.PhotoDesc(nlevels=0)      # noqa: E731
ROWS = [
    Row('act_bwd_bias', 9, 10, [2, 3], _act_bwd_bias, ('ccb_act_bwd_bias_workspace_floats', (0, 3, 9216))),
    Row('bn_fwd', 13, 14, [3, 4, 5, 6], _bn, ('ccb_bn_workspace_floats', (2, 0, 35))),
    Row('bn_bwd', 10, 11, [4, 5, 6], _bn, ('ccb_bn_workspace_floats', (2, 3, 0))),
    Row('corr81_fwd', 8, 9, [2], _corr81, ('ccb_corr81_fwd_workspace_floats', (1, 64, 0, 8))),
    Row('corr81_bwd', 10, 11, [3, 4], _corr81, ('ccb_corr81_bwd_workspace_floats', (1, 64, 8, -1))),
    Row('ssim_bwd', 9, 10, [7, 8], _ssim, ('ccb_ssim_bwd_workspace_floats', (0, 12, 20))),
    Row('flow_warp_bwd', 10, 11, [8, 9], _flow_warp, None),
    Row('featwarp_bwd', 9, 10, [7, 8], _featwarp, None),
    Row('inverse_warp_bwd', 14, 15, [12, 13], _inverse_warp, ('ccb_warp_pose_partials_floats', (1, 0, 32))),
    Row('pose2flow_bwd', 13, 14, [11, 12], _pose2flow, ('ccb_warp_pose_partials_floats', (1, 16, 0))),
    Row('photo_loss_fwd', 'partials', 'partials_floats', ['loss', 'scal'], _photo, ('ccb_photo_partials_floats', _PHOTO_BAD)),
    Row('photo_loss_bwd', 'pose_partials', 'pose_partials_floats', ['d_pose', 'd_depth[0]'], _photo,
        ('ccb_photo_pose_partials_floats', _PHOTO_BAD)),
    Row('smooth_fwd', 'partials', 'partials_floats', ['loss'], _smooth,
        ('ccb_smooth_partials_floats', lambda: _lib.SmoothDesc(kind=_lib.SMOOTH_SECOND, B=1, C=1, nlevels=0))),
    Row('bce_fwd', 'partials', 'partials_floats', ['loss'], _bce,
        ('ccb_bce_partials_floats', lambda: _lib.BceDesc(kind=_lib.BCE_ONES, B=1, C=1, nlevels=9))),
    Row('flow_metrics', 16, 17, [15, 18], _flow_metrics, ('ccb_flow_metrics_workspace_bytes', (2, 12, 0))),
    Row('depth_errors', 6, 7, [8], _depth_errors, ('ccb_depth_errors_workspace_bytes', (0, 12, 20))),
    Row('mask_iou', 14, 15, [13, 16], _mask_iou, ('ccb_mask_iou_workspace_bytes', (1, 8, 12, 10, 0))),
    Row('flow_color', 5, 6, [7], _flow_color, ('ccb_flow_color_workspace_bytes', (1, 2, 0, 9))),
    Row('kitti_flow_errors', 5, 6, [7, 8], _kitti_flow_errors, ('ccb_kitti_flow_errors_workspace_bytes', (1, 6, -9))),
    Row('resize_u8', 7, 8, [1], _resize_u8, ('ccb_resize_u8_workspace_bytes', (2, 9, 13, 0, 17))),
    Row('normalize_local', 6, 7, [5, 0], _normalize_local, ('ccb_normalize_local_workspace_bytes', (2, 0, 9))),
]
IDS = [r.entry for r in ROWS]


class _Recorded:
    """Tensors handed to _lib.ptr while a caller runs, by address: what a descriptor's pointer fields point at."""

    def __init__(self):
        self.by_ptr = {}
        self.ptr = _lib.ptr

    def __call__(self, t, *a, **k):
        p = self.ptr(t, *a, **k)
        if p is not None:
            self.by_ptr[p] = t
        return p


def _field(d, path):
    m = re.match(r'(\w+)(?:\[(\d+)\])?$', path)
    v = getattr(d, m.group(1))
    return v[int(m.group(2))] if m.group(2) else v


class _Call:
    """One intercepted call of the row's entry point: its buffer, size and outputs can be replaced and it can be re-run."""

    def __init__(self, row, name, args, recorded):
        self.row, self.name, self.args = row, name, list(args)
        self.desc = self.args[0] if isinstance(row.buf, str) else None
        self.size0, self.buf0 = self.get(row.size), self.get(row.buf)
        outs = [self.get(o) for o in row.outs]
        if self.desc is not None:
            outs = [recorded.by_ptr[p] for p in outs if p]
        # optional outputs may be absent; a list of tensors (normalize_local's frames) counts frame by frame
        self.outs = [t for o in outs if o is not None for t in (o if isinstance(o, list) else [o])]

    def get(self, key):
        return _field(self.desc, key) if isinstance(key, str) else self.args[key]

    def run(self, buf, size, real_call):
        if self.desc is not None:
            setattr(self.desc, self.row.buf, buf.data_ptr() if buf is not None else None)
            setattr(self.desc, self.row.size, size)
        else:
            self.args[self.row.buf], self.args[self.row.size] = buf, size
        try:
            return real_call(self.name, *self.args)
        finally:
            if self.desc is not None:
                setattr(self.desc, self.row.buf, self.buf0)
                setattr(self.desc, self.row.size, self.size0)
            else:
                self.args[self.row.buf], self.args[self.row.size] = self.buf0, self.size0


def _sentinel(t):
    return t.fill_(float('nan')) if t.is_floating_point() else t.fill_(-7)


def _bits(t):
    return t.detach().contiguous().view(torch.uint8).cpu()


def check_row(device, row, monkeypatch):
    """The row's caller with the contract checks spliced into its call of the entry point."""
    real_call, recorded, seen = _lib.call, _Recorded(), []
    entry = 'ccb_' + row.entry

    def spy(name, *args):
        if name != entry:
            return real_call(name, *args)
        c = _Call(row, name, args, recorded)
        need = c.size0
        buf0 = c.buf0 if c.desc is None else recorded.by_ptr.get(c.buf0)
        assert need > 0 and buf0 is not None and buf0.numel() == need, (row.entry, need)
        unit = {t: u for u, t in UNITS.items()}[buf0.dtype]
        init = [o.clone() for o in c.outs]
        results = []
        for n in (need, 8 * need + 4096):                     # the queried size, and a much larger buffer
            for o, i in zip(c.outs, init):
                o.copy_(i)
            buf = torch.empty(n, dtype=UNITS[unit], device=buf0.device)
            assert c.run(buf, n, real_call) == 0
            results.append([_bits(o) for o in c.outs])
        for a, b in zip(*results):
            assert torch.equal(a, b), '%s: a larger %s changes the result' % (row.entry, row.buf)
        for o in c.outs:
            _sentinel(o)
        marks = [_bits(o) for o in c.outs]
        before = _lib.lib().ccb_launch_count()
        short = torch.empty(need - 1, dtype=UNITS[unit], device=buf0.device) if need > 1 else None
        buf_name = row.buf if isinstance(row.buf, str) else ('work' if row.entry not in ('inverse_warp_bwd', 'pose2flow_bwd')
                                                             else 'pose_partials')
        with pytest.raises(RuntimeError, match=r'%s failed \(status -1\): %s: %s of %d %s, %d needed'
                           % (entry, row.entry, buf_name, need - 1, unit, need)):
            c.run(short, need - 1, real_call)
        assert _lib.lib().ccb_launch_count() == before, '%s: a refused call launched kernels' % row.entry
        for o, m in zip(c.outs, marks):
            assert torch.equal(_bits(o), m), '%s: a refused call wrote an output' % row.entry
        for o, i in zip(c.outs, init):
            o.copy_(i)
        seen.append(need)
        return real_call(name, *args)

    monkeypatch.setattr(_lib, 'call', spy)
    monkeypatch.setattr(_lib, 'ptr', recorded)
    row.run(device)
    if device.type == 'cuda':
        torch.cuda.synchronize()
    assert seen, '%s was not called' % entry
    if row.invalid is not None:
        query, args = row.invalid
        args = (args(),) if callable(args) else args
        fn = getattr(_lib.lib(), query)
        assert fn(*[C.byref(a) if isinstance(a, C.Structure) else a for a in args]) == -1, (query, args)
        with pytest.raises(RuntimeError, match=query):
            _lib.workspace(query, *args, like=torch.empty(0, device=device))


# Where a buffer is not needed its size is 0 and NULL is accepted.
def _zero_need_calls(dev):
    x = _rand(dev, 2, 3, 5, 7, seed=41)
    y = torch.empty_like(x)
    yield 'bn_fwd', ('ccb_bn_fwd', x, torch.ones(3, device=dev), torch.zeros(3, device=dev), y, None,
                     torch.zeros(3, device=dev), torch.ones(3, device=dev), 2, 3, 35, 1e-5, 0.1, 0, None, 0, x)
    f1, f2, g = _rand(dev, 1, 64, 8, 8, seed=42), _rand(dev, 1, 64, 8, 8, seed=43), _rand(dev, 1, 81, 8, 8, seed=44)
    yield 'corr81_bwd', ('ccb_corr81_bwd', f1, f2, g, torch.empty_like(f1), None, 1, 64, 8, 8, 0, None, 0, f1)
    img, flow, go = _rand(dev, 2, 3, 10, 14, seed=45), _rand(dev, 2, 2, 10, 14, seed=46), _rand(dev, 2, 3, 10, 14, seed=47)
    yield 'flow_warp_bwd', ('ccb_flow_warp_bwd', img, flow, 2, 3, 10, 14, 0, go, torch.empty_like(flow), None, None, 0, img)
    yield 'featwarp_bwd', ('ccb_featwarp_bwd', img, flow, 2, 3, 10, 14, go, torch.empty_like(flow), None, None, 0, img)
    gb = _rand(dev, 1, 3, 96, 96, seed=48)
    yield 'act_bwd_bias', ('ccb_act_bwd_bias', gb, gb, torch.empty_like(gb), None, 1, 3, 9216, _lib.ACT_RELU, 0.0, None, 0, gb)


def check_zero_need(device):
    for entry, args in _zero_need_calls(device):
        assert _lib.call(*args) == 0, entry
