#!/usr/bin/env python
"""Generate tests/golden/flow_submit_small.npz from the UNMODIFIED reference flowutils (flowlib.py, flow_io.py) and
evaluate_flow.py.  Run:  python tests/golden/make_flow_submit.py   (the reference checkout is found as in make_golden.py;
the other fixtures are not touched).

Called as they are:
  flowlib.flow_to_image, flowlib.make_color_wheel
  flow_io.flow_write_png     under a `png` stand-in whose Writer.write records the uint16 rows (pypng is not installed)
  flow_io.flow_write         writes a real file; its bytes are frozen (as a sha256 digest where the file is large)
  flow_io.flow_read_png      under a `png` stand-in whose Reader yields recorded rows as pypng does (array('H') rows)
  evaluate_flow.compute_err  with empty stand-ins for tqdm, path and logger, which it does not use
flowlib imports torchvision at module level for a function not used here; it gets an empty stand-in too.
submit_flow.py's sample body lives inside main(): the full-resolution flows are computed here by the same torch calls on
the CPU (F.upsample, then the in-place scale by the python float ratio) and pinned as a restatement only.

Cases (all names prefixed by the case):
  small  64x128 -> 96x200 and  odd  32x96 -> 47x150: inputs emask [1,3,h,w], cam, fwd [1,2,h,w] (values on a 1/256
         grid, so the file compresses; about a third of the pixels pass the census), THRESH 0.01; outputs the combined
         mask, the KITTI rows of the total flow, the .flo bytes, row 2 of the visualisation as uint8 levels (stack of
         cam, fwd, total with one radius)
  wrap   a [2,8,40] flow written as it is: values past +-512 px, on the truncation boundaries and past the int32 range
  unknown_nan  |u| > 1e7 and NaN pixels (python's max(-1, nan) makes the radius -1)
  zero   an all-zero flow (radius 0)
  stack3 three panels whose radii differ by 10x
  err    compute_err of two decoded 47x150 KITTI images (valid 0/1, outliers present)"""
import array
import hashlib
import os
import sys
import tempfile
import types
import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG                      # noqa: E402  (reference import path, save helpers)


class _Absent(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith('__'):
            raise AttributeError(name)
        return _Absent(self.__name__ + '.' + name)


WRITTEN, TO_READ = [], {}


class _Writer:
    def __init__(self, width, height, bitdepth, planes):
        self.shape = (height, width, planes)
        assert bitdepth == 16

    def write(self, f, rows):
        WRITTEN.append(np.array(rows, dtype=np.uint16).reshape(self.shape))


class _Reader:
    def __init__(self, fpath):
        self.img = TO_READ[str(fpath)]

    def asDirect(self):
        h, w, _ = self.img.shape
        return w, h, (array.array('H', row.reshape(-1).tolist()) for row in self.img), {}


def import_reference():
    png = types.ModuleType('png')
    png.Writer, png.Reader = _Writer, _Reader
    stand_ins = {'png': png, 'torchvision': _Absent('torchvision'), 'torchvision.transforms': _Absent('torchvision.transforms'),
                 'tqdm': _Absent('tqdm'), 'path': _Absent('path'), 'logger': _Absent('logger')}
    added = [m for m in stand_ins if m not in sys.modules]
    for m in added:
        sys.modules[m] = stand_ins[m]
    try:
        from flowutils import flowlib, flow_io
        import evaluate_flow
    finally:
        for m in added:
            del sys.modules[m]
    for mod in (flowlib, flow_io, evaluate_flow):
        assert os.path.abspath(mod.__file__).startswith(os.path.abspath(MG.REF)), mod.__file__
    assert flow_io.has_png
    return flowlib, flow_io, evaluate_flow


def q256(a):
    return (np.round(np.asarray(a, np.float64) * 256) / 256).astype(np.float32)


def submit_inputs(rs, h, w):
    emask = q256(rs.rand(1, 3, h, w) * 0.6)
    cam = q256(rs.randn(1, 2, h, w) * 6)
    fwd = cam + q256(rs.randn(1, 2, h, w) * 4)
    near = rs.rand(1, 1, h, w) < 0.4                        # the census: |cam - fwd| < 0.01 in u and v
    fwd = np.where(near, cam + q256(rs.randint(-1, 2, size=(1, 2, h, w)) / 256.), fwd).astype(np.float32)
    return emask, cam, fwd


def script_flows(emask, cam, fwd, Hg, Wg, THRESH):
    """submit_flow.py:119-145 verbatim in its torch calls (CPU)."""
    explainability_mask, flow_cam, flow_fwd = (torch.from_numpy(a) for a in (emask, cam, fwd))
    rigidity_mask = 1 - (1 - explainability_mask[:, 1]) * (1 - explainability_mask[:, 2]).unsqueeze(1) > 0.5
    soft = (flow_cam - flow_fwd).abs()
    census = (soft[:, 0] < THRESH).type_as(flow_fwd) * (soft[:, 1] < THRESH).type_as(flow_fwd)
    combined = 1 - (1 - rigidity_mask.type_as(explainability_mask)) * (1 - census.type_as(explainability_mask))
    _, _, h_pred, w_pred = flow_cam.size()
    pred_mask = F.upsample(combined, size=(h_pred, w_pred), mode='bilinear')
    total = (pred_mask <= THRESH).type_as(flow_fwd).expand_as(flow_fwd) * flow_fwd + \
        (pred_mask > THRESH).type_as(flow_cam).expand_as(flow_cam) * flow_cam
    out = []
    for f in (flow_cam, flow_fwd, total):
        full = F.upsample(f, size=(Hg, Wg), mode='bilinear')
        full[:, 0, :, :] = full[:, 0, :, :] * (Wg / w_pred)
        full[:, 1, :, :] = full[:, 1, :, :] * (Hg / h_pred)
        out.append(full[0].numpy())
    return combined[0].numpy(), out


def gen():
    import warnings
    warnings.filterwarnings('ignore')
    flowlib, flow_io, evaluate_flow = import_reference()
    rs = np.random.RandomState(61)
    d, tmp = {}, tempfile.mkdtemp()

    def written(u, v):
        del WRITTEN[:]
        flow_io.flow_write_png(os.path.join(tmp, 'x_10.png'), u=u, v=v)
        assert len(WRITTEN) == 1
        return WRITTEN[0]

    def flo(u, v):
        p = os.path.join(tmp, 'x_10.flo')
        flow_io.flow_write(p, u, v)
        with open(p, 'rb') as f:
            return f.read()

    def levels(flow):
        img = flowlib.flow_to_image(np.array(flow))
        lv = np.round(img * 255).astype(np.uint8)
        assert img.dtype == np.float64 and np.array_equal(lv / 255., img)
        return lv

    def encoded(name, u, v, keep_flo):
        d[name + '_png'] = written(u, v)
        b = flo(u, v)
        d[name + '_flo_sha256'] = np.array(hashlib.sha256(b).hexdigest())
        if keep_flo:
            d[name + '_flo'] = np.frombuffer(b, np.uint8)

    for name, (h, w, Hg, Wg) in (('small', (64, 128, 96, 200)), ('odd', (32, 96, 47, 150))):
        emask, cam, fwd = submit_inputs(rs, h, w)
        combined, (cam_f, fwd_f, total_f) = script_flows(emask, cam, fwd, Hg, Wg, 0.01)
        assert 0.2 < combined.mean() < 0.9
        d[name + '_emask'], d[name + '_cam'], d[name + '_fwd'], d[name + '_mask'] = emask, cam, fwd, combined
        encoded(name, total_f[0], total_f[1], keep_flo=(name == 'odd'))
        d[name + '_viz'] = levels(np.hstack((cam_f, fwd_f, total_f)))
        assert d[name + '_viz'].shape == (3, 3 * Hg, Wg)

    wrap = (rs.rand(2, 8, 40) * 3000 - 1500).astype(np.float32)
    special = [-512.0234375, -512.0078125, -511.9921875, 511.9921875, 512.0, 512.5, 1024.0, -1024.0, 1e6, -1e6, 4e7, -4e7,
               3.3554432e7, -3.3554432e7, 0.0, -0.0, 1e-30, -1e-30, 0.0078125, -0.0078125]
    wrap[0, 0, :len(special)] = special
    wrap[1, 1, :len(special)] = special[::-1]
    d['wrap_flow'] = wrap
    encoded('wrap', wrap[0], wrap[1], keep_flo=True)
    d['wrap_viz'] = levels(wrap)

    un = (rs.randn(2, 12, 20) * 3).astype(np.float32)
    un[0, 1, 2], un[1, 3, 4], un[0, 5, 5], un[1, 5, 6] = 2e7, -1.5e7, 1e7, -1e7      # unknown, unknown, known, known
    un[0, 7, 7], un[1, 8, 9] = np.nan, np.nan
    d['unknown_nan_flow'] = un
    d['unknown_nan_viz'] = levels(un)
    d['zero_flow'] = np.zeros((2, 6, 10), np.float32)
    d['zero_viz'] = levels(d['zero_flow'])
    panels = [(rs.randn(2, 10, 16) * s).astype(np.float32) for s in (0.5, 5.0, 50.0)]
    d['stack3_flow'] = np.stack(panels)
    d['stack3_viz'] = levels(np.hstack(panels))
    d['wheel'] = flowlib.make_color_wheel()

    gu, gv = rs.randn(47, 150) * 20, rs.randn(47, 150) * 8
    valid = (rs.rand(47, 150) < 0.7).astype(np.float64)
    pu = gu + rs.randn(47, 150) * np.where(rs.rand(47, 150) < 0.2, 8, 0.5)
    pv = gv + rs.randn(47, 150) * 0.5
    d['err_gt'] = written(gu, gv)
    d['err_gt'][:, :, 2] = valid
    d['err_pred'] = written(pu, pv)
    TO_READ['gt'], TO_READ['pred'] = d['err_gt'], d['err_pred']
    u_gt, v_gt, valid_gt = flow_io.flow_read_png('gt')
    u_pred, v_pred, valid_pred = flow_io.flow_read_png('pred')
    d['err_out'] = np.array(evaluate_flow.compute_err(u_gt, v_gt, valid_gt, u_pred, v_pred, valid_pred), np.float64)
    d['err_decoded_row0'] = np.stack([u_gt[0], v_gt[0], valid_gt[0], u_pred[0], v_pred[0]]).astype(np.float64)
    assert 0.02 < d['err_out'][1] < 0.5, d['err_out']
    MG.save('flow_submit_small', d)


if __name__ == '__main__':
    gen()
