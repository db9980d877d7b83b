"""Oracle: the reference's KITTI-2015 flow submission (submit_flow.py:109-175), its file formats (flowutils/flow_io.py
flow_write_png :120-150, flow_write :57-93, flow_read_png :96-117), the Middlebury colour coding of its visualisation
(flowutils/flowlib.py flow_to_image :189-226, compute_color :345-386, make_color_wheel :389-436) and the scoring of
evaluate_flow.py (compute_err :44-53), restated in torch on the CPU and numpy.  TEST INFRASTRUCTURE."""
import numpy as np
import torch
import torch.nn.functional as F
from . import nets as ON, geometry as OG

UNKNOWN_FLOW_THRESH = 1e7


def submit_flows(emask, flow_cam, flow_fwd, Hg, Wg, THRESH=0.01):
    """submit_flow.py:119-145 on [B,...] tensors: (combined [B,1,h,w], cam, fwd, total [B,2,Hg,Wg]) at full resolution,
    u scaled by w_gt / w_pred and v by h_gt / h_pred (python floats) as the script scales them in place."""
    bare = 1 - (1 - emask[:, 1]) * (1 - emask[:, 2]).unsqueeze(1) > 0.5
    soft = (flow_cam - flow_fwd).abs()
    census = (soft[:, 0] < THRESH).type_as(flow_fwd) * (soft[:, 1] < THRESH).type_as(flow_fwd)
    combined = 1 - (1 - bare.type_as(emask)) * (1 - census.type_as(emask))
    h, w = flow_cam.shape[2:]
    pred_mask = F.interpolate(combined, size=(h, w), mode='bilinear', align_corners=False)
    total = (pred_mask <= THRESH).type_as(flow_fwd).expand_as(flow_fwd) * flow_fwd + \
        (pred_mask > THRESH).type_as(flow_cam).expand_as(flow_cam) * flow_cam
    out = []
    for f in (flow_cam, flow_fwd, total):
        full = F.interpolate(f, size=(Hg, Wg), mode='bilinear', align_corners=False)
        full[:, 0] = full[:, 0] * (Wg / w)
        full[:, 1] = full[:, 1] * (Hg / h)
        out.append(full)
    return combined, out[0], out[1], out[2]


def kitti_png_rows(u, v):
    """flow_write_png's image: uint16 [H, W, 3] = (u*64 + 2^15, v*64 + 2^15, 1), the float64 -> uint16 cast of numpy."""
    enc = lambda x: ((np.asarray(x).astype('float64') * 64.0) + 2 ** 15).astype('uint16')     # noqa: E731
    with np.errstate(invalid='ignore'):
        return np.dstack((enc(u), enc(v), np.ones(np.shape(u), dtype='uint16')))


def flo_bytes(u, v):
    """The bytes flow_write writes: 'PIEH', int32 width, int32 height, then u, v interleaved as float32."""
    h, w = np.shape(u)
    tmp = np.zeros((h, w * 2))
    tmp[:, 0::2] = u
    tmp[:, 1::2] = v
    return b'PIEH' + np.array([w, h], np.int32).tobytes() + tmp.astype(np.float32).tobytes()


def decode_png_rows(img):
    """flow_read_png's decoding of a uint16 [H, W, 3] image: (u, v, valid)."""
    return (img[:, :, 0].astype('float64') - 2 ** 15) / 64.0, (img[:, :, 1].astype('float64') - 2 ** 15) / 64.0, img[:, :, 2]


def make_color_wheel():
    """[55, 3] float64: the Middlebury wheel, RY 15, YG 6, GC 4, CB 11, BM 13, MR 6 steps with ramps floor(255 k / n)."""
    wheel = []
    for n, fixed, ramp, rising in ((15, 0, 1, True), (6, 1, 0, False), (4, 1, 2, True), (11, 2, 1, False),
                                   (13, 2, 0, True), (6, 0, 2, False)):
        for k in range(n):
            c = [0.0, 0.0, 0.0]
            c[fixed] = 255.0
            step = np.floor(255 * k / n)
            c[ramp] = step if rising else 255 - step
            wheel.append(c)
    return np.array(wheel)


def flow_to_image(flow):
    """flowlib.flow_to_image of a [2, H, W] array (not modified): float64 [3, H, W] = uint8 levels / 255."""
    u, v = np.array(flow[0]), np.array(flow[1])
    unknown = (abs(u) > UNKNOWN_FLOW_THRESH) | (abs(v) > UNKNOWN_FLOW_THRESH)
    u[unknown] = 0
    v[unknown] = 0
    maxrad = max(-1, np.max(np.sqrt(u ** 2 + v ** 2)))       # a NaN maximum loses to -1 in python's max
    u = u / (maxrad + np.finfo(float).eps)
    v = v / (maxrad + np.finfo(float).eps)
    img = compute_color(u, v)
    img[unknown] = 0
    return img.transpose(2, 0, 1) / 255.


def compute_color(u, v):
    """flowlib.compute_color: float64 [H, W, 3] of uint8 levels; NaN pixels black.  u and v are zeroed where NaN."""
    nan = np.isnan(u) | np.isnan(v)
    u[nan] = 0
    v[nan] = 0
    wheel = make_color_wheel()
    ncols = wheel.shape[0]
    rad = np.sqrt(u ** 2 + v ** 2)
    fk = (np.arctan2(-v, -u) / np.pi + 1) / 2 * (ncols - 1) + 1
    k0 = np.floor(fk).astype(int)
    k1 = k0 + 1
    k1[k1 == ncols + 1] = 1
    f = fk - k0
    img = np.zeros(u.shape + (3,))
    inside = rad <= 1
    for i in range(3):
        col = (1 - f) * (wheel[k0 - 1, i] / 255) + f * (wheel[k1 - 1, i] / 255)
        col[inside] = 1 - rad[inside] * (1 - col[inside])
        col[~inside] *= 0.75
        img[:, :, i] = np.uint8(np.floor(255 * col * (1 - nan)))
    return img


def compute_err(u_gt, v_gt, valid_gt, u_pred, v_pred, tau=(3, 0.05)):
    """evaluate_flow.compute_err: [aepe, Fl] in float64, plus the outlier count (weighted by valid_gt)."""
    epe = np.sqrt((u_gt - u_pred) ** 2 + (v_gt - v_pred) ** 2) * valid_gt
    mag = np.sqrt(u_gt ** 2 + v_gt ** 2)
    n_err = (epe > tau[0]) * ((epe / (mag + 1e-8)) > tau[1]) * valid_gt
    return [epe.sum() / valid_gt.sum(), n_err.sum() / valid_gt.sum()], int(n_err.sum())


def submission_sample(P, tgt, refs, K, Kinv, Hg, Wg, THRESH=0.01, flownet='Back2Future'):
    """submit_flow.py:109-175 for one sample on the functional oracle nets: (net outputs (emask, flow_cam, flow_fwd),
    submit_flows of them, the uint16 KITTI image [Hg, Wg, 3] of the total flow, row 2 of the visualisation as float64
    [3, 3*Hg, Wg])."""
    with torch.no_grad():
        disp = ON.disp_forward(P['disp'], tgt, training=False)
        pose = ON.pose_forward(P['pose'], tgt, refs)
        emask = ON.mask_forward(P['mask'], tgt, refs, training=False)
        flow_fwd = ON.flow_eval(P['flow'], tgt, refs, flownet)
        flow_cam = OG.pose2flow((1 / disp).squeeze(1), pose[:, 2], K, Kinv)
        combined, cam, fwd, total = submit_flows(emask, flow_cam, flow_fwd, Hg, Wg, THRESH)
    png = kitti_png_rows(total[0, 0].numpy(), total[0, 1].numpy())
    viz = flow_to_image(np.hstack((cam[0].numpy(), fwd[0].numpy(), total[0].numpy())))
    return (emask, flow_cam, flow_fwd), (combined, cam, fwd, total), png, viz
