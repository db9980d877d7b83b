"""Drop-in for the reference's ``inverse_warp`` module (inverse_warp.py), backed by libccb200.

Same names, argument meaning and AssertionError text as the reference; every function launches
hand-written sm_90a kernels (cc_b200/csrc/warp_ops.cu) and supports autograd through
hand-derived backward kernels.  ``train.py:22`` imports inverse_warp, pose2flow, flow2oob, flow_warp."""
from __future__ import division
import torch
from . import _lib

_ROT = {'euler': _lib.ROT_EULER, 'quat': _lib.ROT_QUAT}
_PAD = {'zeros': _lib.PAD_ZEROS, 'border': _lib.PAD_BORDER, None: _lib.PAD_NONE}


def check_sizes(input, input_name, expected):
    """Reference inverse_warp.py:23-28."""
    condition = [input.ndimension() == len(expected)]
    for i, size in enumerate(expected):
        if size.isdigit():
            condition.append(input.size(i) == int(size))
    assert(all(condition)), "wrong size for {}, expected {}, got  {}".format(input_name, 'x'.join(expected), list(input.size()))


def _f(t):
    return _lib.contig(t.detach().float())


class _InverseWarp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img, depth, pose, K, Kinv, rot, pad):
        img, depth, pose, K, Kinv = _f(img), _f(depth), _f(pose), _f(K), _f(Kinv)
        B, _, h, w = img.shape
        out = torch.empty_like(img)
        L = _lib.lib()
        _lib.check(L.ccb_inverse_warp_fwd(_lib.ptr(img), _lib.ptr(depth), _lib.ptr(pose), 6, _lib.ptr(K), _lib.ptr(Kinv),
                                          B, h, w, rot, pad, _lib.ptr(out), _lib.stream(img)), 'inverse_warp_fwd')
        ctx.save_for_backward(img, depth, pose, K, Kinv)
        ctx.cfg = (rot, pad)
        return out

    @staticmethod
    def backward(ctx, g):
        img, depth, pose, K, Kinv = ctx.saved_tensors
        rot, pad = ctx.cfg
        B, _, h, w = img.shape
        g = _f(g)
        L = _lib.lib()
        d_depth = torch.empty_like(depth)
        d_pose = torch.empty_like(pose)
        part = torch.empty(L.ccb_warp_pose_partials_floats(B, h, w), device=img.device)
        _lib.check(L.ccb_inverse_warp_bwd(_lib.ptr(img), _lib.ptr(depth), _lib.ptr(pose), 6, _lib.ptr(K), _lib.ptr(Kinv),
                                          B, h, w, rot, pad, _lib.ptr(g), _lib.ptr(d_depth), _lib.ptr(d_pose),
                                          _lib.ptr(part), _lib.stream(img)), 'inverse_warp_bwd')
        return None, d_depth, d_pose, None, None, None, None


class _Pose2Flow(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth, pose, K, Kinv, rot, pad):
        depth, pose, K, Kinv = _f(depth), _f(pose), _f(K), _f(Kinv)
        B, h, w = depth.shape
        out = torch.empty(B, 2, h, w, device=depth.device)
        L = _lib.lib()
        _lib.check(L.ccb_pose2flow_fwd(_lib.ptr(depth), _lib.ptr(pose), 6, _lib.ptr(K), _lib.ptr(Kinv), B, h, w, rot, pad,
                                       _lib.ptr(out), _lib.stream(depth)), 'pose2flow_fwd')
        ctx.save_for_backward(depth, pose, K, Kinv)
        ctx.cfg = (rot, pad)
        return out

    @staticmethod
    def backward(ctx, g):
        depth, pose, K, Kinv = ctx.saved_tensors
        rot, pad = ctx.cfg
        B, h, w = depth.shape
        g = _f(g)
        L = _lib.lib()
        d_depth = torch.empty_like(depth)
        d_pose = torch.empty_like(pose)
        part = torch.empty(L.ccb_warp_pose_partials_floats(B, h, w), device=depth.device)
        _lib.check(L.ccb_pose2flow_bwd(_lib.ptr(depth), _lib.ptr(pose), 6, _lib.ptr(K), _lib.ptr(Kinv), B, h, w, rot, pad,
                                       _lib.ptr(g), _lib.ptr(d_depth), _lib.ptr(d_pose), _lib.ptr(part),
                                       _lib.stream(depth)), 'pose2flow_bwd')
        return d_depth, d_pose, None, None, None, None


class _FlowWarp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img, flow, pad):
        img, flow = _f(img), _f(flow)
        B, Cc, h, w = img.shape
        out = torch.empty_like(img)
        _lib.check(_lib.lib().ccb_flow_warp_fwd(_lib.ptr(img), _lib.ptr(flow), B, Cc, h, w, pad, _lib.ptr(out),
                                                _lib.stream(img)), 'flow_warp_fwd')
        ctx.save_for_backward(img, flow)
        ctx.pad = pad
        return out

    @staticmethod
    def backward(ctx, g):
        img, flow = ctx.saved_tensors
        B, Cc, h, w = img.shape
        g = _f(g)
        d_flow = torch.empty_like(flow) if ctx.needs_input_grad[1] else None
        d_img = torch.zeros_like(img) if ctx.needs_input_grad[0] else None
        work = _lib.scatter_workspace(img) if d_img is not None else None
        _lib.check(_lib.lib().ccb_flow_warp_bwd(_lib.ptr(img), _lib.ptr(flow), B, Cc, h, w, ctx.pad, _lib.ptr(g),
                                                _lib.ptr(d_flow), _lib.ptr(d_img), _lib.ptr(work, 'work', torch.int64),
                                                _lib.stream(img)), 'flow_warp_bwd')
        return d_img, d_flow, None


def euler2mat(angle):
    """Reference inverse_warp.py:82-119 (host-side torch ops; tiny, not on the per-pixel path)."""
    B = angle.size(0)
    x, y, z = angle[:, 0], angle[:, 1], angle[:, 2]
    zeros = z.detach() * 0
    ones = zeros.detach() + 1
    cosz, sinz = torch.cos(z), torch.sin(z)
    zmat = torch.stack([cosz, -sinz, zeros, sinz, cosz, zeros, zeros, zeros, ones], dim=1).view(B, 3, 3)
    cosy, siny = torch.cos(y), torch.sin(y)
    ymat = torch.stack([cosy, zeros, siny, zeros, ones, zeros, -siny, zeros, cosy], dim=1).view(B, 3, 3)
    cosx, sinx = torch.cos(x), torch.sin(x)
    xmat = torch.stack([ones, zeros, zeros, zeros, cosx, -sinx, zeros, sinx, cosx], dim=1).view(B, 3, 3)
    return xmat.bmm(ymat).bmm(zmat)


def quat2mat(quat):
    """Reference inverse_warp.py:122-143."""
    norm_quat = torch.cat([quat[:, :1].detach() * 0 + 1, quat], dim=1)
    norm_quat = norm_quat / norm_quat.norm(p=2, dim=1, keepdim=True)
    w, x, y, z = norm_quat[:, 0], norm_quat[:, 1], norm_quat[:, 2], norm_quat[:, 3]
    B = quat.size(0)
    w2, x2, y2, z2 = w.pow(2), x.pow(2), y.pow(2), z.pow(2)
    wx, wy, wz, xy, xz, yz = w * x, w * y, w * z, x * y, x * z, y * z
    return torch.stack([w2 + x2 - y2 - z2, 2 * xy - 2 * wz, 2 * wy + 2 * xz,
                        2 * wz + 2 * xy, w2 - x2 + y2 - z2, 2 * yz - 2 * wx,
                        2 * xz - 2 * wy, 2 * wx + 2 * yz, w2 - x2 - y2 + z2], dim=1).view(B, 3, 3)


def pose_vec2mat(vec, rotation_mode='euler'):
    """[B,6] -> [B,3,4].  Reference inverse_warp.py:146-162 (used by test_pose.py:77)."""
    translation = vec[:, :3].unsqueeze(-1)
    rot = vec[:, 3:]
    if rotation_mode == 'euler':
        rot_mat = euler2mat(rot)
    elif rotation_mode == 'quat':
        rot_mat = quat2mat(rot)
    return torch.cat([rot_mat, translation], dim=2)


# ---- stand-alone geometry helpers of the reference module (inverse_warp.py:13-79).  Inside the training step these
# are fused into the photometric / warp kernels (csrc/geom.cuh); the module-level functions exist so that code
# importing them by name keeps working.  Plain device-side tensor ops, same arithmetic and shapes as the reference.
pixel_coords = None


def set_id_grid(depth):
    """[1,3,H,W] grid of (x, y, 1) pixel coordinates, cached in the module like the reference (inverse_warp.py:13-20)."""
    global pixel_coords
    b, h, w = depth.size()
    i_range = torch.arange(0, h, device=depth.device).view(1, h, 1).expand(1, h, w).type_as(depth)
    j_range = torch.arange(0, w, device=depth.device).view(1, 1, w).expand(1, h, w).type_as(depth)
    ones = torch.ones(1, h, w, device=depth.device).type_as(depth)
    pixel_coords = torch.stack((j_range, i_range, ones), dim=1)
    return pixel_coords


def pixel2cam(depth, intrinsics_inv):
    """depth [B,H,W], K^-1 [B,3,3] -> camera-frame points [B,3,H,W].  Reference inverse_warp.py:31-45."""
    global pixel_coords
    b, h, w = depth.size()
    if (pixel_coords is None) or pixel_coords.size(2) != h or pixel_coords.size(3) != w or pixel_coords.device != depth.device:
        set_id_grid(depth)
    cur = pixel_coords[:, :, :h, :w].expand(b, 3, h, w).contiguous().view(b, 3, -1)
    return intrinsics_inv.bmm(cur).view(b, 3, h, w) * depth.unsqueeze(1)


def cam2pixel(cam_coords, proj_c2p_rot, proj_c2p_tr, padding_mode):
    """Camera-frame points [B,3,H,W] -> normalised pixel coordinates [B,H,W,2]; 'zeros': out-of-range coordinates are
    rewritten to 2 (no gradient through the rewrite).  Reference inverse_warp.py:48-79."""
    b, _, h, w = cam_coords.size()
    flat = cam_coords.view(b, 3, -1)
    pcoords = proj_c2p_rot.bmm(flat) if proj_c2p_rot is not None else flat
    if proj_c2p_tr is not None:
        pcoords = pcoords + proj_c2p_tr
    X, Y, Z = pcoords[:, 0], pcoords[:, 1], pcoords[:, 2].clamp(min=1e-3)
    X_norm = 2 * (X / Z) / (w - 1) - 1
    Y_norm = 2 * (Y / Z) / (h - 1) - 1
    if padding_mode == 'zeros':
        X_norm = torch.where(((X_norm > 1) | (X_norm < -1)).detach(), torch.full_like(X_norm, 2), X_norm)
        Y_norm = torch.where(((Y_norm > 1) | (Y_norm < -1)).detach(), torch.full_like(Y_norm, 2), Y_norm)
    return torch.stack([X_norm, Y_norm], dim=2).view(b, h, w, 2)


def inverse_warp(img, depth, pose, intrinsics, intrinsics_inv, rotation_mode='euler', padding_mode='zeros'):
    """Inverse warp a source image to the target image plane.  Reference inverse_warp.py:250-283."""
    check_sizes(img, 'img', 'B3HW')
    check_sizes(depth, 'depth', 'BHW')
    check_sizes(pose, 'pose', 'B6')
    check_sizes(intrinsics, 'intrinsics', 'B33')
    check_sizes(intrinsics_inv, 'intrinsics', 'B33')
    assert(intrinsics_inv.size() == intrinsics.size())
    return _InverseWarp.apply(img, depth, pose, intrinsics, intrinsics_inv, _ROT[rotation_mode], _PAD[padding_mode])


def flow_warp(img, flow, padding_mode='zeros'):
    """Reference inverse_warp.py:164-192."""
    check_sizes(img, 'img', 'BCHW')
    check_sizes(flow, 'flow', 'B2HW')
    return _FlowWarp.apply(img, flow, _PAD[padding_mode])


def pose2flow(depth, pose, intrinsics, intrinsics_inv, rotation_mode='euler', padding_mode=None):
    """Converts pose parameters to rigid optical flow.  Reference inverse_warp.py:195-220."""
    check_sizes(depth, 'depth', 'BHW')
    check_sizes(pose, 'pose', 'B6')
    check_sizes(intrinsics, 'intrinsics', 'B33')
    check_sizes(intrinsics_inv, 'intrinsics', 'B33')
    assert(intrinsics_inv.size() == intrinsics.size())
    return _Pose2Flow.apply(depth, pose, intrinsics, intrinsics_inv, _ROT[rotation_mode], _PAD[padding_mode])


def flow2oob(flow):
    """Boolean out-of-bounds map (validation only).  Reference inverse_warp.py:222-238."""
    check_sizes(flow, 'flow', 'B2HW')
    bs, _, h, w = flow.size()
    u, v = flow[:, 0], flow[:, 1]
    gx = torch.arange(0, w, device=flow.device, dtype=flow.dtype).view(1, 1, w).expand_as(u)
    gy = torch.arange(0, h, device=flow.device, dtype=flow.dtype).view(1, h, 1).expand_as(v)
    X = 2 * ((gx + u) / (w - 1.0) - 0.5)
    Y = 2 * ((gy + v) / (h - 1.0) - 0.5)
    return (X.abs() > 1).add(Y.abs() > 1) > 0
