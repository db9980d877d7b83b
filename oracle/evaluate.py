"""Oracle: the per-sample bodies of the reference's evaluation scripts (test_disp.py:84-150,171-187;
test_pose.py:50-90,107-122; test_flow.py:112-140) restated on the functional oracle nets.  TEST INFRASTRUCTURE."""
import numpy as np
import torch
from . import nets as ON, geometry as OG, metrics as OM


def _inp(img):
    t = torch.from_numpy(np.ascontiguousarray(np.transpose(np.asarray(img, np.float32), (2, 0, 1)))).unsqueeze(0)
    return (t / 255 - 0.5) / 0.5


def compute_errors(gt, pred):
    """test_disp.py:171-187."""
    thresh = np.maximum((gt / pred), (pred / gt))
    a1 = (thresh < 1.25).mean()
    a2 = (thresh < 1.25 ** 2).mean()
    a3 = (thresh < 1.25 ** 3).mean()
    rmse = np.sqrt(((gt - pred) ** 2).mean())
    rmse_log = np.sqrt(((np.log(gt) - np.log(pred)) ** 2).mean())
    abs_rel = np.mean(np.abs(gt - pred) / gt)
    sq_rel = np.mean(((gt - pred) ** 2) / gt)
    return abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3


def depth_sample_errors(Pd, tgt_img, gt_depth, mask, min_depth, max_depth, Pp=None, ref_imgs=None, displacements=None):
    """test_disp.py:84-150 for one sample."""
    from scipy.ndimage import zoom
    with torch.no_grad():
        tgt = _inp(tgt_img)
        pred_disp = ON.disp_forward(Pd, tgt, training=False).numpy()[0, 0]
        pred_depth = 1 / pred_disp
        z = zoom(pred_depth, (gt_depth.shape[0] / pred_depth.shape[0], gt_depth.shape[1] / pred_depth.shape[1])).clip(min_depth, max_depth)
        gt = gt_depth
        if mask is not None:
            z, gt = z[mask], gt[mask]
        errors = np.zeros((2, 7), np.float32)
        if Pp is not None:
            poses = ON.pose_forward(Pp, tgt, [_inp(r) for r in ref_imgs])
            d = poses[0, :, :3].norm(2, 1).numpy()
            sf = [s1 / s2 for s1, s2 in zip(displacements, d) if s1 > 0]
            errors[0] = compute_errors(gt, z * (np.mean(sf) if len(sf) > 0 else 0))
        errors[1] = compute_errors(gt, z * (np.median(gt) / np.median(z)))
    return errors


def compute_pose_error(gt, pred):
    """test_pose.py:107-122."""
    RE = 0
    snippet_length = gt.shape[0]
    scale_factor = np.sum(gt[:, :, -1] * pred[:, :, -1]) / np.sum(pred[:, :, -1] ** 2)
    ATE = np.linalg.norm((gt[:, :, -1] - scale_factor * pred[:, :, -1]).reshape(-1))
    for gt_pose, pred_pose in zip(gt, pred):
        R = gt_pose[:, :3] @ np.linalg.inv(pred_pose[:, :3])
        s = np.linalg.norm([R[0, 1] - R[1, 0], R[1, 2] - R[2, 1], R[0, 2] - R[2, 0]])
        c = np.trace(R) - 1
        RE += np.arctan2(s, c)
    return ATE / snippet_length, RE / snippet_length


def pose_snippet_errors(Pp, imgs, gt_poses, rotation_mode='euler'):
    """test_pose.py:50-90 for one snippet."""
    with torch.no_grad():
        ts = [_inp(i) for i in imgs]
        mid = len(ts) // 2
        poses = ON.pose_forward(Pp, ts[mid], ts[:mid] + ts[mid + 1:])[0]
        poses = torch.cat([poses[:mid], torch.zeros(1, 6).float(), poses[mid:]])
        inv_t = OG.pose_vec2mat(poses, rotation_mode=rotation_mode).numpy().astype(np.float64)
    rot = np.linalg.inv(inv_t[:, :, :3])
    tr = -rot @ inv_t[:, :, -1:]
    tm = np.concatenate([rot, tr], axis=-1)
    first = inv_t[0]
    final = first[:, :3] @ tm
    final[:, :, -1:] += first[:, -1:]
    return compute_pose_error(gt_poses, final) + (final,)


def flow_sample_errors(P, tgt, refs, K, Kinv, flow_gt, obj_map_gt, THRESH=0.01, flownet='Back2Future'):
    """test_flow.py:112-140 for one sample; P = {'disp','pose','mask','flow'} parameter dicts, P['flow'] of `flownet`."""
    with torch.no_grad():
        disp = ON.disp_forward(P['disp'], tgt, training=False)
        depth = 1 / disp
        pose = ON.pose_forward(P['pose'], tgt, refs)
        emask = ON.mask_forward(P['mask'], tgt, refs, training=False)
        flow_fwd = ON.flow_eval(P['flow'], tgt, refs, flownet)
        flow_cam = OG.pose2flow(depth.squeeze(1), pose[:, 2], K, Kinv)
        rigidity_mask = 1 - (1 - emask[:, 1]) * (1 - emask[:, 2]).unsqueeze(1) > 0.5
        soft = (flow_cam - flow_fwd).abs()
        census = (soft[:, 0] < THRESH).type_as(flow_fwd) * (soft[:, 1] < THRESH).type_as(flow_fwd)
        combined = 1 - (1 - rigidity_mask.type_as(emask)) * (1 - census.type_as(emask))
        non_rigid = (combined <= THRESH).type_as(flow_fwd).expand_as(flow_fwd) * flow_fwd
        rigid = (combined > THRESH).type_as(flow_cam).expand_as(flow_cam) * flow_cam
        total = rigid + non_rigid
        obj = obj_map_gt.unsqueeze(1).type_as(flow_fwd)
        errs = list(OM.compute_all_epes(flow_gt, flow_cam, flow_fwd, combined)) + list(OM.compute_all_epes(flow_gt, flow_cam, flow_fwd, 1 - obj))
    return errs, total
