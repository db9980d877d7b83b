"""Per-sample cores of the reference's evaluation scripts (SURVEY.md row N3) on the libccb200 forward kernels:

  depth_sample_errors   test_disp.py:84-150 (+ compute_errors :171-187)   abs_rel sq_rel rms log_rms a1 a2 a3
  pose_snippet_errors   test_pose.py:50-90  (+ compute_pose_error :107-122) ATE, RE of one snippet
  flow_sample_errors    test_flow.py:112-140                               the 8 EPE / Fl numbers of one KITTI-2015 pair

The scripts' dataset crawlers, image IO and visualisation are out of scope (SURVEY.md section 2); these functions take what the
reference's `test_framework` iterators yield (uint8 HxWx3 frames, ground truth arrays) and return what the scripts
accumulate, so a maintainer swaps the loop body.  Nets run in eval mode through the CUDA kernels; the spline `zoom` of
the predicted depth to the ground-truth size (scipy, order 3) and the 3x4 pose algebra stay on the host like in the
reference - they are a few hundred flops per sample."""
import numpy as np
import torch
from .inverse_warp import pose2flow, pose_vec2mat
from . import loss_functions as LF, models


def _to_net_input(img_hwc, device):
    """uint8/float HxWx3 -> [1,3,H,W] in [-1,1]: ((x/255 - 0.5)/0.5), test_disp.py:97-99."""
    t = torch.from_numpy(np.ascontiguousarray(np.transpose(np.asarray(img_hwc, np.float32), (2, 0, 1)))).unsqueeze(0)
    return ((t / 255 - 0.5) / 0.5).to(device)


def compute_errors_np(gt, pred):
    """test_disp.py:171-187 (numpy, on the masked 1-D arrays)."""
    thresh = np.maximum(gt / pred, pred / gt)
    a1, a2, a3 = (thresh < 1.25).mean(), (thresh < 1.25 ** 2).mean(), (thresh < 1.25 ** 3).mean()
    rmse = np.sqrt(((gt - pred) ** 2).mean())
    rmse_log = np.sqrt(((np.log(gt) - np.log(pred)) ** 2).mean())
    return np.mean(np.abs(gt - pred) / gt), np.mean(((gt - pred) ** 2) / gt), rmse, rmse_log, a1, a2, a3


@torch.no_grad()
def depth_sample_errors(disp_net, tgt_img, gt_depth, mask=None, min_depth=1e-3, max_depth=80.0, pose_net=None, ref_imgs=None,
                        displacements=None, device=None):
    """-> float32 [2,7]: row 0 scaled by the PoseNet displacement ratio (zeros without a pose net), row 1 by the
    median ratio (test_disp.py:129-150)."""
    from scipy.ndimage import zoom
    device = device or next(disp_net.parameters()).device
    disp_net.eval()
    tgt = _to_net_input(tgt_img, device)
    pred_disp = disp_net(tgt)[0, 0].float().cpu().numpy()
    pred_depth = 1 / pred_disp
    z = zoom(pred_depth, (gt_depth.shape[0] / pred_depth.shape[0], gt_depth.shape[1] / pred_depth.shape[1])).clip(min_depth, max_depth)
    gt = gt_depth
    if mask is not None:
        z, gt = z[mask], gt[mask]
    out = np.zeros((2, 7), np.float32)
    if pose_net is not None:
        pose_net.eval()
        refs = [_to_net_input(r, device) for r in ref_imgs]
        res = pose_net(tgt, refs)
        poses = res[1] if isinstance(res, tuple) else res           # PoseExpNet returns (mask, pose)
        disp_pred = poses[0, :, :3].norm(2, 1).cpu().numpy()
        sf = [s1 / s2 for s1, s2 in zip(displacements, disp_pred) if s1 > 0]
        out[0] = compute_errors_np(gt, z * (np.mean(sf) if len(sf) > 0 else 0))
    out[1] = compute_errors_np(gt, z * (np.median(gt) / np.median(z)))
    return out


def compute_pose_error(gt, pred):
    """ATE / RE of one snippet, test_pose.py:107-122."""
    n = gt.shape[0]
    scale = np.sum(gt[:, :, -1] * pred[:, :, -1]) / np.sum(pred[:, :, -1] ** 2)
    ate = np.linalg.norm((gt[:, :, -1] - scale * pred[:, :, -1]).reshape(-1))
    re = 0.0
    for g, p in zip(gt, pred):
        R = g[:, :3] @ np.linalg.inv(p[:, :3])
        s = np.linalg.norm([R[0, 1] - R[1, 0], R[1, 2] - R[2, 1], R[0, 2] - R[2, 0]])
        re += np.arctan2(s, np.trace(R) - 1)
    return ate / n, re / n


@torch.no_grad()
def pose_snippet_errors(pose_net, imgs, gt_poses, rotation_mode='euler', device=None):
    """imgs: odd-length list of HxWx3 frames (target = the middle one); gt_poses [len,3,4] -> (ATE, RE, final_poses)."""
    device = device or next(pose_net.parameters()).device
    pose_net.eval()
    ts = [_to_net_input(i, device) for i in imgs]
    mid = len(ts) // 2
    res = pose_net(ts[mid], ts[:mid] + ts[mid + 1:])
    poses = (res[1] if isinstance(res, tuple) else res)[0].float().cpu()
    poses = torch.cat([poses[:mid], torch.zeros(1, 6), poses[mid:]])
    inv_t = pose_vec2mat(poses.to(device), rotation_mode=rotation_mode).cpu().numpy().astype(np.float64)
    rot = np.linalg.inv(inv_t[:, :, :3])
    tr = -rot @ inv_t[:, :, -1:]
    tm = np.concatenate([rot, tr], axis=-1)
    first = inv_t[0]
    final = first[:, :3] @ tm
    final[:, :, -1:] += first[:, -1:]
    ate, re = compute_pose_error(gt_poses, final)
    return ate, re, final


@torch.no_grad()
def flow_sample_errors(disp_net, pose_net, mask_net, flow_net, tgt, refs, K, Kinv, flow_gt, obj_map_gt, THRESH=0.01):
    """tgt/refs: normalised device tensors [1,3,H,W] (4 refs), flow_gt [1,3,Hg,Wg], obj_map_gt [1,Hg,Wg] ->
    [epe_total, epe_sp, epe_mv, Fl] with the learned rigidity mask and the same four with the ground-truth object map
    (test_flow.py:112-140), plus the composed flow."""
    for n in (disp_net, pose_net, mask_net, flow_net):
        n.eval()
    disp = disp_net(tgt)
    depth = 1 / disp
    pose = pose_net(tgt, refs)
    emask = mask_net(tgt, refs)
    # test_flow.py:122-125: Back2Future takes both neighbours, another flow net (FlowNetC6) the forward one
    flow_fwd = flow_net(tgt, refs[1:3])[0] if isinstance(flow_net, models.Back2Future) else flow_net(tgt, refs[2])
    flow_cam = pose2flow(depth.squeeze(1), pose[:, 2], K, Kinv)
    rigidity = (1 - (1 - emask[:, 1]) * (1 - emask[:, 2])).unsqueeze(1) > 0.5
    soft = (flow_cam - flow_fwd).abs()
    census = (soft[:, 0] < THRESH).type_as(flow_fwd) * (soft[:, 1] < THRESH).type_as(flow_fwd)
    combined = 1 - (1 - rigidity.type_as(emask)) * (1 - census.type_as(emask))
    non_rigid = (combined <= THRESH).type_as(flow_fwd).expand_as(flow_fwd) * flow_fwd
    rigid = (combined > THRESH).type_as(flow_cam).expand_as(flow_cam) * flow_cam
    total = rigid + non_rigid
    obj = obj_map_gt.unsqueeze(1).type_as(flow_fwd)
    errs = list(LF.compute_all_epes(flow_gt, flow_cam, flow_fwd, combined)) + list(LF.compute_all_epes(flow_gt, flow_cam, flow_fwd, 1 - obj))
    return errs, total
