"""Per-sample cores of the reference's evaluation scripts (SURVEY.md row N3) on the libccb200 forward kernels:

  depth_sample_errors   test_disp.py:84-150 (+ compute_errors :171-187)   abs_rel sq_rel rms log_rms a1 a2 a3
  pose_snippet_errors   test_pose.py:50-90  (+ compute_pose_error :107-122) ATE, RE of one snippet
  flow_sample_errors    test_flow.py:112-140                               the 8 EPE / Fl numbers of one KITTI-2015 pair
  mask_sample_errors    test_mask.py:119-156 (+ mask_error :224-262)       tp fp fn per class of the three rigidity masks
                        (motion_mask_counts: the masks and counts alone; mask_iou: the script's final IoUs :199-201)
  flow_submission_sample  submit_flow.py:109-175                           KITTI-2015 test-set files of one sample
                        (flow_submission, flow_colors: the fused kernels; write_flow_submission: the script's files;
                        kitti_flow_errors: evaluate_flow.py compute_err :44-53 of decoded 16-bit PNGs)

The scripts' dataset crawlers, image IO and visualisation are out of scope (SURVEY.md section 2); these functions take what the
reference's `test_framework` iterators yield (uint8 HxWx3 frames, ground truth arrays) and return what the scripts
accumulate, so a maintainer swaps the loop body.  Nets run in eval mode through the CUDA kernels; the spline `zoom` of
the predicted depth to the ground-truth size (scipy, order 3) and the 3x4 pose algebra stay on the host like in the
reference - they are a few hundred flops per sample."""
import numpy as np
import torch
from .inverse_warp import pose2flow, pose_vec2mat
from . import _lib, loss_functions as LF, models


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


@torch.no_grad()
def motion_mask_counts(emask, flow_cam, flow_fwd, obj_map_gt, semantic_map_gt, THRESH=0.94, want_masks=False):
    """The rigidity masks of test_mask.py:129-134 and mask_error (:224-262) of each against the ground truth, per sample,
    in one fused call (ccb_mask_iou): emask [B,C,h,w] the mask net's eval output, flow_cam / flow_fwd [B,2,h,w], obj_map_gt /
    semantic_map_gt [B,Hg,Wg] -> int64 [B,3,6] on the device: for combined, census and bare the script's
    [tp_0, fp_0, fn_0, tp_1, fp_1, fn_1] (class 0 = rigid background, class 1 = moving car; pixels whose semantic label is
    not 26 are ignored).  The maximum that normalises the census is taken per sample; the reference runs batch 1.
    want_masks: also [B,4,h,w] = combined, census, bare (0/1) and the soft census.  No host synchronisation."""
    emask, flow_cam, flow_fwd = (_lib.f32(t) for t in (emask, flow_cam, flow_fwd))
    obj, sem = _lib.f32(obj_map_gt), _lib.f32(semantic_map_gt)
    B, C, h, w = (int(v) for v in emask.shape)
    Hg, Wg = int(obj.shape[1]), int(obj.shape[2])
    assert flow_cam.shape == (B, 2, h, w) and flow_fwd.shape == (B, 2, h, w), (flow_cam.shape, flow_fwd.shape)
    assert obj.shape == (B, Hg, Wg) and sem.shape == (B, Hg, Wg), (obj.shape, sem.shape)
    nbytes = int(_lib.call('ccb_mask_iou_workspace_bytes', B, h, w, Hg, Wg))
    work = torch.empty(max(nbytes, 0) // 8 + 1, device=emask.device, dtype=torch.int64)
    n = torch.empty(B, 3, 4, device=emask.device, dtype=torch.int64)
    masks = torch.empty(B, 4, h, w, device=emask.device) if want_masks else None
    _lib.call('ccb_mask_iou', emask, flow_cam, flow_fwd, obj, sem, B, C, h, w, Hg, Wg, float(THRESH), 26, masks, work, nbytes, n,
              emask)
    # n[pred][gt] = n00 n01 n10 n11 -> tp_0 fp_0 fn_0 tp_1 fp_1 fn_1: fp_1 = fn_0 = n10, fn_1 = fp_0 = n01
    counts = torch.cat([n, n[..., 2:3], n[..., 1:2]], -1)
    return (counts, masks) if want_masks else counts


@torch.no_grad()
def mask_sample_errors(disp_net, pose_net, mask_net, flow_net, tgt, refs, K, Kinv, obj_map_gt, semantic_map_gt, THRESH=0.94):
    """tgt/refs: normalised device tensors [1,3,H,W] (4 refs), obj_map_gt / semantic_map_gt [1,Hg,Wg] ->
    (errors, errors_census, errors_bare, masks): the three lists of six counts test_mask.py:150-152 accumulates, and
    masks [1,4,H,W] on the device (combined is what the script saves, the soft census what it draws)."""
    for n in (disp_net, pose_net, mask_net, flow_net):
        n.eval()
    disp = disp_net(tgt)
    depth = 1 / disp
    pose = pose_net(tgt, refs)
    emask = mask_net(tgt, refs)
    # test_mask.py:123-126: Back2Future takes both neighbours, another flow net (FlowNetC6) the forward one
    flow_fwd = flow_net(tgt, refs[1:3])[0] if isinstance(flow_net, models.Back2Future) else flow_net(tgt, refs[2])
    flow_cam = pose2flow(depth.squeeze(1), pose[:, 2], K, Kinv)
    counts, masks = motion_mask_counts(emask, flow_cam, flow_fwd, obj_map_gt, semantic_map_gt, THRESH, want_masks=True)
    errors, errors_census, errors_bare = counts[0].cpu().tolist()
    return errors, errors_census, errors_bare, masks


def mask_iou(summed_counts):
    """[tp_0, fp_0, fn_0, tp_1, fp_1, fn_1] summed over a dataset -> (avg_iou, bg_iou, fg_iou), test_mask.py:199-201.
    A class with no pixel at all gives nan."""
    c = np.asarray(summed_counts, np.float64)
    with np.errstate(divide='ignore', invalid='ignore'):
        bg_iou = c[0] / (c[0] + c[1] + c[2])
        fg_iou = c[3] / (c[3] + c[4] + c[5])
    return float((bg_iou + fg_iou) / 2), float(bg_iou), float(fg_iou)


@torch.no_grad()
def flow_submission(emask, flow_cam, flow_fwd, Hg, Wg, THRESH=0.01, want_full=False):
    """The per-sample files of submit_flow.py:119-156 in one fused call (ccb_flow_submit): emask [B,C,h,w], flow_cam /
    flow_fwd [B,2,h,w] at the nets' resolution -> dict of device tensors:
      mask [B,1,h,w]        the combined rigidity mask (what the script saves as mask/NNN.npy)
      png  [B,Hg,Wg,3]      uint16 KITTI triplet of the full-resolution total flow (testing/NNNNNN_10.png)
      flo  [B,Hg,Wg,2]      fp32 payload of testing_flo/NNNNNN_10.flo
      full [B,3,2,Hg,Wg]    (want_full) the cam, fwd and total flows at full resolution, scaled as the script scales them
    No host synchronisation."""
    emask, flow_cam, flow_fwd = (_lib.f32(t) for t in (emask, flow_cam, flow_fwd))
    B, C, h, w = (int(v) for v in emask.shape)
    assert flow_cam.shape == (B, 2, h, w) and flow_fwd.shape == (B, 2, h, w), (flow_cam.shape, flow_fwd.shape)
    dev = emask.device
    out = dict(mask=torch.empty(B, 1, h, w, device=dev), png=torch.empty(B, Hg, Wg, 3, device=dev, dtype=torch.uint16),
               flo=torch.empty(B, Hg, Wg, 2, device=dev))
    if want_full:
        out['full'] = torch.empty(B, 3, 2, Hg, Wg, device=dev)
    _lib.call('ccb_flow_submit', emask, flow_cam, flow_fwd, B, C, h, w, int(Hg), int(Wg), float(THRESH), out['mask'],
              out.get('full'), out['png'], out['flo'], emask)
    return out


@torch.no_grad()
def flow_colors(flow):
    """Middlebury colours (flowlib.flow_to_image) on the device (ccb_flow_color): flow [B,P,2,H,W] -> uint8 [B,3,P*H,W],
    the P panels of each image stacked along H as np.hstack stacks [2,H,W] arrays and normalised by one maximum radius.
    The levels are the reference's float image times 255.  No host synchronisation."""
    flow = _lib.f32(flow)
    B, P, two, H, W = (int(v) for v in flow.shape)
    assert two == 2, flow.shape
    nbytes = int(_lib.call('ccb_flow_color_workspace_bytes', B, P, H, W))
    work = torch.empty(max(nbytes, 0) // 8 + 1, device=flow.device, dtype=torch.int64)
    out = torch.empty(B, 3, P * H, W, device=flow.device, dtype=torch.uint8)
    _lib.call('ccb_flow_color', flow, B, P, H, W, work, nbytes, out, flow)
    return out


@torch.no_grad()
def flow_submission_sample(disp_net, pose_net, mask_net, flow_net, tgt, refs, K, Kinv, Hg, Wg, THRESH=0.01, want_viz=False):
    """submit_flow.py:109-175 for one batch: tgt/refs normalised device tensors [B,3,h,w] (4 refs), (Hg, Wg) the original
    frame size -> flow_submission's dict of device tensors; want_viz adds 'full' and 'viz' = uint8 [B,3,3*Hg,Wg], row 2
    of the script's visualisation (cam, fwd and total flow stacked, one radius).  Row 1 (matplotlib's magma map of the
    target, disparity and mask) is not produced.  No host synchronisation."""
    for n in (disp_net, pose_net, mask_net, flow_net):
        n.eval()
    disp = disp_net(tgt)
    depth = 1 / disp
    pose = pose_net(tgt, refs)
    emask = mask_net(tgt, refs)
    # submit_flow.py:113-116: Back2Future takes both neighbours, another flow net (FlowNetC6) the forward one
    flow_fwd = flow_net(tgt, refs[1:3])[0] if isinstance(flow_net, models.Back2Future) else flow_net(tgt, refs[2])
    flow_cam = pose2flow(depth.squeeze(1), pose[:, 2], K, Kinv)
    out = flow_submission(emask, flow_cam, flow_fwd, Hg, Wg, THRESH, want_full=want_viz)
    if want_viz:
        out['viz'] = flow_colors(out['full'])
    return out


def write_flow_submission(out_dir, i, sample, tgt):
    """Sample `i` (batch 1) of flow_submission_sample written as submit_flow.py:150-175 names it under `out_dir`:
    images/iii.npy (the normalised target [3,h,w]), mask/iii.npy (the combined mask [1,h,w]), testing/iiiiii_10.png
    (16-bit KITTI flow), testing_flo/iiiiii_10.flo and, when the sample has it, viz/iii02.png (8-bit RGB)."""
    import os
    from .flowutils import flow_io
    for sub in ('images', 'mask', 'viz', 'testing', 'testing_flo'):
        os.makedirs(os.path.join(out_dir, sub), exist_ok=True)
    np.save(os.path.join(out_dir, 'images', str(i).zfill(3)), tgt[0].detach().cpu().numpy())
    np.save(os.path.join(out_dir, 'mask', str(i).zfill(3)), sample['mask'][0].cpu().numpy())
    flow_io.write_png(os.path.join(out_dir, 'testing', str(i).zfill(6) + '_10.png'), sample['png'][0].cpu().numpy())
    flow_io.write_flo_payload(os.path.join(out_dir, 'testing_flo', str(i).zfill(6) + '_10.flo'), sample['flo'][0].cpu().numpy())
    if 'viz' in sample:
        flow_io.write_png(os.path.join(out_dir, 'viz', str(i).zfill(3) + '02.png'),
                          np.ascontiguousarray(sample['viz'][0].cpu().numpy().transpose(1, 2, 0)))


@torch.no_grad()
def kitti_flow_errors(gt_png, pred_png):
    """evaluate_flow.py compute_err (:44-53) of decoded KITTI flow images on the device (ccb_kitti_flow_errors): gt_png and
    pred_png uint16 [B,H,W,3] (or [H,W,3]; numpy arrays are copied to the current CUDA device) -> (errors fp64 [B,2] =
    aepe, Fl; counts int64 [B,2] = outliers, valid pixels), both on the device.  The script averages the per-image rows."""
    dev = pred_png.device if torch.is_tensor(pred_png) else (torch.device('cpu') if _lib.is_simulator() else torch.device('cuda'))
    gt, pred = (torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a).to(dev).contiguous() for a in (gt_png, pred_png))
    if gt.dim() == 3:
        gt, pred = gt[None], pred[None]
    assert gt.shape == pred.shape and gt.shape[-1] == 3 and gt.dtype == torch.uint16, (gt.shape, pred.shape, gt.dtype)
    B, H, W = (int(v) for v in gt.shape[:3])
    nbytes = int(_lib.call('ccb_kitti_flow_errors_workspace_bytes', B, H, W))
    work = torch.empty(max(nbytes, 0) // 8 + 1, device=dev, dtype=torch.int64)
    out = torch.empty(B, 2, device=dev, dtype=torch.float64)
    counts = torch.empty(B, 2, device=dev, dtype=torch.int64)
    _lib.call('ccb_kitti_flow_errors', gt, pred, B, H, W, work, nbytes, out, counts, gt)
    return out, counts
