"""Per-sample cores of the reference's evaluation scripts (SURVEY.md row N3) on the libccb200 forward kernels:

  depth_sample_errors   test_disp.py:84-150 (+ compute_errors :171-187)   abs_rel sq_rel rms log_rms a1 a2 a3
  pose_snippet_errors   test_pose.py:50-90  (+ compute_pose_error :107-122) ATE, RE of one snippet
  flow_sample_errors    test_flow.py:112-140                               the 8 EPE / Fl numbers of one KITTI-2015 pair
  mask_sample_errors    test_mask.py:119-156 (+ mask_error :224-262)       tp fp fn per class of the three rigidity masks
                        (motion_mask_counts: the masks and counts alone; mask_iou: the script's final IoUs :199-201)
  flow_submission_sample  submit_flow.py:109-175                           KITTI-2015 test-set files of one sample
                        (flow_submission, flow_colors: the fused kernels; write_flow_submission: the script's files;
                        kitti_flow_errors: evaluate_flow.py compute_err :44-53 of decoded 16-bit PNGs)
  colorize              utils.py tensor2array's 'bone' and 'rainbow' colormaps as run_inference.py saves them, in one
                        call for a batch (colormap_table: matplotlib's lookup tables as uint8; cc_b200.run_inference
                        runs the script)
  depth_eval_batch      test_disp.py:98-141 for a batch on the device, no host synchronisation
                        (velodyne_depth: generate_depth_map's ground truth; spline_zoom: scipy's zoom(order=3);
                        depth_errors: both scalings and compute_errors; depth_summary: the script's printed rows;
                        kitti_depth_framework / stillbox_depth_framework: the two test_frameworks' files and
                        displacements; cc_b200.test_disp runs the script)
  make3d_eval_batch     test_make3d.py:97-148 for a batch on the device, no host synchronisation
                        (make3d_files / load_make3d: test_framework's files and samples; make3d_frames: imresize's contrast
                        stretch, Pillow's resize and the normalisation; make3d_depth_errors: the capped median scaling and
                        compute_errors :174-190 with log10; depth_summary: the printed row, row 1)
  pose_eval_batch       test_pose.py:50-92 / test_sintel_pose.py:55-97 for a batch of snippets on the device, no host
                        synchronisation (kitti_pose_framework / sintel_pose_framework: the frameworks' files, snippets and
                        compensated ground truth, load_pose_frames; pose_errors: the pose algebra, ATE and RE in one kernel;
                        load_pose_net; pose_summary: the printed rows; write_pose_predictions: predictions.npy)
  flow_eval_batch       test_flow.py:112-140 (and train.py's validate_flow_with_gt) for a batch of KITTI-2015 samples on the
  back2future_eval_batch  device, no host synchronisation; test_back2future.py with the flow net alone
                        (kitti_flow_framework / load_kitti_flow_samples: ValidationFlow's files and samples, grouped by
                        frame size; flow_eval: the rigidity masks and both compute_all_epes in one kernel;
                        load_flow_eval_nets; flow_summary: the printed row; write_flow_eval_outputs: --output-dir's files)

The scripts' dataset crawlers, image IO and visualisation are out of scope (SURVEY.md section 2); these functions take what the
reference's `test_framework` iterators yield (uint8 HxWx3 frames, ground truth arrays) and return what the scripts
accumulate, so a maintainer swaps the loop body.  Nets run in eval mode through the CUDA kernels; the spline `zoom` of
the predicted depth to the ground-truth size (scipy, order 3) and the 3x4 pose algebra stay on the host like in the
reference in the per-sample cores; depth_eval_batch does the depth sample on the device."""
import numpy as np
import torch
from .inverse_warp import pose2flow, pose_vec2mat
from . import _lib, loss_functions as LF, models
from .input_pipeline import device_tensor, flow_intrinsics, scale_frames


def _to_net_input(img_hwc, device):
    """uint8/float HxWx3 -> [1,3,H,W] in [-1,1]: ((x/255 - 0.5)/0.5), test_disp.py:97-99."""
    t = torch.from_numpy(np.ascontiguousarray(np.transpose(np.asarray(img_hwc, np.float32), (2, 0, 1)))).unsqueeze(0)
    return ((t / 255 - 0.5) / 0.5).to(device)


def _pose(res):
    """The pose of a pose net's output: PoseExpNet returns (mask, pose), PoseNet the pose alone."""
    return res[1] if isinstance(res, tuple) else res


def _flow_nets(disp_net, pose_net, mask_net, flow_net, tgt, refs, K, Kinv, spatial_normalize=False):
    """The four nets in eval mode on tgt and its 4 refs -> (emask, flow_cam, flow_fwd): the mask net's output, the camera
    flow of the depth and the pose to ref 2, and the flow net's forward flow (test_flow.py:112-125, test_mask.py:119-126,
    submit_flow.py:109-116); spatial_normalize divides the disparity by its mean first (train.py:665-669)."""
    for n in (disp_net, pose_net, mask_net, flow_net):
        n.eval()
    disp = disp_net(tgt)
    if spatial_normalize:
        disp = LF.spatial_normalize(disp)
    depth = 1 / disp
    pose = pose_net(tgt, refs)
    emask = mask_net(tgt, refs)
    # Back2Future takes both neighbours, another flow net (FlowNetC6) the forward one
    flow_fwd = flow_net(tgt, refs[1:3])[0] if isinstance(flow_net, models.Back2Future) else flow_net(tgt, refs[2])
    flow_cam = pose2flow(depth.squeeze(1), pose[:, 2], K, Kinv)
    return emask, flow_cam, flow_fwd


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
        poses = _pose(pose_net(tgt, refs))
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
    poses = _pose(pose_net(ts[mid], ts[:mid] + ts[mid + 1:]))[0].float().cpu()
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
    emask, flow_cam, flow_fwd = _flow_nets(disp_net, pose_net, mask_net, flow_net, tgt, refs, K, Kinv)
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
    work, nbytes = _lib.workspace('ccb_mask_iou_workspace_bytes', B, h, w, Hg, Wg, like=emask)
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
    emask, flow_cam, flow_fwd = _flow_nets(disp_net, pose_net, mask_net, flow_net, tgt, refs, K, Kinv)
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
    work, nbytes = _lib.workspace('ccb_flow_color_workspace_bytes', B, P, H, W, like=flow)
    out = torch.empty(B, 3, P * H, W, device=flow.device, dtype=torch.uint8)
    _lib.call('ccb_flow_color', flow, B, P, H, W, work, nbytes, out, flow)
    return out


# ------------------------------------------------------------------------------------------------
# utils.py tensor2array's colormaps (run_inference.py): matplotlib's lookup tables built on the host, the lookup on the device

# matplotlib's _bone_data (cm.get_cmap('bone', 10000)) and utils.py opencv_rainbow()'s stops (from_list(..., N=1000)):
# per channel the (x, y0, y1) rows of LinearSegmentedColormap's segment data, and the table size
_BONE = ([(0., 0., 0.), (0.746032, 0.652778, 0.652778), (1.0, 1.0, 1.0)],
         [(0., 0., 0.), (0.365079, 0.319444, 0.319444), (0.746032, 0.777778, 0.777778), (1.0, 1.0, 1.0)],
         [(0., 0., 0.), (0.365079, 0.444444, 0.444444), (1.0, 1.0, 1.0)])
_RAINBOW_STOPS = ((0.000, (1.00, 0.00, 0.00)), (0.400, (1.00, 1.00, 0.00)), (0.600, (0.00, 1.00, 0.00)),
                  (0.800, (0.00, 0.00, 1.00)), (1.000, (0.60, 0.00, 1.00)))
# matplotlib's _hot_data (cm.get_cmap('hot'), N = 256): test_disp.py's --output-dir images
_HOT = ([(0., 0.0416, 0.0416), (0.365079, 1.0, 1.0), (1.0, 1.0, 1.0)],
        [(0., 0., 0.), (0.365079, 0., 0.), (0.746032, 1.0, 1.0), (1.0, 1.0, 1.0)],
        [(0., 0., 0.), (0.746032, 0., 0.), (1.0, 1.0, 1.0)])
COLORMAPS = {'bone': (_BONE, 10000),
             'rainbow': (tuple([(x, c[k], c[k]) for x, c in _RAINBOW_STOPS] for k in range(3)), 1000),
             'hot': (_HOT, 256)}


def _segment_table(N, data):
    """matplotlib's _create_lookup_table(N, data) with gamma 1: fp64 [N] in [0, 1]."""
    a = np.array(data, np.float64)
    x, y0, y1 = a[:, 0] * (N - 1), a[:, 1], a[:, 2]
    xind = (N - 1) * np.linspace(0, 1, N)
    ind = np.searchsorted(x, xind)[1:-1]
    distance = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
    lut = np.concatenate([[y1[0]], distance * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]])
    return np.clip(lut, 0.0, 1.0)


def colormap_table(name):
    """The uint8 [N,3] table of COLORMAPS[name]: entry i is trunc(float32(255 * float32(lut[i]))), what
    (255 * tensor2array(...)).astype(np.uint8) makes of colour i of matplotlib's fp64 table."""
    data, N = COLORMAPS[name]
    lut = np.stack([_segment_table(N, d) for d in data], 1).astype(np.float32)
    return (np.float32(255) * lut).astype(np.uint8)


_TABLES = {}


def _device_table(name, device):
    """colormap_table(name) on `device`, copied there once: later calls (and CUDA-graph captures) reuse it."""
    key = (name, str(device))
    if key not in _TABLES:
        _TABLES[key] = torch.from_numpy(colormap_table(name)).to(device)
    return _TABLES[key]


@torch.no_grad()
def colorize(maps, colormap, max_value=None, invert=False):
    """(255 * tensor2array(x, max_value, colormap)).astype(np.uint8) of each map, HWC, on the device (ccb_colorize):
    maps [B,H,W] (or [B,1,H,W]) -> uint8 [B,H,W,3].  invert takes 1/x first in fp32 (depth from disparity); max_value None
    scales each image by its own maximum.  colormap is a name of COLORMAPS.  No host synchronisation once
    the colormap's table is on the device."""
    if colormap not in COLORMAPS:
        raise ValueError('colorize: colormap must be one of %s, got %r' % (sorted(COLORMAPS), colormap))
    maps = _lib.f32(maps)
    if maps.dim() == 4 and maps.size(1) == 1:
        maps = maps[:, 0]
    assert maps.dim() == 3, maps.shape
    B, H, W = (int(v) for v in maps.shape)
    lut = _device_table(colormap, maps.device)
    per_image = max_value is None
    work, nbytes = _lib.workspace('ccb_colorize_workspace_bytes', B, H, W, int(per_image), like=maps)
    out = torch.empty(B, H, W, 3, device=maps.device, dtype=torch.uint8)
    _lib.call('ccb_colorize', maps, B, H, W, lut, lut.shape[0], int(bool(invert)), int(per_image),
              0.0 if per_image else float(max_value), work, nbytes, out, maps)
    return out


@torch.no_grad()
def flow_submission_sample(disp_net, pose_net, mask_net, flow_net, tgt, refs, K, Kinv, Hg, Wg, THRESH=0.01, want_viz=False):
    """submit_flow.py:109-175 for one batch: tgt/refs normalised device tensors [B,3,h,w] (4 refs), (Hg, Wg) the original
    frame size -> flow_submission's dict of device tensors; want_viz adds 'full' and 'viz' = uint8 [B,3,3*Hg,Wg], row 2
    of the script's visualisation (cam, fwd and total flow stacked, one radius).  Row 1 (matplotlib's magma map of the
    target, disparity and mask) is not produced.  No host synchronisation."""
    emask, flow_cam, flow_fwd = _flow_nets(disp_net, pose_net, mask_net, flow_net, tgt, refs, K, Kinv)
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
    dev = pred_png.device if torch.is_tensor(pred_png) else _lib.device()
    gt, pred = (torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a).to(dev).contiguous() for a in (gt_png, pred_png))
    if gt.dim() == 3:
        gt, pred = gt[None], pred[None]
    assert gt.shape == pred.shape and gt.shape[-1] == 3 and gt.dtype == torch.uint16, (gt.shape, pred.shape, gt.dtype)
    B, H, W = (int(v) for v in gt.shape[:3])
    work, nbytes = _lib.workspace('ccb_kitti_flow_errors_workspace_bytes', B, H, W, like=gt)
    out = torch.empty(B, 2, device=dev, dtype=torch.float64)
    counts = torch.empty(B, 2, device=dev, dtype=torch.int64)
    _lib.call('ccb_kitti_flow_errors', gt, pred, B, H, W, work, nbytes, out, counts, gt)
    return out, counts


# ------------------------------------------------------------------------------------------------
# test_disp.py on the device: the velodyne ground truth, the spline zoom and the errors of each sample


def read_calib_file(path):
    """kitti_eval/depth_evaluation_utils.py read_calib_file (:104-121): {key: fp64 array, or the string when a value is
    not a list of numbers}."""
    float_chars = set('0123456789.e+- ')
    data = {}
    with open(path, 'r') as f:
        for line in f.readlines():
            key, value = line.split(':', 1)
            value = value.strip()
            data[key] = value
            if float_chars.issuperset(value):
                try:
                    data[key] = np.array(list(map(float, value.split(' '))))
                except ValueError:
                    pass
    return data


def kitti_velo_to_image(calib_dir, cam=2):
    """P_velo2im [3,4] fp64 of generate_depth_map (:150-160): P_rect_0<cam> @ R_cam2rect @ velo2cam, in the reference's
    np.dot order, from calib_cam_to_cam.txt and calib_velo_to_cam.txt under `calib_dir`."""
    import os
    cam2cam = read_calib_file(os.path.join(calib_dir, 'calib_cam_to_cam.txt'))
    velo2cam = read_calib_file(os.path.join(calib_dir, 'calib_velo_to_cam.txt'))
    velo2cam = np.hstack((velo2cam['R'].reshape(3, 3), velo2cam['T'][..., np.newaxis]))
    velo2cam = np.vstack((velo2cam, np.array([0, 0, 0, 1.0])))
    R_cam2rect = np.eye(4)
    R_cam2rect[:3, :3] = cam2cam['R_rect_00'].reshape(3, 3)
    P_rect = cam2cam['P_rect_0' + str(cam)].reshape(3, 4)
    return np.dot(np.dot(P_rect, R_cam2rect), velo2cam)


def load_velodyne_points(file_name):
    """A KITTI velodyne .bin as float32 [N,4] (forward, left, up, reflectance), the 4th column set to 1 (:97-101)."""
    points = np.fromfile(file_name, dtype=np.float32).reshape(-1, 4)
    points[:, 3] = 1
    return points


@torch.no_grad()
def velodyne_depth(points, offsets, P_velo2im, H, W):
    """generate_depth_map (:148-191) of B sweeps of one frame size on the device (ccb_velo_depth): points float32 [total,4]
    (the sweeps one after the other), offsets int64 [B+1], P_velo2im fp64 [B,3,4] -> depth fp64 [B,H,W].  KITTI frames
    come in a few sizes: group them by size, one call per size.  No host synchronisation."""
    points, offsets, P = points.detach().contiguous(), offsets.detach().contiguous(), P_velo2im.detach().contiguous()
    B = int(offsets.shape[0]) - 1
    assert points.dim() == 2 and points.shape[1] == 4 and P.shape == (B, 3, 4), (points.shape, offsets.shape, P.shape)
    work, nbytes = _lib.workspace('ccb_velo_depth_workspace_bytes', B, int(H), int(W), like=P)
    depth = torch.empty(B, int(H), int(W), device=P.device, dtype=torch.float64)
    _lib.call('ccb_velo_depth', points, offsets, P, int(points.shape[0]), B, int(H), int(W), work, nbytes, depth, P)
    return depth


@torch.no_grad()
def spline_zoom(x, H, W, lo, hi):
    """scipy.ndimage.zoom(x[n], (H/h, W/w), order=3).clip(lo, hi) of every image of x [N,h,w] on the device
    (ccb_spline_zoom) -> fp32 [N,H,W].  No host synchronisation."""
    x = _lib.f32(x)
    N, h, w = (int(v) for v in x.shape)
    work, nbytes = _lib.workspace('ccb_spline_zoom_workspace_bytes', N, h, w, like=x)
    out = torch.empty(N, int(H), int(W), device=x.device)
    _lib.call('ccb_spline_zoom', x, N, h, w, int(H), int(W), float(lo), float(hi), work, nbytes, out, x)
    return out


# generate_mask crops as fractions of (H, H, W, W): kitti_eval (Garg ECCV16, :194-206) and stillbox_eval (:68-80)
CROPS = {'eigen': (0.40810811, 0.99189189, 0.03594771, 0.96405229), 'stillbox': (0.05, 0.95, 0.05, 0.95)}


@torch.no_grad()
def depth_errors(gt, pred, min_depth=1e-3, max_depth=80.0, crop='eigen', poses=None, displacements=None):
    """The errors of test_disp.py:124-141 (compute_errors :171-187) per sample on the device (ccb_eigen_depth_errors):
    gt fp64 [B,H,W], pred the zoomed and clipped prediction fp32 [B,H,W], crop a name of CROPS or four fractions, poses
    [B,R,6] and displacements [B,R] (optional) -> fp64 [B,2,7] (abs_rel sq_rel rms log_rms a1 a2 a3); row 0 scaled by
    PoseNet (zeros without poses), row 1 by the median ratio.  No host synchronisation."""
    gt = gt.detach().to(torch.float64).contiguous()
    pred = _lib.f32(pred)
    B, H, W = (int(v) for v in gt.shape)
    assert pred.shape == (B, H, W), (gt.shape, pred.shape)
    fr = [float(f) for f in (CROPS[crop] if isinstance(crop, str) else crop)]
    R = 0
    if poses is not None:
        poses = _lib.f32(poses)
        R = int(poses.shape[1])
        displacements = torch.as_tensor(displacements, dtype=torch.float64).to(gt.device).contiguous()
        assert poses.shape == (B, R, 6) and displacements.shape == (B, R), (poses.shape, displacements.shape)
    work, nbytes = _lib.workspace('ccb_eigen_depth_errors_workspace_bytes', B, H, W, like=gt)
    out = torch.empty(B, 2, 7, device=gt.device, dtype=torch.float64)
    _lib.call('ccb_eigen_depth_errors', gt, pred, B, H, W, float(min_depth), float(max_depth), fr, poses, displacements, R, work,
              nbytes, out, gt)
    return out


@torch.no_grad()
def depth_eval_batch(disp_net, tgt, gt_depth, min_depth=1e-3, max_depth=80.0, crop='eigen', pose_net=None, refs=None,
                     displacements=None, spatial_normalize=False, want_disp=False):
    """test_disp.py:100-141 for a batch: tgt [B,3,h,w] and refs (list of [B,3,h,w]) normalised device tensors (DeviceScale
    makes them from uint8 frames), gt_depth fp64 [B,H,W] (velodyne_depth), displacements [B,R] -> fp64 [B,2,7] on the
    device, row 0 scaled by the pose net's displacements (zeros without a pose net), row 1 by the median ratio.  The pose
    net may return PoseExpNet's (mask, pose).  want_disp also returns the disparity the errors come from, [B,1,h,w]
    (after spatial_normalize).  No host synchronisation."""
    disp_net.eval()
    disp = disp_net(tgt)
    if spatial_normalize:
        disp = LF.spatial_normalize(disp)
    H, W = int(gt_depth.shape[1]), int(gt_depth.shape[2])
    pred = spline_zoom(1 / disp[:, 0], H, W, min_depth, max_depth)
    poses = None
    if pose_net is not None:
        pose_net.eval()
        poses = _pose(pose_net(tgt, refs))
    errors = depth_errors(gt_depth, pred, min_depth, max_depth, crop, poses, displacements if poses is not None else None)
    return (errors, disp) if want_disp else errors


def depth_summary(per_sample):
    """The rows test_disp.py prints (:143-158) from the [N,2,7] per-sample errors of a dataset: stored as float32 like the
    script's `errors`, then averaged over the samples -> float32 [2,7]."""
    per_sample = np.asarray(per_sample)
    errors = np.zeros((2, 7, per_sample.shape[0]), np.float32)
    errors[:] = per_sample.transpose(1, 2, 0)
    return errors.mean(2)


def _depth_shifts(seq_length, step=1):
    """The reference frames' offsets of read_scene_data: -demi..-1, 1..demi (times step), demi = (seq_length - 1) // 2."""
    demi = (seq_length - 1) // 2
    return [step * i for i in list(range(-demi, 0)) + list(range(1, demi + 1))]


def kitti_displacements(oxts_root, index, shifts, timestamps=None):
    """kitti_eval's get_displacements: speed |oxts[8:11]| of frame `index` times |t_index - t_index+shift| per shift, the
    times parsed as the reference parses them (strptime(ts[:-3]).timestamp(); only their differences are used, so the
    time zone drops out).  timestamps: a dict that caches each drive's timestamps.txt across calls."""
    import datetime
    import os
    cache = {} if timestamps is None else timestamps
    if oxts_root not in cache:
        with open(os.path.join(oxts_root, 'timestamps.txt')) as f:
            cache[oxts_root] = [datetime.datetime.strptime(ts[:-3], '%Y-%m-%d %H:%M:%S.%f').timestamp()
                                for ts in f.read().splitlines()]
    t = cache[oxts_root]
    speed = np.linalg.norm(np.genfromtxt(os.path.join(oxts_root, 'data', '{:010d}.txt'.format(index)))[8:11])
    if not all(0 <= index + s < len(t) for s in shifts):
        raise ValueError('%s: frames %s are outside the drive\'s %d timestamps' % (oxts_root, [index + s for s in shifts],
                                                                                  len(t)))
    return [speed * abs(t[index] - t[index + s]) for s in shifts]


def kitti_depth_framework(root, test_files, seq_length=3, step=1):
    """kitti_eval/depth_evaluation_utils.py test_framework_KITTI's read_scene_data -> one dict per test file that exists,
    in list order: 'path' (root joined to the line), 'refs' (the frames at the shifts of _depth_shifts in the same folder,
    always .png; a missing one is the target itself with shift 0, so its displacement is 0), 'velo' (the drive's
    velodyne_points/data/<index>.bin), 'calib_dir' (root/<date>), 'cam' (the camera folder's last two digits) and
    'displacements' (kitti_displacements).  Prints 'getting test metadata ... ' and '<path> missing' as the reference."""
    import os
    shifts = _depth_shifts(seq_length, step)
    samples, timestamps = [], {}
    print('getting test metadata ... ')
    for sample in test_files:
        tgt = os.path.join(root, sample)
        parts = sample[:-4].split('/')
        if len(parts) != 5:
            raise ValueError('%s: a KITTI test file is <date>/<drive>/<camera>/data/<index>.<ext>' % sample)
        date, scene, cam_id, _, index = parts
        refs = [os.path.join(os.path.dirname(tgt), '{:010d}.png'.format(int(index) + s)) for s in shifts]
        capped = list(shifts)
        for i, r in enumerate(refs):
            if not os.path.isfile(r):
                refs[i], capped[i] = tgt, 0
        if not os.path.isfile(tgt):
            print('{} missing'.format(tgt))
            continue
        samples.append(dict(path=tgt, refs=refs, cam=int(cam_id[-2:]), calib_dir=os.path.join(root, date),
                            velo=os.path.join(root, date, scene, 'velodyne_points', 'data', '{}.bin'.format(index[:10])),
                            displacements=kitti_displacements(os.path.join(root, date, scene, 'oxts'), int(index), capped,
                                                              timestamps)))
    return samples


def stillbox_depth_framework(root, test_files, seq_length=3, step=1):
    """stillbox_eval/depth_evaluation_utils.py test_framework_stillbox's read_scene_data, as kitti_depth_framework: the
    metadata.json of every directory under root; a line is <folder>/RGB_<scene>_<index>.<ext>; the reference indices are
    clamped into the scene (at its edges a reference is the target itself, displacement 0); 'depth' is the scene's .npy of
    the target and 'displacements' round(|speed|, 3) * time_step * |index - ref index|."""
    import json
    import os
    meta = {}
    for d in os.listdir(root):
        if os.path.isdir(os.path.join(root, d)):
            with open(os.path.join(root, d, 'metadata.json')) as f:
                meta[d] = json.load(f)
    shifts = _depth_shifts(seq_length, step)
    samples = []
    print('getting test metadata ... ')
    for sample in test_files:
        parts = sample.split('/')
        names = parts[-1][:-4].split('_')
        if len(parts) != 2 or len(names) != 3:
            raise ValueError('%s: a Stillbox test file is <folder>/RGB_<scene>_<index>.<ext>' % sample)
        folder, index = parts[0], int(names[2])
        scene = meta[folder]['scenes'][int(names[1])]
        tgt = os.path.join(root, sample)
        if not os.path.isfile(tgt):
            print('{} missing'.format(tgt))
            continue
        capped = [min(max(0, index + s), scene['length'] - 1) for s in shifts]
        speed = np.around(np.linalg.norm(scene['speed']), decimals=3)
        samples.append(dict(path=tgt, refs=[os.path.join(root, folder, '{}'.format(scene['imgs'][i])) for i in capped],
                            depth=os.path.join(root, folder, '{}'.format(scene['depth'][index])),
                            displacements=[speed * scene['time_step'] * abs(index - i) for i in capped]))
    return samples


# ------------------------------------------------------------------------------------------------
# test_make3d.py on the device: imresize's contrast stretch and resize, the zoom and the capped, log10 errors

MAKE3D_ROWS = ((2272 - 852) // 2, (2272 + 852) // 2)       # test_make3d.py:50,62: the image rows kept, whatever its height
MAKE3D_GT_ROWS = ((55 - 21) // 2, (55 + 21) // 2)           # :51,66: the ground-truth rows kept


def make3d_files(root):
    """test_framework's file lists (test_make3d.py:41-46): the sorted Test134/*.jpg and Gridlaserdata/*.mat under `root`,
    element 61 popped from each (a corrupted file of the original dataset).  The lists are paired by index, not by name."""
    import glob
    import os
    img_files = sorted(glob.glob(os.path.join(root, 'Test134', '*.jpg')))
    depth_files = sorted(glob.glob(os.path.join(root, 'Gridlaserdata', '*.mat')))
    img_files.pop(61)
    depth_files.pop(61)
    return img_files, depth_files


def load_make3d(img_file, depth_file, min_depth=1e-3, max_depth=70.0):
    """One sample of test_framework (test_make3d.py:53-71): {'tgt': uint8 [852,W,3] image rows 710:1562 (the reference's
    float32 copy holds the same integers), 'gt_depth': fp64 [21,C] rows 17:38 of Position3DGrid[:, :, 3],
    'mask': min_depth < gt_depth < max_depth}."""
    from PIL import Image
    from scipy import io
    tgt = np.array(Image.open(img_file))[MAKE3D_ROWS[0]:MAKE3D_ROWS[1]]
    gt = io.loadmat(depth_file)['Position3DGrid'][:, :, 3][MAKE3D_GT_ROWS[0]:MAKE3D_GT_ROWS[1]]
    return {'tgt': tgt, 'gt_depth': gt, 'mask': np.logical_and(gt > min_depth, gt < max_depth)}


@torch.no_grad()
def make3d_frames(crops_u8, h=256, w=256, resize=True):
    """The net input of test_make3d.py:98-106 for a batch: crops_u8 uint8 [B,Hs,Ws,3] (load_make3d's 'tgt'; numpy arrays
    go to the library's device) -> normalised fp32 [B,3,h,w] (or [B,3,Hs,Ws] without resizing).  Unless resize is False
    or the crops already are h x w, each crop is contrast-stretched and resized as scipy.misc.imresize does to a float32
    image (input_pipeline.scale_frames); then (x/255 - 0.5)/0.5.  No host synchronisation."""
    src = device_tensor(crops_u8)[:, None]
    if not resize:
        h, w = src.shape[2:4]
    return scale_frames(src, h, w)[0][0]


@torch.no_grad()
def make3d_depth_errors(gt, pred, min_depth=1e-3, max_depth=70.0):
    """The errors of test_make3d.py:141-148 (compute_errors :174-190) per sample on the device (ccb_make3d_depth_errors):
    gt fp64 [B,H,W], pred the zoomed and clipped prediction fp32 [B,H,W] -> fp64 [B,2,7] (abs_rel sq_rel rms log_rms a1 a2
    a3).  Row 0 is zeros, as the script leaves it; row 1 scales by the median ratio over min_depth < gt < max_depth (no
    crop), caps the scaled prediction at max_depth and takes log_rms in log10.  An empty mask gives a NaN row.  No host
    synchronisation."""
    gt = gt.detach().to(torch.float64).contiguous()
    pred = _lib.f32(pred)
    B, H, W = (int(v) for v in gt.shape)
    assert pred.shape == (B, H, W), (gt.shape, pred.shape)
    work, nbytes = _lib.workspace('ccb_make3d_depth_errors_workspace_bytes', B, H, W, like=gt)
    out = torch.empty(B, 2, 7, device=gt.device, dtype=torch.float64)
    _lib.call('ccb_make3d_depth_errors', gt, pred, B, H, W, float(min_depth), float(max_depth), work, nbytes, out, gt)
    return out


@torch.no_grad()
def make3d_eval_batch(disp_net, crops_u8, gt_depth, h=256, w=256, min_depth=1e-3, max_depth=70.0, resize=True):
    """test_make3d.py:97-148 for a batch: crops_u8 uint8 [B,852,W,3] and gt_depth fp64 [B,21,C] (load_make3d's 'tgt' and
    'gt_depth', stacked; numpy arrays go to the library's device), disp_net any disparity net of cc_b200.models ->
    fp64 [B,2,7] on the device, row 1 the script's errors and row 0 zeros (depth_summary gives the printed row).
    No host synchronisation."""
    disp_net.eval()
    disp = disp_net(make3d_frames(crops_u8, h, w, resize))
    gt = device_tensor(gt_depth)
    H, W = int(gt.shape[1]), int(gt.shape[2])
    pred = spline_zoom(1 / disp[:, 0], H, W, min_depth, max_depth)
    return make3d_depth_errors(gt, pred, min_depth, max_depth)


# ------------------------------------------------------------------------------------------------
# test_pose.py / test_sintel_pose.py on the device: every frame stretched and resized once, the snippets gathered on the
# device, the pose net on all of them in one call, the pose algebra and the errors in one kernel

POSE_NETS = ('PoseNetB6', 'PoseNet6', 'PoseExpNet')


def load_pose_net(weights, name='PoseNetB6', device=None):
    """The pose net of test_pose.py:35-38 -> (net, seq_length): weights a checkpoint path or the loaded dict holding
    'state_dict'; seq_length = conv1.0.weight.size(1) / 3, the net built for seq_length - 1 references and loaded with
    strict=False.  name is one of POSE_NETS (PoseNet6 and PoseExpNet from models/alternates.py)."""
    assert name in POSE_NETS, name
    if not isinstance(weights, dict):
        weights = torch.load(weights, map_location='cpu')
    seq_length = int(weights['state_dict']['conv1.0.weight'].size(1) / 3)
    net = getattr(models, name)(nb_ref_imgs=seq_length - 1)
    net.load_state_dict(weights['state_dict'], strict=False)
    return net.to(device or torch.device('cuda')), seq_length


def _snippet_indices(n, seq_length):
    """read_scene_data's snippets of a sequence of n frames: the target frames demi..n-1-demi, each with its demi
    neighbours either side (step 1) -> int64 [S, seq_length]."""
    demi = (seq_length - 1) // 2
    return np.arange(-demi, demi + 1).reshape(1, -1) + np.arange(demi, n - demi).reshape(-1, 1)


def _compensate(poses):
    """The framework's ground truth of the snippets' poses [S,L,3,4], in their dtype: every row loses the original first
    translation (the reference subtracts through a view of row 0; numpy buffers the overlap, so row 0 ends at zero), then
    is rotated by inv(R_0) (rotation unaffected)."""
    poses = poses.copy()
    poses[:, :, :, -1] -= poses[:, :1, :, -1].copy()
    return np.linalg.inv(poses[:, 0, :, :3])[:, None] @ poses


def _matching(parent, patterns, isdir):
    """path.Path(parent).dirs(p) (isdir) or .files(p) for each pattern p, united and sorted: fnmatch on the entry names
    (the reference iterates its sequences as a set, in hash order; here always in sorted order)."""
    import fnmatch
    import os
    keep = os.path.isdir if isdir else os.path.isfile
    names = [d for d in os.listdir(parent) if keep(os.path.join(parent, d))]
    return sorted({os.path.join(parent, d) for p in patterns for d in names if fnmatch.fnmatch(d, p)})


def kitti_pose_framework(root, sequences, seq_length):
    """kitti_eval/pose_evaluation_utils.py test_framework_KITTI (step 1) -> (seqs, n_rows).  seqs: one dict per directory
    under root/sequences matching a pattern of `sequences`, in sorted order: 'name', 'files' (sorted image_2/*.png),
    'snippets' int64 [S,L] and 'gt' fp64 [S,L,3,4], the compensated poses of poses/<name>.txt.  n_rows = len(framework):
    the image count, which the scripts size their arrays with (seq_length - 1 zero rows per sequence)."""
    import os
    seqs = []
    for d in _matching(os.path.join(root, 'sequences'), sequences, True):
        name = os.path.basename(d)
        poses = np.genfromtxt(os.path.join(root, 'poses', '{}.txt'.format(name))).astype(np.float64).reshape(-1, 3, 4)
        files = _matching(os.path.join(d, 'image_2'), ['*.png'], False)
        snippets = _snippet_indices(len(files), seq_length)
        seqs.append(dict(name=name, files=files, snippets=snippets, gt=_compensate(poses[snippets])))
    return seqs, sum(len(s['files']) for s in seqs)


def sintel_cam_read(path):
    """sintel_io.cam_read(path, pose_only=True): the 202021.25 tag, then 9 + 12 fp64 values -> N, fp64 [3,4]."""
    with open(path, 'rb') as f:
        tag = np.fromfile(f, np.float32, 1)
        assert tag.size == 1 and tag[0] == 202021.25, 'sintel_cam_read: %s: wrong tag %s' % (path, tag)
        np.fromfile(f, np.float64, 9)
        return np.fromfile(f, np.float64, 12).reshape(3, 4)


def sintel_pose_framework(root, sequences, seq_length):
    """sintel_eval/pose_evaluation_utils.py test_framework_Sintel (step 1) -> (seqs, n_rows), as kitti_pose_framework:
    the directories under root/clean, their sorted *.png, and the .cam files of the same path with /clean/ replaced by
    /camdata_left/.  The ground truth is float32 as the reference computes it (cam_read(...).astype(np.float32))."""
    import os
    seqs = []
    for d in _matching(os.path.join(root, 'clean'), sequences, True):
        cams = _matching(d.replace('/clean/', '/camdata_left/'), ['*.cam'], False)
        files = _matching(d, ['*.png'], False)
        snippets = _snippet_indices(len(files), seq_length)
        poses = np.array([sintel_cam_read(c).astype(np.float32) for c in cams], np.float32).reshape(-1, 3, 4)
        seqs.append(dict(name=os.path.basename(d), files=files, snippets=snippets, gt=_compensate(poses[snippets])))
    return seqs, sum(len(s['files']) for s in seqs)


def load_pose_frames(files):
    """The frames of one sequence (or a chunk of one) decoded by Pillow on the host -> uint8 [N,H,W,3] (the reference's
    imread(...).astype(np.float32) holds the same integers)."""
    from PIL import Image
    frames = np.stack([np.asarray(Image.open(f)) for f in files])
    assert frames.dtype == np.uint8 and frames.ndim == 4 and frames.shape[3] == 3, (frames.dtype, frames.shape)
    return frames


@torch.no_grad()
def pose_errors(poses, gt=None, rotation_mode='euler'):
    """test_pose.py:74-92 per snippet on the device (ccb_pose_errors): poses [S,L-1,6] the pose net's output, gt the
    framework's compensated ground truth [S,L,3,4] (numpy arrays go to the library's device, fp64; Sintel's float32
    exactly upcast) -> (out fp64 [S,2] = ATE, RE or None without gt, final fp64 [S,L,3,4]).  Sintel's script keeps RE
    alone.  No host synchronisation."""
    poses = _lib.f32(poses)
    S, R, six = (int(v) for v in poses.shape)
    assert six == 6, poses.shape
    L = R + 1
    final = torch.empty(S, L, 3, 4, device=poses.device, dtype=torch.float64)
    out = None
    if gt is not None:
        gt = device_tensor(gt).to(poses.device, torch.float64).contiguous()
        assert gt.shape == (S, L, 3, 4), (gt.shape, poses.shape)
        out = torch.empty(S, 2, device=poses.device, dtype=torch.float64)
    rot = {'euler': _lib.ROT_EULER, 'quat': _lib.ROT_QUAT}[rotation_mode]
    _lib.call('ccb_pose_errors', poses, S, L, rot, gt, final, out, poses)
    return out, final


@torch.no_grad()
def pose_eval_batch(pose_net, frames_u8, snippets, gt_poses=None, rotation_mode='euler', h=256, w=832, resize=True):
    """test_pose.py:50-92 (test_sintel_pose.py:55-97 with h, w = 128, 416) for a batch of snippets: frames_u8 uint8
    [N,H,W,3] the frames of one sequence or a chunk of one, snippets int64 [S,L] indices into them, gt_poses the
    framework's [S,L,3,4] (numpy arrays go to the library's device) -> pose_errors' (out, final).  Each frame is
    stretched, resized and normalised once (make3d_frames: imresize unless resize is False or the frames already are
    h x w); the snippets are gathered on the device (target = column L/2, refs = the others in order) and the pose net runs
    on all of them in one call.  No host synchronisation."""
    x = make3d_frames(frames_u8, h, w, resize)
    idx = device_tensor(snippets).to(x.device, torch.int64)
    L = int(idx.shape[1])
    mid = L // 2
    pose_net.eval()
    tgt = x[idx[:, mid]]
    refs = [x[idx[:, j]] for j in range(L) if j != mid]
    return pose_errors(_pose(pose_net(tgt, refs)), gt_poses, rotation_mode)


def pose_summary(per_snippet, n_rows, sintel=False):
    """The rows the scripts print (test_pose.py:44,92-101; test_sintel_pose.py:49,96-102) from the [S,2] per-snippet
    (ATE, RE) of a whole framework in its order: stored as float32 in an array of n_rows = len(framework) rows, the
    rest zero, then its mean and std -> float32 [2,2] (rows mean, std; columns ATE, RE), or [2,1] (RE) for Sintel."""
    per_snippet = np.asarray(per_snippet).reshape(-1, 2)
    errors = np.zeros((n_rows, 1 if sintel else 2), np.float32)
    errors[:len(per_snippet)] = per_snippet[:, 1:] if sintel else per_snippet
    return np.stack([errors.mean(0), errors.std(0)])


def write_pose_predictions(path, finals, n_rows):
    """predictions.npy of --output-dir (test_pose.py:48,89,104) under the directory `path`: the [S,L,3,4] final poses of
    the framework in its order, in an fp64 array of n_rows = len(framework) snippets, the rest zero."""
    import os
    finals = np.asarray(finals)
    os.makedirs(path, exist_ok=True)
    predictions = np.zeros((n_rows,) + finals.shape[1:])
    predictions[:len(finals)] = finals
    np.save(os.path.join(path, 'predictions.npy'), predictions)


# ------------------------------------------------------------------------------------------------
# test_flow.py / test_back2future.py on the device: ValidationFlow's samples batched within a frame size, the nets at
# batch B, the rigidity masks and both compute_all_epes of every sample in one kernel

FLOW_ERROR_NAMES = ('epe_total', 'epe_sp', 'epe_mv', 'Fl', 'epe_total_gt_mask', 'epe_sp_gt_mask', 'epe_mv_gt_mask',
                    'Fl_gt_mask')
FLOW_EVAL_NETS = {'disp': ('DispResNet6', 'DispNetS6'), 'pose': ('PoseNetB6', 'PoseNet6'),
                  'mask': ('MaskNet6', 'MaskResNet6'), 'flow': ('Back2Future', 'FlowNetC6')}


def kitti_flow_framework(root, phase='training', occ='flow_occ', N=200, sequence_length=5):
    """ValidationFlow's files (datasets/validation_flow.py:94-141) -> dict(samples, groups).  samples: N dicts, index i:
    'frames' (image_2/iiiiii_10.png, then the references _08 _09 _11 _12 for sequence_length 5), 'flow'
    (data_scene_flow/<phase>/<occ>/iiiiii_10.png; occ 'flow_occ' or 'flow_noc'), 'obj' (obj_map/iiiiii_10.png, or None
    where it is missing: the reference then uses ones), 'calib' (calib_cam_to_cam/iiiiii.txt) and 'size' (H, W) of the
    target frame, read from its PNG header.  groups: {(H, W): [indices in order]}; KITTI-2015 frames come in several sizes
    and a batch takes one."""
    import os
    from PIL import Image
    half = int(sequence_length / 2)
    seq_ids = [k + 10 for k in range(-half, half + 1) if k != 0]
    samples, groups = [], {}
    for i in range(N):
        name = str(i).zfill(6)
        img = os.path.join(root, 'data_scene_flow_multiview', phase, 'image_2', name + '_%s.png')
        obj = os.path.join(root, 'data_scene_flow', phase, 'obj_map', name + '_10.png')
        with Image.open(img % '10') as im:
            size = (im.size[1], im.size[0])
        samples.append(dict(frames=[img % '10'] + [img % str(k).zfill(2) for k in seq_ids],
                            flow=os.path.join(root, 'data_scene_flow', phase, occ, name + '_10.png'),
                            obj=obj if os.path.isfile(obj) else None,
                            calib=os.path.join(root, 'data_scene_flow_calib', phase, 'calib_cam_to_cam', name + '.txt'),
                            size=size))
        groups.setdefault(size, []).append(i)
    return dict(samples=samples, groups=groups)


def kitti_cam_intrinsics(path, cid='02'):
    """get_intrinsics (validation_flow.py:33-37) as ValidationFlow uses it: P_rect_<cid>[:, :3] of a calib_cam_to_cam file,
    parsed as read_raw_calib_file parses it (the last line of a key wins), in float32."""
    data = {}
    with open(path, 'r') as f:
        for line in f.readlines():
            key, value = line.split(':', 1)
            try:
                data[key] = np.array([float(x) for x in value.split()])
            except ValueError:
                pass
    return np.reshape(data['P_rect_' + cid], (3, 4))[:, :3].astype('float32')


def load_kitti_flow_samples(framework, indices):
    """Samples `indices` of kitti_flow_framework, all of one frame size, decoded on the host -> dict of numpy arrays:
    frames uint8 [B,F,Hs,Ws,3] (target first; the reference's imread(...).astype(np.float32) holds the same integers),
    gt fp32 [B,3,Hg,Wg] (flow_read_png's u, v, valid), obj fp32 [B,Hg,Wg] (ones where the file is missing; the
    reference's ones are float64, the same values), obj_found bool [B], K fp32 [B,3,3] (P_rect_02[:, :3])."""
    from PIL import Image
    from .flowutils import flow_io
    ss = [framework['samples'][i] for i in indices]
    assert len({s['size'] for s in ss}) == 1, 'a batch takes one frame size: %s' % sorted({s['size'] for s in ss})
    frames = np.stack([np.stack([np.asarray(Image.open(f)) for f in s['frames']]) for s in ss])
    assert frames.dtype == np.uint8 and frames.ndim == 5 and frames.shape[4] == 3, (frames.dtype, frames.shape)
    gt = np.stack([np.stack(flow_io.flow_read_png(s['flow'])) for s in ss]).astype(np.float32)
    obj = np.stack([np.asarray(Image.open(s['obj'])).astype(np.float32) if s['obj'] else np.ones(frames.shape[2:4], np.float32)
                    for s in ss])
    K = np.stack([kitti_cam_intrinsics(s['calib']) for s in ss])
    return dict(frames=frames, gt=gt, obj=obj, obj_found=np.array([s['obj'] is not None for s in ss]), K=K)


@torch.no_grad()
def flow_eval(emask, flow_cam, flow_fwd, flow_gt, obj_map_gt, THRESH=0.01, epe_thresh=0.5, tau=(3, 0.05), want_mask=False):
    """The numbers of test_flow.py:127-140 per sample in one fused call (ccb_flow_eval): emask [B,C,h,w] the mask net's eval
    output, flow_cam / flow_fwd [B,2,h,w], flow_gt [B,3,Hg,Wg], obj_map_gt [B,Hg,Wg] -> fp32 [B,8] on the device =
    compute_all_epes(gt, cam, fwd, combined) + compute_all_epes(gt, cam, fwd, 1 - obj), each {all, rigid, non-rigid EPE,
    Fl}, at batch-1 semantics.  THRESH is the script's --THRESH (the census and the composite); epe_thresh is
    compute_all_epes' own THRESH, which the script leaves at 0.5.  want_mask: also the combined mask [B,1,h,w] (0/1).
    emask and flow_cam None: test_back2future.py's compute_all_epes(gt, fwd, fwd, 1 - obj) alone -> [B,4].
    No host synchronisation."""
    flow_fwd, flow_gt, obj = _lib.f32(flow_fwd), _lib.f32(flow_gt), _lib.f32(obj_map_gt)
    B, two, h, w = (int(v) for v in flow_fwd.shape)
    Hg, Wg = int(flow_gt.shape[2]), int(flow_gt.shape[3])
    assert two == 2 and flow_gt.shape == (B, 3, Hg, Wg) and obj.shape == (B, Hg, Wg), (flow_fwd.shape, flow_gt.shape, obj.shape)
    C = 0
    if emask is not None:
        emask, flow_cam = _lib.f32(emask), _lib.f32(flow_cam)
        C = int(emask.shape[1])
        assert emask.shape == (B, C, h, w) and flow_cam.shape == (B, 2, h, w), (emask.shape, flow_cam.shape)
    else:
        assert flow_cam is None and not want_mask
    work, nbytes = _lib.workspace('ccb_flow_eval_workspace_bytes', B, h, w, Hg, Wg, like=flow_fwd)
    out = torch.empty(B, 8, device=flow_fwd.device)
    mask = torch.empty(B, 1, h, w, device=flow_fwd.device) if want_mask else None
    _lib.call('ccb_flow_eval', emask, flow_cam, flow_fwd, flow_gt, obj, B, C, h, w, Hg, Wg, float(THRESH), float(epe_thresh),
              float(tau[0]), float(tau[1]), mask, work, nbytes, out, flow_fwd)
    if emask is None:
        return out[:, 4:]
    return (out, mask) if want_mask else out


@torch.no_grad()
def flow_eval_batch(disp_net, pose_net, mask_net, flow_net, frames_u8, K, flow_gt, obj_map, THRESH=0.01, h=256, w=832,
                    spatial_normalize=False, want_mask=False, normalization='global'):
    """test_flow.py:112-140 for a batch of one frame size: frames_u8 uint8 [B,5,Hs,Ws,3] (target, then _08 _09 _11 _12),
    K the raw intrinsics [B,3,3] (or the (K, Kinv) pair flow_intrinsics returns), flow_gt [B,3,Hg,Wg],
    obj_map [B,Hg,Wg] (load_kitti_flow_samples' arrays; numpy arrays go to the library's device) -> flow_eval's fp32 [B,8]
    on the device (and the combined mask with want_mask).  The frames go through scale_frames (Scale), the four
    nets run at batch B (Back2Future on refs 1 and 2, another flow net on ref 2), flow_cam = pose2flow with pose[:, 2].
    spatial_normalize: train.py's validate_flow_with_gt with --spatial-normalize; normalization: its --data-normalization
    ('global' or 'local', as scale_frames takes it).  No host synchronisation."""
    x, _ = scale_frames(frames_u8, h, w, normalization)
    Hs, Ws = int(frames_u8.shape[2]), int(frames_u8.shape[3])
    K, Kinv = K if isinstance(K, tuple) else flow_intrinsics(K, Hs, Ws, h, w, x[0].device)
    emask, flow_cam, flow_fwd = _flow_nets(disp_net, pose_net, mask_net, flow_net, x[0], x[1:], K, Kinv, spatial_normalize)
    return flow_eval(emask, flow_cam, flow_fwd, device_tensor(flow_gt), device_tensor(obj_map), THRESH,
                     want_mask=want_mask)


@torch.no_grad()
def back2future_eval_batch(flow_net, frames_u8, flow_gt, obj_map, h=256, w=832):
    """test_back2future.py on KITTI-2015 for a batch of one frame size (frames, flow_gt and obj_map as flow_eval_batch takes
    them; the script's nlevels 5 and 6 give the same eval output from the same checkpoint) -> fp32 [B,4] on the device =
    compute_all_epes(gt, fwd, fwd, 1 - obj).  No host synchronisation."""
    x, _ = scale_frames(frames_u8, h, w)
    flow_net.eval()
    flow_fwd = flow_net(x[0], x[2:4])[0]
    return flow_eval(None, None, flow_fwd, device_tensor(flow_gt), device_tensor(obj_map))


def load_flow_eval_nets(pretrained_disp, pretrained_pose, pretrained_mask, pretrained_flow, dispnet='DispResNet6',
                        posenet='PoseNetB6', masknet='MaskNet6', flownet='Back2Future', nlevels=6, device=None):
    """The four nets of test_flow.py:88-106 -> (disp, pose, mask, flow) in eval mode: each argument a checkpoint path or
    the loaded dict holding 'state_dict', loaded strictly; the pose and mask nets built for 4 references, the flow net
    with nlevels; the choices are FLOW_EVAL_NETS'."""
    out = []
    for kind, name, weights in (('disp', dispnet, pretrained_disp), ('pose', posenet, pretrained_pose),
                                ('mask', masknet, pretrained_mask), ('flow', flownet, pretrained_flow)):
        assert name in FLOW_EVAL_NETS[kind], (kind, name)
        kw = {'nb_ref_imgs': 4} if kind in ('pose', 'mask') else {'nlevels': nlevels} if kind == 'flow' else {}
        net = getattr(models, name)(**kw)
        if not isinstance(weights, dict):
            weights = torch.load(weights, map_location='cpu')
        net.load_state_dict(weights['state_dict'])
        out.append(net.to(device or torch.device('cuda')).eval())
    return tuple(out)


def flow_summary(per_sample):
    """AverageMeter's averages of the per-sample rows in sample order -> (avg, row): each column summed as python floats
    (fp64) in index order, then divided by the count, as test_flow.py / test_back2future.py accumulate .item() values.
    row is the line the script prints: test_flow.py's 'Errors' row of 8 columns, or test_back2future.py's
    'Averge EPE [...]' of 4.  test_back2future.py labels its 2nd and 3rd columns non-rigid and rigid, but its values are
    compute_all_epes' rigid then non-rigid; avg keeps the values' order."""
    per_sample = np.asarray(per_sample).reshape(len(per_sample), -1)
    sums = [0] * per_sample.shape[1]
    for r in per_sample.tolist():
        for k, v in enumerate(r):
            sums[k] += v
    avg = [s / len(per_sample) for s in sums]
    if len(avg) == 8:
        row = 'Errors \t {:10.4f}, {:10.4f}, {:10.4f}, {:10.4f}, {:10.4f}, {:10.4f}, {:10.4f}, {:10.4f}'.format(*avg)
    else:
        row = 'Averge EPE ' + str(avg)
    return avg, row


def write_flow_eval_outputs(out_dir, i, tgt, mask, obj_map, obj_found=True):
    """Sample `i` (batch 1) written as test_flow.py:142-153 names it under `out_dir`: images/iii.npy (the normalised target
    [3,h,w] fp32), gt/iii.npy (the object map [Hg,Wg]: fp32, or the reference's fp64 ones where the file is missing) and
    mask/iii.npy (the combined mask [1,h,w] fp32)."""
    import os
    for sub in ('images', 'gt', 'mask'):
        os.makedirs(os.path.join(out_dir, sub), exist_ok=True)
    name = str(i).zfill(3)
    obj = obj_map[0].cpu().numpy() if torch.is_tensor(obj_map) else np.asarray(obj_map)[0]
    np.save(os.path.join(out_dir, 'images', name), tgt[0].detach().cpu().numpy())
    np.save(os.path.join(out_dir, 'gt', name), obj.astype(np.float32 if obj_found else np.float64))
    np.save(os.path.join(out_dir, 'mask', name), mask[0].detach().cpu().numpy())
