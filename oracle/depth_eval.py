"""test_disp.py's depth evaluation restated on numpy and scipy: the ground truth of kitti_eval/depth_evaluation_utils.py
(generate_depth_map :148-191 from the points and the projection, generate_mask :194-206 and stillbox_eval's :68-80 as crop
fractions), compute_errors (:171-187) and the sample body (:124-141).  tests/golden/depth_eval_small.npz holds what the
reference's own functions return for the same inputs."""
from collections import Counter
import numpy as np

EIGEN = (0.40810811, 0.99189189, 0.03594771, 0.96405229)
STILLBOX = (0.05, 0.95, 0.05, 0.95)


def generate_depth_map(points, P_velo2im, im_shape):
    """points float32 [N,4] as the .bin holds them (load_velodyne_points sets column 3 to 1), P_velo2im fp64 [3,4] ->
    fp64 depth [H,W]."""
    velo = np.array(points, np.float32)
    velo[:, 3] = 1
    velo = velo[velo[:, 0] >= 0, :]
    with np.errstate(divide='ignore', invalid='ignore'):
        velo_pts_im = np.dot(P_velo2im, velo.T).T
        velo_pts_im[:, :2] = velo_pts_im[:, :2] / velo_pts_im[:, -1:]
    velo_pts_im[:, 0] = np.round(velo_pts_im[:, 0]) - 1
    velo_pts_im[:, 1] = np.round(velo_pts_im[:, 1]) - 1
    with np.errstate(invalid='ignore'):
        val_inds = (velo_pts_im[:, 0] >= 0) & (velo_pts_im[:, 1] >= 0)
        val_inds = val_inds & (velo_pts_im[:, 0] < im_shape[1]) & (velo_pts_im[:, 1] < im_shape[0])
    velo_pts_im = velo_pts_im[val_inds, :]
    depth = np.zeros(im_shape)
    depth[velo_pts_im[:, 1].astype(int), velo_pts_im[:, 0].astype(int)] = velo_pts_im[:, 2]
    inds = velo_pts_im[:, 1] * (im_shape[1] - 1) + velo_pts_im[:, 0] - 1          # the reference's sub2ind
    for dd in [item for item, count in Counter(inds).items() if count > 1]:
        pts = np.where(inds == dd)[0]
        depth[int(velo_pts_im[pts[0], 1]), int(velo_pts_im[pts[0], 0])] = velo_pts_im[pts, 2].min()
    depth[depth < 0] = 0
    return depth


def generate_mask(gt_depth, min_depth, max_depth, crop=EIGEN):
    mask = np.logical_and(gt_depth > min_depth, gt_depth < max_depth)
    gt_height, gt_width = gt_depth.shape
    c = np.array([crop[0] * gt_height, crop[1] * gt_height, crop[2] * gt_width, crop[3] * gt_width]).astype(np.int32)
    crop_mask = np.zeros(mask.shape)
    crop_mask[c[0]:c[1], c[2]:c[3]] = 1
    return np.logical_and(mask, crop_mask)


def compute_errors(gt, pred):
    with np.errstate(divide='ignore', invalid='ignore'):
        thresh = np.maximum((gt / pred), (pred / gt))
        a1 = (thresh < 1.25).mean()
        a2 = (thresh < 1.25 ** 2).mean()
        a3 = (thresh < 1.25 ** 3).mean()
        rmse = np.sqrt(((gt - pred) ** 2).mean())
        rmse_log = np.sqrt(((np.log(gt) - np.log(pred)) ** 2).mean())
        abs_rel = np.mean(np.abs(gt - pred) / gt)
        sq_rel = np.mean(((gt - pred) ** 2) / gt)
    return abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3


def pose_norms(poses):
    """|pose[:3]| of fp32 poses [R,6] as the correctly rounded fp32 norm (the kernel's and, to rounding, torch's)."""
    p = np.asarray(poses, np.float64)[:, :3]
    return np.sqrt((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2]).astype(np.float32)


def sample_errors(gt_depth, pred_zoomed, min_depth=1e-3, max_depth=80.0, crop=EIGEN, poses=None, displacements=None):
    """test_disp.py:126-141 of one sample: gt_depth fp64 [H,W], pred_zoomed the zoomed, clipped fp32 prediction [H,W],
    poses fp32 [R,6] -> fp64 [2,7] (row 0 zeros without poses)."""
    mask = generate_mask(gt_depth, min_depth, max_depth, crop)
    pred, gt = pred_zoomed[mask], gt_depth[mask]
    out = np.zeros((2, 7))
    with np.errstate(divide='ignore', invalid='ignore'):
        if poses is not None:
            disp = pose_norms(poses)
            scale_factors = [s1 / s2 for s1, s2 in zip(np.asarray(displacements, np.float64), disp) if s1 > 0]
            scale_factor = np.mean(scale_factors) if len(scale_factors) > 0 else 0
            out[0] = compute_errors(gt, pred * scale_factor)
        scale_factor = np.median(gt) / np.median(pred)
        out[1] = compute_errors(gt, pred * scale_factor)
    return out

