"""Oracle: the per-sample body of the reference's motion segmentation benchmark (test_mask.py:119-156, mask_error :224-262)
restated on the functional oracle nets, beside the other evaluation loops of oracle/evaluate.py.  TEST INFRASTRUCTURE."""
import numpy as np
import torch
from . import nets as ON, geometry as OG


def mask_error(mot_gt, seg_gt, pred):
    """test_mask.py:224-262: [tp_0, fp_0, fn_0, tp_1, fp_1, fn_1] of a rigidity mask `pred` (1 = rigid = class 0) against
    the object map, over the pixels whose semantic label is 26 (car).
    The reference relabels its `mot_gt` argument in place and the script calls it three times on the same array, so the
    second and third calls see labels 0 / 1 / 255.  The relabelling is idempotent (non-zero -> 1, then 255 wherever the
    semantic label is not 26: a 255 from an earlier call lies outside the car pixels and becomes 255 again), so labelling
    a copy once per call gives what each of the three calls computes."""
    from scipy.ndimage import zoom
    gt = np.array(mot_gt)
    gt[gt != 0] = 1
    gt[seg_gt != 26] = 255
    pred = zoom(pred, (float(gt.shape[0]) / float(pred.shape[0]), float(gt.shape[1]) / float(pred.shape[1])), order=0)
    label = np.stack([pred, 1. - pred]).argmax(axis=0)
    out = []
    for class_id in range(2):
        class_gt = gt == class_id
        class_result = (label == class_id) & (gt != 255)
        out += [np.count_nonzero(class_gt & class_result), np.count_nonzero(class_result & ~class_gt),
                np.count_nonzero(~class_result & class_gt)]
    return [float(v) for v in out]


def mask_sample_errors(P, tgt, refs, K, Kinv, obj_map, semantic_map, THRESH=0.94, flownet='Back2Future'):
    """test_mask.py:119-156 for one sample (batch 1, where the bare mask's broadcast means what it says); P as in
    flow_sample_errors -> (errors, errors_census, errors_bare, masks [4,h,w] = combined, census, bare, soft census)."""
    with torch.no_grad():
        disp = ON.disp_forward(P['disp'], tgt, training=False)
        depth = 1 / disp
        pose = ON.pose_forward(P['pose'], tgt, refs)
        emask = ON.mask_forward(P['mask'], tgt, refs, training=False)
        flow_fwd = ON.flow_eval(P['flow'], tgt, refs, flownet)
        flow_cam = OG.pose2flow(depth.squeeze(1), pose[:, 2], K, Kinv)
        bare, census, combined, soft = rigidity_masks(emask, flow_cam, flow_fwd, THRESH)
    gt, seg = obj_map[0].numpy(), semantic_map[0].numpy()
    errs = [mask_error(gt, seg, m[0, 0].numpy()) for m in (combined, census, bare)]
    masks = torch.cat([combined, census.type_as(combined), bare.type_as(combined), soft], 1)[0]
    return errs[0], errs[1], errs[2], masks


def rigidity_masks(emask, flow_cam, flow_fwd, THRESH):
    """test_mask.py:129-134 at batch 1: (bare, census) bool and (combined, soft) float, each [1,1,h,w].
    The square root is taken in fp64 and rounded to fp32, which is the correctly rounded fp32 root: torch's vectorised fp32
    sqrt on the CPU can be an ulp off (seen with the AVX-512 kernels of torch 2.11 on about 1 % of random inputs), and the
    census threshold turns that ulp into a pixel."""
    assert emask.shape[0] == 1
    bare = 1 - (1 - emask[:, 1]) * (1 - emask[:, 2]).unsqueeze(1) > 0.5
    soft = (flow_cam - flow_fwd).pow(2).sum(dim=1).unsqueeze(1).double().sqrt().float()
    soft = 1 - soft / soft.max()
    census = soft > THRESH
    combined = 1 - (1 - bare.type_as(emask)) * (1 - census.type_as(emask))
    return bare, census, combined, soft
