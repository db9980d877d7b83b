"""test_make3d.py's evaluation restated on numpy, Pillow and scipy: scipy 1.1's imresize of a float32 image (toimage's
bytescale, then Pillow's BILINEAR resize; test_make3d.py:100-102), compute_errors (:174-190) and the sample body
(:139-148).  tests/golden/make3d_eval_small.npz holds what the reference's own code returns for the same inputs."""
import warnings
import numpy as np


def bytescale(img):
    """scipy 1.1 bytescale of a float32 image: cmin, cmax over the whole array, every step in float32."""
    x = np.asarray(img, np.float32)
    cmin, cmax = x.min(), x.max()
    cscale = cmax - cmin
    if cscale == 0:
        cscale = np.float32(1)
    scale = np.float32(255) / cscale
    return (((x - cmin) * scale).clip(0, 255) + np.float32(0.5)).astype(np.uint8)


def imresize(img, size):
    """scipy.misc.imresize(float32 HxWx3, (h, w)) (bilinear) -> uint8 [h,w,3]."""
    from PIL import Image
    return np.array(Image.fromarray(bytescale(img)).resize((size[1], size[0]), Image.BILINEAR))


def net_input(tgt_img, h=256, w=256, resize=True):
    """test_make3d.py:98-106: the float32 HxWx3 crop -> [1,3,h,w] fp32 numpy in [-1, 1]."""
    x = np.asarray(tgt_img, np.float32)
    if resize and x.shape[:2] != (h, w):
        x = imresize(x, (h, w)).astype(np.float32)
    x = np.transpose(x, (2, 0, 1))[None]
    return (x / np.float32(255) - np.float32(0.5)) / np.float32(0.5)


def compute_errors(gt, pred):
    """test_make3d.py:174-190: test_disp's errors with log_rms in log10."""
    with np.errstate(divide='ignore', invalid='ignore'), warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)            # an empty mask: means of empty arrays are nan
        thresh = np.maximum((gt / pred), (pred / gt))
        a1 = (thresh < 1.25).mean()
        a2 = (thresh < 1.25 ** 2).mean()
        a3 = (thresh < 1.25 ** 3).mean()
        rmse = np.sqrt(((gt - pred) ** 2).mean())
        rmse_log = np.sqrt(((np.log10(gt) - np.log10(pred)) ** 2).mean())
        abs_rel = np.mean(np.abs(gt - pred) / gt)
        sq_rel = np.mean(((gt - pred) ** 2) / gt)
    return abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3


def sample_errors(gt_depth, pred_zoomed, min_depth=1e-3, max_depth=70.0):
    """test_make3d.py:141-148 of one sample: gt_depth fp64 [21,C], pred_zoomed the zoomed, clipped fp32 prediction ->
    fp64 [2,7], row 0 zeros."""
    mask = np.logical_and(gt_depth > min_depth, gt_depth < max_depth)
    pred, gt = pred_zoomed[mask], gt_depth[mask]
    out = np.zeros((2, 7))
    with np.errstate(divide='ignore', invalid='ignore'), warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)
        scale_factor = np.median(gt) / np.median(pred)            # an empty mask: nan
        pred = scale_factor * pred
        pred[pred > max_depth] = max_depth
        out[1] = compute_errors(gt, pred)
    return out
