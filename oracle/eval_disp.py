"""test_disp.py restated on numpy, scipy, Pillow and torch's CPU ops: both test frameworks (kitti_eval/ and
stillbox_eval/depth_evaluation_utils.py: read_scene_data, get_displacements, the velodyne ground truth and the masks),
the script's sample loop (test_disp.py:58-155) one sample at a time, and its --output-dir images (:104-121) with
matplotlib's 'hot' (N = 256) and tensor2array.  The nets are the oracle's functional forwards: DispResNet6
(oracle.nets.disp_forward) and the pose trunks of PoseNetB6, PoseNet6 and PoseExpNet (pose_forward below).
tests/golden/test_disp_small.npz holds what the reference's own main() printed, computed and wrote for the same trees;
tests/golden/make_test_disp.py runs it."""
import datetime
import json
import os
import numpy as np
import torch
import torch.nn.functional as F
from scipy import interpolate
from scipy.ndimage import zoom
from . import depth_eval as OD, nets as ON, run_inference as ORI
from .make3d_eval import imresize

HOT_DATA = {'red': ((0., 0.0416, 0.0416), (0.365079, 1.0, 1.0), (1.0, 1.0, 1.0)),
            'green': ((0., 0., 0.), (0.365079, 0., 0.), (0.746032, 1.0, 1.0), (1.0, 1.0, 1.0)),
            'blue': ((0., 0., 0.), (0.746032, 0., 0.), (1.0, 1.0, 1.0))}
HOT = ORI.LinearSegmentedColormap('hot', HOT_DATA, 256)


def hot_table():
    """The uint8 [256,3] image of every colour of 'hot', as (255 * ...).astype(np.uint8) makes it."""
    HOT(np.zeros(1, np.float32))
    return (255 * HOT._lut[:HOT.N, :3].astype(np.float32)).astype(np.uint8)


def hot_image(x):
    """(255 * tensor2array(x, None, 'hot')).astype(np.uint8) of a float32 [H,W] map, HWC."""
    x = np.asarray(x, np.float32)
    arr = HOT(x / x.max()).astype(np.float32)[:, :, :3]
    return (255 * arr).astype(np.uint8)


def input_image(tgt):
    """(255 * tensor2array(tgt)).astype(np.uint8) of a normalised [3,h,w] float32 frame (0.5 + x * 0.5), HWC."""
    return np.ascontiguousarray((255 * (0.5 + np.asarray(tgt, np.float32) * 0.5)).astype(np.uint8).transpose(1, 2, 0))


# ---- frameworks ---------------------------------------------------------------------------------------------------------
def _shifts(seq_length):
    d = (seq_length - 1) // 2
    return [i for i in range(-d, d + 1) if i != 0]


def _calib(path):
    out = {}
    for line in open(path).read().splitlines():
        key, value = line.split(':', 1)
        try:
            out[key] = np.array([float(v) for v in value.split()])
        except ValueError:
            pass
    return out


def projection(calib_dir, cam):
    """P_rect_0<cam> @ R_rect_00 (4x4) @ [R | T] (4x4) of a date's two calibration files."""
    c2c, v2c = _calib(os.path.join(calib_dir, 'calib_cam_to_cam.txt')), _calib(os.path.join(calib_dir, 'calib_velo_to_cam.txt'))
    velo2cam = np.eye(4)
    velo2cam[:3, :3], velo2cam[:3, 3] = v2c['R'].reshape(3, 3), v2c['T']
    rect = np.eye(4)
    rect[:3, :3] = c2c['R_rect_00'].reshape(3, 3)
    return np.dot(np.dot(c2c['P_rect_0%d' % cam].reshape(3, 4), rect), velo2cam)


def read_frame(path):
    from PIL import Image
    return np.asarray(Image.open(path)).astype(np.float32)


def kitti_framework(root, test_files, seq_length, printed):
    """-> samples: dict(path, tgt, refs, gt_depth, displacements, crop) per existing target; messages appended to printed."""
    shifts = _shifts(seq_length)
    printed.append('getting test metadata ... ')
    samples = []
    for f in test_files:
        tgt = os.path.join(root, f)
        date, drive, cam, _, index = f[:-4].split('/')
        index = int(index)
        if not os.path.isfile(tgt):
            printed.append('%s missing' % tgt)
            continue
        refs, used = [], []
        for s in shifts:
            r = os.path.join(os.path.dirname(tgt), '%010d.png' % (index + s))
            refs.append(r if os.path.isfile(r) else tgt)
            used.append(s if os.path.isfile(r) else 0)
        oxts = os.path.join(root, date, drive, 'oxts')
        stamps = [datetime.datetime.strptime(t[:-3], '%Y-%m-%d %H:%M:%S.%f').timestamp()
                  for t in open(os.path.join(oxts, 'timestamps.txt')).read().splitlines()]
        speed = np.linalg.norm(np.genfromtxt(os.path.join(oxts, 'data', '%010d.txt' % index))[8:11])
        img = read_frame(tgt)
        points = np.fromfile(os.path.join(root, date, drive, 'velodyne_points', 'data', '%010d.bin' % index),
                             np.float32).reshape(-1, 4)
        gt = OD.generate_depth_map(points, projection(os.path.join(root, date), int(cam[-2:])), img.shape[:2])
        samples.append(dict(path=tgt, tgt=img, refs=[read_frame(r) for r in refs], gt_depth=gt, crop=OD.EIGEN,
                            displacements=np.array([speed * abs(stamps[index] - stamps[index + s]) for s in used])))
    return samples


def stillbox_framework(root, test_files, seq_length, printed):
    meta = {d: json.load(open(os.path.join(root, d, 'metadata.json'))) for d in os.listdir(root)
            if os.path.isdir(os.path.join(root, d))}
    shifts = _shifts(seq_length)
    printed.append('getting test metadata ... ')
    samples = []
    for f in test_files:
        folder, name = f.split('/')
        _, scene_index, index = name[:-4].split('_')
        index = int(index)
        scene = meta[folder]['scenes'][int(scene_index)]
        tgt = os.path.join(root, f)
        if not os.path.isfile(tgt):
            printed.append('%s missing' % tgt)
            continue
        idx = [int(np.clip(index + s, 0, scene['length'] - 1)) for s in shifts]
        speed = np.around(np.linalg.norm(scene['speed']), decimals=3)
        samples.append(dict(path=tgt, tgt=read_frame(tgt), refs=[read_frame(os.path.join(root, folder, scene['imgs'][i]))
                                                                 for i in idx],
                            gt_depth=np.load(os.path.join(root, folder, scene['depth'][index])), crop=OD.STILLBOX,
                            displacements=np.array([speed * scene['time_step'] * abs(index - i) for i in idx])))
    return samples


# ---- nets ---------------------------------------------------------------------------------------------------------------
def pose_forward(p, tgt, refs):
    """The pose of PoseNetB6 (8 convolutions), PoseExpNet (7) or PoseNet6 (conv0 then 7): stride-2 convolutions with
    ReLU, the 1x1 pose_pred, the spatial mean, times 0.01."""
    nb = p['pose_pred.weight'].size(0) // 6
    x = torch.cat([tgt] + list(refs), 1)
    names = [n for n in ['conv%d' % i for i in range(9)] if n + '.0.weight' in p]
    for n in names:
        w = p[n + '.0.weight']
        x = F.relu(F.conv2d(x, w, p[n + '.0.bias'], 2, (w.shape[-1] - 1) // 2))
    pose = F.conv2d(x, p['pose_pred.weight'], p['pose_pred.bias']).mean(3).mean(2)
    return 0.01 * pose.view(pose.size(0), nb, 6)


def net_input(img, h, w, no_resize):
    """test_disp.py:80-89: float32 HxWx3 -> [1,3,h,w], imresize'd unless no_resize or already h x w, (x/255 - 0.5)/0.5."""
    if not no_resize and img.shape[:2] != (h, w):
        img = imresize(img, (h, w)).astype(np.float32)
    t = torch.from_numpy(np.ascontiguousarray(np.transpose(img, (2, 0, 1)))).unsqueeze(0)
    return (t / 255 - 0.5) / 0.5


def interp_gt_disp(mat):
    """test_disp.py:157-169 on a copy."""
    mat = np.array(mat, np.float64)
    mat[mat == 0] = np.nan
    xx, yy = np.meshgrid(np.arange(mat.shape[1]), np.arange(mat.shape[0]))
    valid = np.isfinite(mat)
    return interpolate.griddata((xx[valid], yy[valid]), mat[valid], (xx, yy), method='linear', fill_value=0)


def run(gt_type, test_files, dataset_dir, Pd, Pp=None, img_height=256, img_width=832, no_resize=False,
        spatial_normalize=False, min_depth=1e-3, max_depth=80.0, output=False):
    """test_disp.py main() on parameter dicts (any dtype: fp64 for the oracle nets) -> dict(stdout, errors float32
    [2,7,N], and with output: predictions fp64 [N,h,w] and images {'0000img.png': uint8 HWC, ...})."""
    printed = []
    seq_length = 0
    if Pp is None:
        printed.append('no PoseNet specified, scale_factor will be determined by median ratio, which is kiiinda cheating'
                       '            (but consistent with original paper)')
    else:
        seq_length = Pp['conv1.0.weight'].size(1) // 3
    framework = kitti_framework if gt_type == 'KITTI' else stillbox_framework
    samples = framework(dataset_dir, test_files, seq_length, printed)
    printed.append('%d files to test' % len(test_files))
    errors = np.zeros((2, 7, len(test_files)), np.float32)
    dtype = Pd['conv1.0.weight'].dtype
    predictions, images = None, {}
    for j, s in enumerate(samples):
        tgt = net_input(s['tgt'], img_height, img_width, no_resize)
        refs = [net_input(r, img_height, img_width, no_resize) for r in s['refs']]
        with torch.no_grad():
            disp = ON.disp_forward(Pd, tgt.to(dtype), training=False)
            if spatial_normalize:
                disp = disp / disp.mean(dim=1, keepdim=True).mean(dim=2, keepdim=True).mean(dim=3, keepdim=True)
        pred_disp = disp.float().numpy()[0, 0]
        gt = s['gt_depth']
        if output:
            if predictions is None:
                predictions = np.zeros((len(test_files),) + pred_disp.shape)
            predictions[j] = 1 / pred_disp
            g = interp_gt_disp(gt).astype(np.float32)
            g[g == 0] = 1000
            name = '%04d' % j
            images[name + 'img.png'] = input_image(tgt[0].numpy())
            images[name + 'depth.png'] = hot_image(pred_disp)
            images[name + 'gt.png'] = hot_image(np.clip(1 / g, 0, 10))
        z = zoom(1 / pred_disp, (gt.shape[0] / pred_disp.shape[0], gt.shape[1] / pred_disp.shape[1])).clip(min_depth, max_depth)
        mask = OD.generate_mask(gt, min_depth, max_depth, s['crop'])
        z, g = z[mask], gt[mask]
        if seq_length > 0:
            with torch.no_grad():
                poses = pose_forward(Pp, tgt.to(dtype), [r.to(dtype) for r in refs]).float()
            norms = poses[0, :, :3].norm(2, 1).numpy()
            sf = [a / b for a, b in zip(s['displacements'], norms) if a > 0]
            if not sf:
                printed.append('not good !  %s %s' % (s['path'], s['displacements']))
            errors[0, :, j] = OD.compute_errors(g, z * (np.mean(sf) if sf else 0))
        with np.errstate(divide='ignore', invalid='ignore'):
            errors[1, :, j] = OD.compute_errors(g, z * (np.median(g) / np.median(z)))
    mean = errors.mean(2)
    names = ['abs_rel', 'sq_rel', 'rms', 'log_rms', 'a1', 'a2', 'a3']
    rows = [0, 1] if Pp is not None else [1]
    for r in rows:
        printed.append('Results with scale factor determined by PoseNet : ' if r == 0 else
                       'Results with scale factor determined by GT/prediction ratio (like the original paper) : ')
        printed.append(', '.join('%10s' % n for n in names))
        printed.append(', '.join('%10.4f' % v for v in mean[r]))
    return dict(stdout='\n'.join(printed) + '\n', errors=errors, predictions=predictions, images=images)
