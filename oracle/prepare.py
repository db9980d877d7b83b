"""data/prepare_train_data.py with data/kitti_raw_loader.py and data/cityscapes_loader.py restated on numpy and Pillow,
one scene after another in one process: scipy.misc.imread is np.asarray(Image.open(p)), imresize of a uint8 RGB frame is
Pillow's BILINEAR resize, imsave of one is Image.fromarray(a).save(p), and the depth map is oracle.depth_eval's
generate_depth_map (the reference's duplicate loop and sub2ind key) at the output size, as float32.
tests/golden/prepare_small.npz holds what the reference itself writes for the trees of tests/prepare_cases.py."""
import json
import os
import shutil
import fnmatch
import numpy as np
from PIL import Image

from oracle.depth_eval import generate_depth_map

DATES = ['2011_09_26', '2011_09_28', '2011_09_29', '2011_09_30', '2011_10_03']


def _dirs(p):
    return [os.path.join(p, f) for f in os.listdir(p) if os.path.isdir(os.path.join(p, f))]


def _files(p, pattern):
    return [os.path.join(p, f) for f in os.listdir(p) if os.path.isfile(os.path.join(p, f)) and fnmatch.fnmatch(f, pattern)]


def _calib(path):
    out = {}
    with open(path) as f:
        for line in f:
            key, value = line.split(':', 1)
            try:
                out[key] = np.array([float(x) for x in value.split()])
            except ValueError:
                pass
    return out


def _by_speed(speeds):
    acc = np.zeros(3)
    for i, s in enumerate(speeds):
        acc += s
        if np.linalg.norm(acc) > 2:
            yield i
            acc *= 0


def _resize(a, h, w):
    return np.asarray(Image.fromarray(np.asarray(a)).resize((w, h), Image.BILINEAR))


def kitti_scenes(raw, height, width, test_scenes, static=None, with_gt=False):
    """Every KITTI scene as (rel_path, intrinsics, [(frame id, uint8 frame, depth or None)])."""
    out = []
    drives = [d for date in DATES for d in _dirs(os.path.join(raw, date)) if os.path.basename(d)[:-5] not in test_scenes]
    for drive in drives:
        name = os.path.basename(drive)
        oxts = sorted(_files(os.path.join(drive, 'oxts', 'data'), '*.txt'))
        ids = ['%010d' % n for n in range(len(oxts))]
        spd = [np.genfromtxt(f)[8:11] for f in oxts]
        png = lambda cam, fid: os.path.join(drive, 'image_' + cam, 'data', fid + '.png')     # noqa: E731
        if not all(os.path.isfile(png(c, ids[0])) for c in ('02', '03')):
            continue
        calib = _calib(os.path.join(os.path.dirname(drive), 'calib_cam_to_cam.txt'))
        velo = _calib(os.path.join(os.path.dirname(drive), 'calib_velo_to_cam.txt'))
        v2c = np.vstack((np.hstack((velo['R'].reshape(3, 3), velo['T'][:, None])), [0, 0, 0, 1.0]))
        R4 = np.eye(4)
        R4[:3, :3] = calib['R_rect_00'].reshape(3, 3)
        for cam in ('02', '03'):
            h0, w0 = np.asarray(Image.open(png(cam, ids[0]))).shape[:2]
            P = calib['P_rect_' + cam].reshape(3, 4).copy()
            P[0] *= width / w0
            P[1] *= height / h0
            P_velo = np.dot(np.dot(P, R4), v2c)
            if static is None:
                keep = list(_by_speed(spd))
            else:
                keep = [i for i, f in enumerate(ids) if f not in static.get(name, ())]
            frames = []
            for i in keep:
                img = _resize(np.asarray(Image.open(png(cam, ids[i]))), height, width)
                depth = None
                if with_gt:
                    pts = np.fromfile(os.path.join(drive, 'velodyne_points', 'data', ids[i] + '.bin'), np.float32)
                    depth = generate_depth_map(pts.reshape(-1, 4), P_velo, (height, width)).astype(np.float32)
                frames.append((ids[i], img, depth))
            out.append((name + '_' + cam, P[:, :3], frames))
    return out


def cityscapes_scenes(raw, height, width):
    """Every Cityscapes sub-scene as (rel_path, intrinsics, [(frame id, uint8 frame, None)])."""
    out = []
    for city in _dirs(os.path.join(raw, 'leftImg8bit_sequence', 'train')):
        cname = os.path.basename(city)
        scenes = {}
        for f in sorted(_files(city, '*.png')):
            sid, fid = os.path.basename(f).split('_')[1:3]
            scenes.setdefault(sid, []).append(fid)
        for sid, fids in scenes.items():
            cam = _files(os.path.join(raw, 'camera', 'train', cname), '%s_%s_*_camera.json' % (cname, sid))[0]
            with open(cam) as f:
                c = json.load(f)['intrinsic']
            K = np.array([[c['fx'], 0, c['u0']], [0, c['fy'], c['v0']], [0, 0, 1]])
            h0, w0 = np.asarray(Image.open(os.path.join(city, '%s_%s_%s_leftImg8bit.png' % (
                cname, sid, cam.split('_')[2])))).shape[:2]
            K[0] *= width / w0
            K[1] *= height / h0
            runs = []
            for k, fid in enumerate(fids):
                if k == 0 or int(fid) - int(fids[k - 1]) > 1:
                    runs.append([])
                runs[-1].append(fid)
            for run in runs:
                for half in (0, 1):
                    sub = run[half::2]
                    spd = []
                    for fid in sub:
                        with open(os.path.join(raw, 'vehicle_sequence', 'train', cname,
                                               '%s_%s_%s_vehicle.json' % (cname, sid, fid))) as f:
                            spd.append(json.load(f)['speed'])
                    frames = []
                    for i in _by_speed(spd):
                        img = np.asarray(Image.open(os.path.join(city, '%s_%s_%s_leftImg8bit.png' % (cname, sid, sub[i]))))
                        frames.append((sub[i], _resize(img, height, width)[:int(height * 0.75)], None))
                    out.append(('%s_%s_%s_%d' % (cname, sid, run[0], half), K, frames))
    return out


def static_frames(path):
    out = {}
    with open(path) as f:
        for line in f:
            if line == '\n':
                continue
            _, drive, fid = line.split(' ')
            out.setdefault(drive, set()).add('%.10d' % int(fid[:-1]))
    return out


def prepare(raw, fmt, dump, height=128, width=416, static=None, with_gt=False, test_scenes=None):
    """Write the dump as the reference does -> dict(frames={rel jpg: uint8}, depth={rel npy: float32}, order=[the
    folders in listdir order at the split], train=[...], val=[...]).  `static` and `test_scenes` are file paths."""
    os.makedirs(dump, exist_ok=True)
    if fmt == 'kitti':
        with open(test_scenes) as f:
            scenes = kitti_scenes(raw, height, width, [t[:-1] for t in f.readlines()],
                                  static_frames(static) if static else None, with_gt)
    else:
        scenes = cityscapes_scenes(raw, height, width)
    rec = dict(frames={}, depth={})
    for rel, K, frames in scenes:
        d = os.path.join(dump, rel)
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, 'cam.txt'), 'w') as f:
            f.write('%f,0.,%f,0.,%f,%f,0.,0.,1.' % (K[0, 0], K[0, 2], K[1, 1], K[1, 2]))
        for fid, img, depth in frames:
            Image.fromarray(img).save(os.path.join(d, fid + '.jpg'))
            rec['frames'][rel + '/' + fid + '.jpg'] = img
            if depth is not None:
                np.save(os.path.join(d, fid + '.npy'), depth)
                rec['depth'][rel + '/' + fid + '.npy'] = depth
        if len(_files(d, '*.jpg')) < 3:
            shutil.rmtree(d)
            for kind in ('frames', 'depth'):
                rec[kind] = {k: v for k, v in rec[kind].items() if not k.startswith(rel + '/')}
    rs = np.random.RandomState(8964)
    rec['order'] = [os.path.basename(p) for p in _dirs(dump)]
    rec['train'], rec['val'] = [], []
    for name in rec['order']:
        if rs.random_sample() < 0.1:
            rec['val'].append(name)
        else:
            rec['train'].append(name)
            for f in _files(os.path.join(dump, name), '*.npy'):
                os.remove(f)
    for split in ('train', 'val'):
        with open(os.path.join(dump, split + '.txt'), 'w') as f:
            f.write(''.join(n + '\n' for n in rec[split]))
    return rec
