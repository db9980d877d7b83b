"""The reference's data/prepare_train_data.py (with data/kitti_raw_loader.py and data/cityscapes_loader.py) on this
stack: `python -m cc_b200.prepare_train_data RAW --dataset-format kitti|cityscapes --dump-root OUT ...` writes the
training dump cc_b200.train reads, the same files as the reference writes.

  scenes      kitti_scenes / cityscapes_scenes: the reference's scenes (one drive x one camera, or one Cityscapes
              sub-sequence) and their frames, chosen on the host by its rules (select_by_speed, read_static_frames).
  frames      host worker processes decode the PNGs (np.asarray(Image.open(p)), what scipy.misc.imread returned) and read
              the velodyne sweeps; each chunk of a scene is resized on the device as Pillow's BILINEAR resize does
              (input_pipeline.resize_frames: scipy.misc.imresize of a uint8 frame) and, with --with-gt, its depth maps
              are projected in one call (evaluate.velodyne_depth: generate_depth_map with its sub2ind key) at the output
              size, cast to float32.  The workers encode the JPEGs (Image.fromarray(a).save(p), what scipy.misc.imsave
              of a uint8 RGB frame wrote) and write the .npy files.
  dump        write_scene: cam.txt, <frame>.jpg, <frame>.npy; a folder with fewer than 3 jpgs is removed.
              split: every folder of the dump in os.listdir order, one draw each of np.random.RandomState(8964) (the
              reference's np.random.seed(8964) stream): below 0.1 to val.txt, else to train.txt and its .npy removed.

Documented deviations:
  --test-scenes FILE   required with --dataset-format kitti: the reference reads the test_scenes.txt beside its loader
                       (data/test_scenes.txt of the reference); here the user names that list.
  workers              the reference runs one joblib process per scene; here the device work runs in this process and
                       --num-threads host processes decode and encode.  The dump is the same for any --num-threads.
  errors               a missing date folder, frame or velodyne file is an error that names it (the reference crashes)."""
import argparse
import fnmatch
import json
import multiprocessing
import os
import shutil
import sys
import numpy as np

DATES = ('2011_09_26', '2011_09_28', '2011_09_29', '2011_09_30', '2011_10_03')
CAMERAS = ('02', '03')
MIN_SPEED = 2
CHUNK = 64                      # frames per device batch: 64 KITTI frames are 89 MB of uint8


# ---- files -----------------------------------------------------------------------------------------------------------
def _dirs(p):
    """path.Path(p).dirs(): the sub-folders of p in os.listdir order."""
    return [os.path.join(p, f) for f in os.listdir(p) if os.path.isdir(os.path.join(p, f))]


def _files(p, pattern):
    """path.Path(p).files(pattern): the regular files of p whose name matches, in os.listdir order."""
    return [os.path.join(p, f) for f in os.listdir(p) if os.path.isfile(os.path.join(p, f)) and fnmatch.fnmatch(f, pattern)]


def _need(path, what):
    if not os.path.isfile(path):
        raise FileNotFoundError('%s not found: %s' % (what, path))
    return path


def read_raw_calib_file(path):
    """kitti_raw_loader.read_raw_calib_file: {key: fp64 array of value.split()}; a key whose value does not parse as
    numbers is dropped (unlike evaluate.read_calib_file, which splits on ' ' and keeps such a value as a string)."""
    data = {}
    with open(path) as f:
        for line in f:
            key, value = line.split(':', 1)
            try:
                data[key] = np.array([float(x) for x in value.split()])
            except ValueError:
                pass
    return data


def read_test_scenes(path):
    """The drive names (without _sync) to leave out, each line minus its last character as the reference reads them."""
    with open(path) as f:
        return [t[:-1] for t in f.readlines()]


def read_static_frames(path):
    """collect_static_frames: {drive folder name: frame ids} from `date drive frame` lines, blank lines skipped; the frame
    id is '%.10d' % int(frame[:-1]), so a last line without a newline loses its last digit, as in the reference."""
    out = {}
    with open(path) as f:
        for line in f:
            if line == '\n':
                continue
            date, drive, frame = line.split(' ')
            out.setdefault(drive, set()).add('%.10d' % int(frame[:-1]))
    return out


# ---- scenes ----------------------------------------------------------------------------------------------------------
def select_by_speed(speeds, min_speed=MIN_SPEED):
    """The indices get_scene_imgs yields: each speed (a 3-vector, or a scalar added to all three components) is added to
    a running fp64 sum; a frame is kept when the sum's norm exceeds min_speed, and the sum is then reset."""
    acc = np.zeros(3)
    out = []
    for i, s in enumerate(speeds):
        acc += s
        if np.linalg.norm(acc) > min_speed:
            out.append(i)
            acc *= 0
    return out


def _image_size(path):
    from PIL import Image
    with Image.open(path) as im:
        return im.size[1], im.size[0]


def kitti_drives(raw, test_scenes):
    """collect_train_folders: the drive folders of each date in DATES, in listdir order, without the test scenes."""
    drives = []
    for date in DATES:
        d = os.path.join(raw, date)
        if not os.path.isdir(d):
            raise FileNotFoundError('KITTI date folder not found: %s (every date of %s must exist)' % (d, ', '.join(DATES)))
        drives += [dr for dr in _dirs(d) if os.path.basename(dr)[:-5] not in test_scenes]
    return drives


def kitti_scenes(drive, height, width, static=None, with_gt=False):
    """collect_scenes + get_scene_imgs of one drive: a scene per camera 02, 03 as dict(rel_path, intrinsics,
    frames=[(frame id, png)], sweeps=[bin] or None, P_velo2im fp64 [3,4] or None, crop=None).  Frame ids number the
    sorted oxts files; no scene at all when frame 0 of either camera is missing.  P_rect_0<cam> is scaled by the output
    size over frame 0's size before the projection P_rect @ R_cam2rect @ velo2cam is built."""
    oxts = sorted(_files(os.path.join(drive, 'oxts', 'data'), '*.txt'))
    if not oxts:
        raise FileNotFoundError('no oxts/data/*.txt in KITTI drive %s' % drive)
    ids = ['{:010d}'.format(n) for n in range(len(oxts))]
    png = lambda c, i: os.path.join(drive, 'image_' + c, 'data', ids[i] + '.png')        # noqa: E731
    if not all(os.path.isfile(png(c, 0)) for c in CAMERAS):
        return []
    name = os.path.basename(drive)
    if static is None:
        keep = select_by_speed([np.genfromtxt(f)[8:11] for f in oxts])
    else:
        keep = [i for i, f in enumerate(ids) if f not in static.get(name, ())]
    calib_dir = os.path.dirname(drive)
    cam2cam = read_raw_calib_file(os.path.join(calib_dir, 'calib_cam_to_cam.txt'))
    velo2cam = read_raw_calib_file(os.path.join(calib_dir, 'calib_velo_to_cam.txt')) if with_gt else None
    scenes = []
    for c in CAMERAS:
        h0, w0 = _image_size(png(c, 0))
        P_rect = np.reshape(cam2cam['P_rect_' + c], (3, 4)).copy()
        P_rect[0] *= width / w0
        P_rect[1] *= height / h0
        scene = dict(rel_path=name + '_' + c, intrinsics=P_rect[:, :3], frames=[(ids[i], png(c, i)) for i in keep],
                     sweeps=None, P_velo2im=None, crop=None)
        if with_gt:
            R_cam2rect = np.eye(4)
            R_cam2rect[:3, :3] = cam2cam['R_rect_00'].reshape(3, 3)
            v2c = np.hstack((velo2cam['R'].reshape(3, 3), velo2cam['T'][..., np.newaxis]))
            v2c = np.vstack((v2c, np.array([0, 0, 0, 1.0])))
            scene['P_velo2im'] = np.dot(np.dot(P_rect, R_cam2rect), v2c)
            scene['sweeps'] = [os.path.join(drive, 'velodyne_points', 'data', ids[i] + '.bin') for i in keep]
        scenes.append(scene)
    return scenes


def cityscapes_cities(raw):
    d = os.path.join(raw, 'leftImg8bit_sequence', 'train')
    if not os.path.isdir(d):
        raise FileNotFoundError('Cityscapes folder not found: %s' % d)
    return _dirs(d)


def cityscapes_scenes(city, raw, height, width):
    """cityscapes_loader.collect_scenes + get_scene_imgs of one city: its frames grouped by scene id, cut into connected
    runs where the frame number jumps by more than 1, each run split into its even (`_0`) and odd (`_1`) positions;
    frames chosen by select_by_speed of the scalar vehicle speeds; resized to (height, width), then cropped to rows
    [:int(height * 0.75)].  The intrinsics come from the first camera json of the scene in listdir order, scaled by the
    size of the frame whose id the reference takes from the json's whole path split on '_'."""
    cname = os.path.basename(city)
    scenes = {}
    for f in sorted(_files(city, '*.png')):
        scene_id, frame_id = os.path.basename(f).split('_')[1:3]
        scenes.setdefault(scene_id, []).append(frame_id)
    out = []
    for scene_id, frame_ids in scenes.items():
        cams = _files(os.path.join(raw, 'camera', 'train', cname), '{}_{}_*_camera.json'.format(cname, scene_id))
        if not cams:
            raise FileNotFoundError('no camera json for Cityscapes scene %s_%s under %s' % (
                cname, scene_id, os.path.join(raw, 'camera', 'train', cname)))
        with open(cams[0]) as f:
            cam = json.load(f)['intrinsic']
        K = np.array([[cam['fx'], 0, cam['u0']], [0, cam['fy'], cam['v0']], [0, 0, 1]])
        sized = os.path.join(city, '{}_{}_{}_leftImg8bit.png'.format(cname, scene_id, cams[0].split('_')[2]))
        h0, w0 = _image_size(_need(sized, "the frame of the camera json (its id is the json path's third '_' field; "
                                          "a dataset path with '_' in it misplaces it, as in the reference)"))
        K[0] *= width / w0
        K[1] *= height / h0
        runs = []
        for k, fid in enumerate(frame_ids):
            if k == 0 or int(fid) - int(frame_ids[k - 1]) > 1:
                runs.append([])
            runs[-1].append(fid)
        for run in runs:
            for half in (0, 1):
                sub = run[half::2]
                speeds = []
                for fid in sub:
                    with open(os.path.join(raw, 'vehicle_sequence', 'train', cname,
                                           '{}_{}_{}_vehicle.json'.format(cname, scene_id, fid))) as f:
                        speeds.append(json.load(f)['speed'])
                frames = [(sub[i], os.path.join(city, '{}_{}_{}_leftImg8bit.png'.format(cname, scene_id, sub[i])))
                          for i in select_by_speed(speeds)]
                out.append(dict(rel_path='%s_%s_%s_%d' % (cname, scene_id, run[0], half), intrinsics=K, frames=frames,
                                sweeps=None, P_velo2im=None, crop=int(height * 0.75)))
    return out


# ---- host workers ----------------------------------------------------------------------------------------------------
def load_frame(png, sweep):
    """One frame's inputs in a worker: the decoded uint8 RGB PNG, and the velodyne sweep (float32 [N,4], column 3 set to
    1) or None."""
    from PIL import Image
    with Image.open(_need(png, 'frame')) as im:
        img = np.asarray(im)
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
        raise ValueError('%s: expected an 8-bit RGB PNG, got %s %s' % (png, img.dtype, img.shape))
    pts = None
    if sweep is not None:
        pts = np.fromfile(_need(sweep, 'velodyne file'), dtype=np.float32).reshape(-1, 4)
        pts[:, 3] = 1
    return img, pts


def write_frame(jpg, img, npy, depth):
    """imsave of the uint8 frame (Pillow's JPEG encoder, default settings) and np.save of the float32 depth map."""
    from PIL import Image
    Image.fromarray(img).save(jpg)
    if depth is not None:
        np.save(npy, depth)


# ---- device stages ---------------------------------------------------------------------------------------------------
def resize_chunk(imgs, height, width, device):
    """uint8 frames (any sizes) -> uint8 [n,height,width,3] on the device: one resize_frames call per source size."""
    import torch
    from .input_pipeline import resize_frames, to_device
    shapes = list(dict.fromkeys(a.shape for a in imgs))
    if len(shapes) == 1:
        return resize_frames(to_device(np.stack(imgs), device), height, width)
    out = torch.empty(len(imgs), height, width, 3, dtype=torch.uint8, device=device)
    for shape in shapes:
        idx = [i for i, a in enumerate(imgs) if a.shape == shape]
        src = to_device(np.stack([imgs[i] for i in idx]), device)
        out[torch.tensor(idx, device=device)] = resize_frames(src, height, width)
    return out


def depth_chunk(sweeps, P_velo2im, height, width, device):
    """float32 [n,height,width] on the device: generate_depth_map of each sweep through one velodyne_depth call, its fp64
    result cast as the reference's float32 depth array holds it."""
    import torch
    from .evaluate import velodyne_depth
    from .input_pipeline import to_device
    offsets = np.concatenate([[0], np.cumsum([len(p) for p in sweeps])]).astype(np.int64)
    P = np.repeat(np.asarray(P_velo2im, np.float64)[None], len(sweeps), 0)
    d = velodyne_depth(to_device(np.concatenate(sweeps), device), to_device(offsets, device), to_device(P, device),
                       height, width)
    return d.to(torch.float32)


def write_scene(scene, dump_root, height, width, device, pool):
    """The reference's dump_example for one scene: cam.txt, then chunks of CHUNK frames decoded by the pool (the next
    chunk's decode runs while the device works on this one), resized (and projected) on the device, encoded and written
    by the pool; the folder is removed when it holds fewer than 3 jpgs.  Returns the folder, or None when removed."""
    d = os.path.join(dump_root, scene['rel_path'])
    os.makedirs(d, exist_ok=True)
    K = scene['intrinsics']
    with open(os.path.join(d, 'cam.txt'), 'w') as f:
        f.write('%f,0.,%f,0.,%f,%f,0.,0.,1.' % (K[0, 0], K[0, 2], K[1, 1], K[1, 2]))
    frames, sweeps = scene['frames'], scene['sweeps']
    chunks = [range(i, min(i + CHUNK, len(frames))) for i in range(0, len(frames), CHUNK)]
    load = lambda c: pool.starmap_async(load_frame, [(frames[i][1], sweeps[i] if sweeps else None) for i in c])  # noqa: E731
    pending = load(chunks[0]) if chunks else None
    writes = []
    for k, c in enumerate(chunks):
        loaded = pending.get()
        pending = load(chunks[k + 1]) if k + 1 < len(chunks) else None
        imgs = resize_chunk([a for a, _ in loaded], height, width, device)
        if scene['crop'] is not None:
            imgs = imgs[:, :scene['crop']]
        depth = depth_chunk([p for _, p in loaded], scene['P_velo2im'], height, width, device) if sweeps else None
        imgs = imgs.cpu().numpy()
        depth = depth.cpu().numpy() if depth is not None else None
        writes.append(pool.starmap_async(write_frame, [
            (os.path.join(d, frames[i][0] + '.jpg'), imgs[j], os.path.join(d, frames[i][0] + '.npy'),
             depth[j] if depth is not None else None) for j, i in enumerate(c)]))
    for w in writes:
        w.get()
    if len(_files(d, '*.jpg')) < 3:
        shutil.rmtree(d)
        return None
    return d


def split(dump_root, seed=8964):
    """The train / val split over every folder of dump_root in os.listdir order (folders of earlier runs included): draw
    k of np.random.RandomState(seed) decides folder k, below 0.1 to val.txt, else to train.txt with its .npy removed.
    Returns (order, train, val)."""
    rs = np.random.RandomState(seed)
    order = [os.path.basename(s) for s in _dirs(dump_root)]
    train, val = [], []
    with open(os.path.join(dump_root, 'train.txt'), 'w') as tf, open(os.path.join(dump_root, 'val.txt'), 'w') as vf:
        for s in order:
            if rs.random_sample() < 0.1:
                vf.write(s + '\n')
                val.append(s)
            else:
                tf.write(s + '\n')
                train.append(s)
                for gt in _files(os.path.join(dump_root, s), '*.npy'):
                    os.remove(gt)
    return order, train, val


# ---- command line ----------------------------------------------------------------------------------------------------
def build_parser():
    p = argparse.ArgumentParser(description='Prepare the training dump of KITTI raw or Cityscapes sequences')
    a = p.add_argument
    a('dataset_dir', metavar='DIR', help='path to original dataset')
    a('--dataset-format', type=str, required=True, choices=['kitti', 'cityscapes'])
    a('--static-frames', default=None, help='list of imgs to discard for being static, if not set will discard them '
                                            'based on speed (careful, on KITTI some frames have incorrect speed)')
    a('--with-gt', action='store_true',
      help='If available (e.g. with KITTI), will store ground truth along with images, for validation')
    a('--dump-root', type=str, required=True, help='Where to dump the data')
    a('--height', type=int, default=128, help='image height')
    a('--width', type=int, default=416, help='image width')
    a('--num-threads', type=int, default=4, help='number of host worker processes')
    a('--test-scenes', default=None, metavar='FILE',
      help="KITTI drives to leave out (the reference's data/test_scenes.txt); required with --dataset-format kitti")
    return p


def parse_args(argv):
    parser = build_parser()
    args = parser.parse_args(argv)
    if args.height <= 0 or args.width <= 0:
        parser.error('--height and --width must be positive, got %d x %d' % (args.height, args.width))
    if args.num_threads < 1:
        parser.error('--num-threads must be at least 1, got %d' % args.num_threads)
    if args.dataset_format == 'kitti' and args.test_scenes is None:
        parser.error("--test-scenes is required with --dataset-format kitti: the reference's data/test_scenes.txt "
                     'lists the drives to leave out')
    return args


def scene_sources(args):
    """(units, scenes_of): the drives (KITTI) or cities (Cityscapes) in the reference's order, found before any frame is
    read, and the function that gives a unit's scenes."""
    if args.dataset_format == 'kitti':
        static = read_static_frames(args.static_frames) if args.static_frames else None
        drives = kitti_drives(args.dataset_dir, read_test_scenes(args.test_scenes))
        return drives, lambda dr: kitti_scenes(dr, args.height, args.width, static, args.with_gt)
    return cityscapes_cities(args.dataset_dir), lambda c: cityscapes_scenes(c, args.dataset_dir, args.height, args.width)


def main(argv=None, device=None):
    """prepare_train_data.py main(): returns dict(dump_root, scenes=[folders kept], order, train, val).  Every worker
    process is joined before it returns or raises."""
    args = parse_args(sys.argv[1:] if argv is None else argv)
    if device is None:
        from . import _lib
        device = _lib.device()
    units, scenes_of = scene_sources(args)
    os.makedirs(args.dump_root, exist_ok=True)
    pool = multiprocessing.get_context('spawn').Pool(args.num_threads)
    try:
        kept = []
        for u in units:
            for s in scenes_of(u):
                d = write_scene(s, args.dump_root, args.height, args.width, device, pool)
                if d is not None:
                    kept.append(d)
        pool.close()
    except BaseException:
        pool.terminate()
        raise
    finally:
        pool.join()
    order, train, val = split(args.dump_root)
    print('{} scene folders written to {}: {} train, {} val'.format(len(kept), args.dump_root, len(train), len(val)))
    return dict(dump_root=args.dump_root, scenes=kept, order=order, train=train, val=val)


if __name__ == '__main__':
    main()
