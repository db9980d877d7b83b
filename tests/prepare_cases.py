"""Synthetic raw trees for the training-data preparation (cc_b200.prepare_train_data, oracle/prepare.py): a KITTI raw tree
and a Cityscapes tree of tiny frames whose bytes tests/golden/prepare_small.npz holds, the runs the fixture records, and
a KITTI-size tree for the GPU test and tools/bench_prepare.py.

Every run is made from a working directory holding raw/, static.txt and test_scenes.txt, with relative paths: the
Cityscapes loader takes a frame id from the whole camera-file path split on '_', so the path above the tree must not
hold one."""
import io
import json
import os
import numpy as np

DATES = ('2011_09_26', '2011_09_28', '2011_09_29', '2011_09_30', '2011_10_03')
EXCLUDED = '2011_09_26_drive_0117'                   # in the reference's data/test_scenes.txt
TEST_SCENES = (EXCLUDED + '\n').encode()
H, W = 16, 48                                        # the KITTI runs' output size
CS_H, CS_W = 24, 48                                  # the Cityscapes run's (cropped to 18 rows)

# (date, drive, frames, raw (h, w), cameras whose frame 0 exists, speed kind)
KITTI_DRIVES = [
    ('2011_09_26', '2011_09_26_drive_0001_sync', 9, (30, 100), ('02', '03'), 'mixed'),
    ('2011_09_26', '2011_09_26_drive_0003_sync', 4, (30, 100), ('02',), 'mixed'),        # camera 03's frame 0 missing
    ('2011_09_26', '2011_09_26_drive_0117_sync', 5, (30, 100), ('02', '03'), 'mixed'),   # a test scene
    ('2011_09_29', '2011_09_29_drive_0004_sync', 4, (36, 90), ('02', '03'), 'slow'),     # < 3 frames kept
    ('2011_09_30', '2011_09_30_drive_0005_sync', 8, (36, 90), ('02', '03'), 'mixed'),
]
# the last line has no newline: its frame id loses its last digit ('...031' -> 3), as in the reference
STATIC = ('2011_09_26 2011_09_26_drive_0001_sync 0000000002\n'
          '\n'
          '2011_09_26 2011_09_26_drive_0001_sync 0000000005\n'
          '2011_09_29 2011_09_29_drive_0004_sync 0000000000\n'
          '2011_09_29 2011_09_29_drive_0004_sync 0000000001\n'
          '2011_09_30 2011_09_30_drive_0005_sync 0000000031').encode()

CITY = 'aachen'
# scene id -> frame numbers (scene 000000 has a gap: two connected runs)
CS_SCENES = {'000000': list(range(0, 8)) + list(range(10, 18)), '000001': list(range(20, 30))}
# sqrt(3) * 1.3 > 2 keeps a frame alone, where a plain sum would need two; 0.7 needs a second frame
CS_SPEEDS = {'000000': [1.3, 1.3, 0.7, 1.3, 1.3, 1.3, 1.3, 0.7, 1.3, 1.3, 1.3, 1.3, 0.7, 1.3, 1.3, 1.3],
             '000001': [1.3, 0.7, 1.3, 1.3, 1.3, 0.7, 1.3, 1.3, 1.3, 1.3]}

RUNS = {
    'kitti_speed': ['raw', '--dataset-format', 'kitti', '--dump-root', 'dump', '--with-gt', '--height', str(H),
                    '--width', str(W), '--num-threads', '1', '--test-scenes', 'test_scenes.txt'],
    'kitti_static': ['raw', '--dataset-format', 'kitti', '--dump-root', 'dump', '--with-gt', '--height', str(H),
                     '--width', str(W), '--num-threads', '1', '--test-scenes', 'test_scenes.txt',
                     '--static-frames', 'static.txt'],
    'cityscapes': ['raw', '--dataset-format', 'cityscapes', '--dump-root', 'dump', '--height', str(CS_H),
                   '--width', str(CS_W), '--num-threads', '1'],
}
RUN_TREE = {'kitti_speed': 'kitti', 'kitti_static': 'kitti', 'cityscapes': 'cityscapes'}


def png(a):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(a).save(b, format='PNG')
    return b.getvalue()


def frame(rs, h, w):
    """A smooth uint8 RGB frame with a little noise (compresses well, every resampling tap matters)."""
    y, x = np.mgrid[0:h, 0:w]
    ph = rs.uniform(0, 6.28, 3)
    base = np.stack([127 + 100 * np.sin(x / (3 + c) + y / (5 + c) + ph[c]) for c in range(3)], -1)
    return np.clip(base + rs.randint(-8, 9, (h, w, 3)), 0, 255).astype(np.uint8)


def calib(date_index, raw_hw):
    """The calibration values of a date: P_rect_02 / P_rect_03 for raw_hw frames, R_rect_00, velodyne R and T."""
    rs = np.random.RandomState(100 + date_index)
    h, w = raw_hw
    f = 0.4 * w
    P2 = np.array([[f, 0, w / 2 + 0.37, 2.1], [0, f * 1.01, h / 2 - 0.21, 0.3], [0, 0, 1, 0.0027]])
    P3 = P2.copy()
    P3[0, 3] = -0.31 * f
    R = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], np.float64) + rs.randn(3, 3) * 0.01
    T = np.array([-0.004, -0.076, -0.27]) + rs.randn(3) * 0.01
    R_rect = np.eye(3) + rs.randn(3, 3) * 0.005
    return dict(P_rect_02=P2, P_rect_03=P3, R_rect_00=R_rect, R=R, T=T)


def calib_text(c):
    """calib_cam_to_cam.txt and calib_velo_to_cam.txt.  P_rect_02's numbers are separated by two spaces (value.split()
    reads them, value.split(' ') would not); the calib_time lines do not parse as numbers and are dropped."""
    fmt = lambda k, sep=' ': '%s: %s\n' % (k, sep.join(repr(float(v)) for v in np.ravel(c[k])))      # noqa: E731
    cam = ('calib_time: 09-Jan-2012 13:57:47\ncorner_dist: 9.950000e-02\n' + fmt('R_rect_00') + fmt('P_rect_02', '  ')
           + fmt('P_rect_03'))
    velo = 'calib_time: 15-Mar-2012 11:37:16\n' + fmt('R') + fmt('T') + 'delta_f: 0.000000e+00 0.000000e+00\n'
    return cam.encode(), velo.encode()


def velo_to_image(c, cam, zoom_x, zoom_y):
    """The scaled projection generate_depth_map builds (P_rect rows 0 and 1 scaled, then @ R_cam2rect @ velo2cam)."""
    P = np.array(c['P_rect_' + cam], np.float64)
    P[0] *= zoom_x
    P[1] *= zoom_y
    R4 = np.eye(4)
    R4[:3, :3] = c['R_rect_00']
    v2c = np.vstack((np.hstack((c['R'], c['T'][:, None])), [0, 0, 0, 1.0]))
    return np.dot(np.dot(P, R4), v2c)


def point_at(P, u, v, Z):
    """The velodyne point that P projects onto pixel (row v, column u) of generate_depth_map (round(.) - 1) at depth Z."""
    x = np.linalg.solve(P[:, :3], np.array([Z * (u + 1), Z * (v + 1), Z]) - P[:, 3])
    return [x[0], x[1], x[2], 0.5]


def sweep(rs, P, h, w, n):
    """n velodyne points around the car on a 1/256 m grid (a fifth behind it, some off the frame), then points made for
    the h x w frame of P: three on one pixel in both depth orders, and the sub2ind collision of (v, w-1) with (v+1, 0)
    in both point orders (the duplicate pass writes the key's minimum at its first point's pixel)."""
    pts = np.stack([rs.uniform(-15, 60, n), rs.uniform(-25, 25, n), rs.uniform(-2.5, 1.5, n), rs.rand(n)], 1)
    pts = list(np.round(pts * 256) / 256)
    for _ in range(2):
        u, v = rs.randint(0, w), rs.randint(0, h)
        for Z in rs.permutation([6.0, 9.5, 7.25]):
            pts.append(point_at(P, u, v, Z))
    v = rs.randint(0, h - 1)
    pts += [point_at(P, w - 1, v, 12.0), point_at(P, 0, v + 1, 8.0)]
    v = rs.randint(0, h - 1)
    pts += [point_at(P, 0, v + 1, 5.0), point_at(P, w - 1, v, 11.0)]
    return np.array(pts, np.float32)


def oxts_line(speed):
    vals = np.zeros(30)
    vals[:3] = [49.01, 8.43, 116.4]
    vals[8:11] = speed
    return (' '.join(repr(float(v)) for v in vals) + '\n').encode()


def speeds(rs, n, kind):
    if kind == 'slow':
        return [np.array([0.8, 0.0, 0.0])] * n
    return [np.array([rs.uniform(0.6, 2.3), rs.uniform(-0.4, 0.4), rs.uniform(-0.1, 0.1)]) for _ in range(n)]


def kitti_tree(put, seed=11, drives=KITTI_DRIVES, out_hw=(H, W), points=160):
    """A KITTI raw tree under raw/, each file handed to put(relative path, bytes) (None: an empty folder): every date
    folder (2011_09_28 and 2011_10_03 empty here), per date calib_cam_to_cam.txt / calib_velo_to_cam.txt, per drive
    oxts/data, image_02/data, image_03/data and velodyne_points/data; the sweeps are made for camera 02 at out_hw."""
    rs = np.random.RandomState(seed)
    for d in DATES:
        put('raw/%s/' % d, None)
    for date, drive, n, hw, cams, kind in drives:
        c = calib(DATES.index(date), hw)
        cam_txt, velo_txt = calib_text(c)
        put('raw/%s/calib_cam_to_cam.txt' % date, cam_txt)
        put('raw/%s/calib_velo_to_cam.txt' % date, velo_txt)
        base = 'raw/%s/%s/' % (date, drive)
        for i, s in enumerate(speeds(rs, n, kind)):
            put(base + 'oxts/data/%010d.txt' % i, oxts_line(s))
        P = velo_to_image(c, '02', out_hw[1] / hw[1], out_hw[0] / hw[0])
        for i in range(n):
            for cam in ('02', '03'):
                if i > 0 or cam in cams:
                    put(base + 'image_%s/data/%010d.png' % (cam, i), png(frame(rs, *hw)))
            put(base + 'velodyne_points/data/%010d.bin' % i, sweep(rs, P, out_hw[0], out_hw[1], points).tobytes())


def kitti_tree_files(**kw):
    """{relative path: bytes} of kitti_tree(**kw)."""
    files = {}
    kitti_tree(files.__setitem__, **kw)
    return files


def write_kitti_tree(root, **kw):
    """kitti_tree(**kw) written under root, file by file; returns root."""
    kitti_tree(lambda rel, b: write_files(root, {rel: b}), **kw)
    return root


def cityscapes_tree_files(seed=12, raw_hw=(32, 64)):
    """{relative path: bytes} of a Cityscapes tree under raw/: leftImg8bit_sequence/train/<city> frames, one camera json
    per scene (on a frame of the scene's second run where it has one), vehicle_sequence speeds."""
    rs = np.random.RandomState(seed)
    files = {}
    for scene, ids in CS_SCENES.items():
        for fid, sp in zip(ids, CS_SPEEDS[scene]):
            name = '%s_%s_%06d' % (CITY, scene, fid)
            files['raw/leftImg8bit_sequence/train/%s/%s_leftImg8bit.png' % (CITY, name)] = png(frame(rs, *raw_hw))
            files['raw/vehicle_sequence/train/%s/%s_vehicle.json' % (CITY, name)] = json.dumps(
                {'speed': sp, 'yawRate': 0.01}).encode()
        cam = dict(intrinsic=dict(fx=2262.52 * raw_hw[1] / 2048, fy=2265.30 * raw_hw[0] / 1024,
                                  u0=1096.98 * raw_hw[1] / 2048, v0=513.137 * raw_hw[0] / 1024))
        files['raw/camera/train/%s/%s_%s_%06d_camera.json' % (CITY, CITY, scene, ids[-3])] = json.dumps(cam).encode()
    return files


def tree_files(kind):
    return kitti_tree_files() if kind == 'kitti' else cityscapes_tree_files()


def write_files(root, files):
    """Write {relative path: bytes} under root (a None value is an empty folder); returns root."""
    for rel, b in files.items():
        p = os.path.join(root, rel)
        if b is None:
            os.makedirs(p, exist_ok=True)
            continue
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, 'wb') as f:
            f.write(b)
    return root


def write_run_dir(root, tree):
    """root/raw (the tree's files), root/static.txt and root/test_scenes.txt; returns root."""
    write_files(root, tree)
    write_files(root, {'static.txt': STATIC, 'test_scenes.txt': TEST_SCENES})
    return root


def tree_from_fixture(g, kind):
    names = g[kind + '_tree_names']
    return {str(n): (None if str(n).endswith('/') else g['%s_tree_%d' % (kind, i)].tobytes()) for i, n in enumerate(names)}


def dump_files(dump):
    """Sorted relative paths of every file under dump."""
    out = []
    for d, _, fs in os.walk(dump):
        out += [os.path.relpath(os.path.join(d, f), dump) for f in fs]
    return sorted(out)


def kitti_size_drives(frames=6, sizes=((375, 1242), (376, 1241))):
    """Two drives of KITTI's two frame sizes on two dates."""
    return [('2011_09_26', '2011_09_26_drive_0001_sync', frames, sizes[0], ('02', '03'), 'mixed'),
            ('2011_09_30', '2011_09_30_drive_0020_sync', frames, sizes[1], ('02', '03'), 'mixed')]
