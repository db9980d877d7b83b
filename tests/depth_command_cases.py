"""Cases of the depth-evaluation command (cc_b200.test_disp over evaluate.kitti_depth_framework /
stillbox_depth_framework, depth_eval_batch, velodyne_depth and colorize's 'hot'), run on the CPU simulator build
(tests/test_depth_command.py) and on the H100 (tests/test_gpu_depth_command.py).

The references are tests/golden/test_disp_small.npz (the reference's own test_disp.main() on the trees written here,
tests/golden/make_test_disp.py) and the oracle restatement (oracle/eval_disp.py).  The trees:
  KITTI     two dates of different frame sizes (40x130 and 41x129, calibrations scaled to them); drive 0001 has cameras 02
            and 03, drive 0003 a frame whose oxts speed is zero (every displacement 0: 'not good !').  The list holds a
            target at each edge of a drive (missing reference frames become the target with shift 0), a missing target,
            and sweeps of 2500 points on ~5000 pixels (many pixels hit twice).
  Stillbox  two folders of different frame sizes, .npy depths of 30x30 float32 with zeros and values past --max-depth;
            the list holds the first and last frame of a scene (references clamped into it) and a missing file."""
import io
import json
import os
import re
import time
import numpy as np
import torch
from cc_b200 import evaluate as CE, models as CM, synth, test_disp as TD
from oracle import eval_disp as OT, nets as ON
from tests.depth_eval_cases import kitti_calib, kitti_sweep
from tests.run_inference_cases import check_image, disp_tolerance, photo
from tests.util import golden

FIXTURE = 'test_disp_small'
SIZE = (64, 128)
DISP_SEED, POSE_SEED = 5, 6
KITTI_DATES = {'2011_09_26': (40, 130), '2011_09_30': (41, 129)}
KITTI_DRIVES = {('2011_09_26', '2011_09_26_drive_0001_sync'): (6, ('image_02', 'image_03')),
                ('2011_09_30', '2011_09_30_drive_0003_sync'): (4, ('image_02',))}
ZERO_SPEED = ('2011_09_30_drive_0003_sync', 2)
KITTI_LIST = ['2011_09_26/2011_09_26_drive_0001_sync/image_02/data/0000000002.png',
              '2011_09_26/2011_09_26_drive_0001_sync/image_02/data/0000000000.png',
              '2011_09_26/2011_09_26_drive_0001_sync/image_02/data/0000000009.png',
              '2011_09_30/2011_09_30_drive_0003_sync/image_02/data/0000000002.png',
              '2011_09_26/2011_09_26_drive_0001_sync/image_03/data/0000000005.png',
              '2011_09_30/2011_09_30_drive_0003_sync/image_02/data/0000000001.png']
STILLBOX_FOLDERS = {'a': ((48, 80), [5, 4]), 'b': ((50, 84), [3])}     # frame size, scene lengths
STILLBOX_LIST = ['a/RGB_0000_00.jpg', 'a/RGB_0000_02.jpg', 'b/RGB_0000_01.jpg', 'a/RGB_0001_07.jpg', 'a/RGB_0001_03.jpg']
_common = ['--pretrained-dispnet', 'disp.pth.tar', '--img-height', '64', '--img-width', '128']
RUNS = {
    'kitti_pose_out': _common + ['--pretrained-posenet', 'pose5.pth.tar', '--dataset-dir', 'kitti', '--dataset-list',
                                 'kitti.txt', '--output-dir', 'out'],
    'kitti_sn': _common + ['--spatial-normalize', '--dataset-dir', 'kitti', '--dataset-list', 'kitti.txt'],
    'kitti_noresize_pose': _common + ['--no-resize', '--pretrained-posenet', 'pose5.pth.tar', '--dataset-dir', 'kitti',
                                      '--dataset-list', 'kitti.txt'],
    'stillbox_pose_out': _common + ['--gt-type', 'stillbox', '--pretrained-posenet', 'pose3.pth.tar', '--dataset-dir',
                                    'stillbox', '--dataset-list', 'stillbox.txt', '--output-dir', 'out',
                                    '--max-depth', '60'],
    'stillbox_sn': _common + ['--gt-type', 'stillbox', '--spatial-normalize', '--dataset-dir', 'stillbox',
                              '--dataset-list', 'stillbox.txt'],
}


def g():
    return golden(FIXTURE)


# ---- trees ------------------------------------------------------------------------------------------------------------
def checkpoints():
    """{'disp.pth.tar': DispResNet6, 'pose5.pth.tar': PoseExpNet of 4 references, 'pose3.pth.tar': of 2}."""
    pose = lambda nb: synth.seeded_fill(CM.PoseExpNet(nb_ref_imgs=nb), POSE_SEED + nb).state_dict()   # noqa: E731
    return {'disp.pth.tar': {'state_dict': ON.disp_params(DISP_SEED)}, 'pose5.pth.tar': {'state_dict': pose(4)},
            'pose3.pth.tar': {'state_dict': pose(2)}}


def _write_calib(calib_dir, c):
    os.makedirs(calib_dir, exist_ok=True)
    line = lambda k: '%s: %s\n' % (k, ' '.join(repr(float(v)) for v in c[k]))      # noqa: E731
    with open(os.path.join(calib_dir, 'calib_cam_to_cam.txt'), 'w') as f:
        f.write('calib_time: 09-Jan-2012 13:57:47\n' + line('R_rect_00') + line('P_rect_02') + line('P_rect_03'))
    with open(os.path.join(calib_dir, 'calib_velo_to_cam.txt'), 'w') as f:
        f.write('calib_time: 15-Mar-2012 11:37:16\n' + line('R') + line('T'))


def write_kitti_tree(root, n_points=2500, sizes=KITTI_DATES, drives=KITTI_DRIVES, seed=1):
    from PIL import Image
    rs = np.random.RandomState(seed)
    for date, (H, W) in sizes.items():
        c = kitti_calib(rs)
        scale = np.array([[W / 1242.0], [H / 375.0], [1.0]])
        P2 = c['P_rect_02'].reshape(3, 4) * scale
        P3 = P2.copy()
        P3[0, 3] -= 0.54 * P3[0, 0]
        c['P_rect_02'], c['P_rect_03'] = P2.ravel(), P3.ravel()
        _write_calib(os.path.join(root, date), c)
    for k, ((date, drive), (n, cams)) in enumerate(sorted(drives.items())):
        H, W = sizes[date]
        base = os.path.join(root, date, drive)
        for cam in cams:
            os.makedirs(os.path.join(base, cam, 'data'), exist_ok=True)
            for i in range(n):
                Image.fromarray(photo(H, W, 10 * k + i + (cam == 'image_03'))).save(
                    os.path.join(base, cam, 'data', '%010d.png' % i))
        os.makedirs(os.path.join(base, 'oxts', 'data'), exist_ok=True)
        os.makedirs(os.path.join(base, 'velodyne_points', 'data'), exist_ok=True)
        t = 1317380000.0 + 0.1 * k + np.cumsum(rs.uniform(0.09, 0.11, n))
        with open(os.path.join(base, 'oxts', 'timestamps.txt'), 'w') as f:
            for v in t:
                sec = int(np.floor(v))
                f.write('%s.%09d\n' % (time.strftime('%Y-%m-%d %H:%M:%S', time.gmtime(sec)), int((v - sec) * 1e9)))
        for i in range(n):
            oxts = rs.randn(30)
            oxts[8:11] = [rs.uniform(5, 15), rs.randn() * 0.3, rs.randn() * 0.1]
            if (drive, i) == ZERO_SPEED:
                oxts[8:11] = 0.0
            np.savetxt(os.path.join(base, 'oxts', 'data', '%010d.txt' % i), oxts[None], fmt='%.10g', delimiter=' ')
            kitti_sweep(rs, n_points).tofile(os.path.join(base, 'velodyne_points', 'data', '%010d.bin' % i))


def write_stillbox_tree(root, folders=STILLBOX_FOLDERS, seed=2):
    from PIL import Image
    rs = np.random.RandomState(seed)
    for k, (folder, ((H, W), lengths)) in enumerate(sorted(folders.items())):
        d = os.path.join(root, folder)
        os.makedirs(d, exist_ok=True)
        scenes = []
        for s, n in enumerate(lengths):
            imgs = ['RGB_%04d_%02d.jpg' % (s, i) for i in range(n)]
            depths = ['depth_%04d_%02d.npy' % (s, i) for i in range(n)]
            for i in range(n):
                Image.fromarray(photo(H, W, 40 + 10 * k + 3 * s + i)).save(os.path.join(d, imgs[i]))
                gt = rs.uniform(1.0, 90.0, (30, 30)).astype(np.float32)
                gt[rs.rand(30, 30) < 0.1] = 0
                np.save(os.path.join(d, depths[i]), gt)
            scenes.append(dict(length=n, imgs=imgs, depth=depths, time_step=0.1 + 0.05 * s,
                               speed=[float(v) for v in rs.uniform(-4, 4, 3)]))
        with open(os.path.join(d, 'metadata.json'), 'w') as f:
            json.dump(dict(scenes=scenes), f)


def write_work_dir(root):
    """root/kitti, root/stillbox, their lists and the checkpoints."""
    write_kitti_tree(os.path.join(root, 'kitti'))
    write_stillbox_tree(os.path.join(root, 'stillbox'))
    for name, lines in (('kitti.txt', KITTI_LIST), ('stillbox.txt', STILLBOX_LIST)):
        with open(os.path.join(root, name), 'w') as f:
            f.write('\n'.join(lines) + '\n')
    for name, ck in checkpoints().items():
        torch.save(ck, os.path.join(root, name))


def opt(argv, flag, default=None):
    return argv[argv.index(flag) + 1] if flag in argv else default


def oracle_run(root, run, dtype=torch.float32):
    """oracle.eval_disp.run on the work folder for RUNS[run] (paths as the command sees them from root)."""
    argv = RUNS[run]
    ck = checkpoints()
    cast = lambda sd: {k: v.to(dtype) if v.is_floating_point() else v for k, v in sd.items()}   # noqa: E731
    pose = opt(argv, '--pretrained-posenet')
    gt_type = opt(argv, '--gt-type', 'KITTI')
    cwd = os.getcwd()
    os.chdir(root)
    try:
        with open(opt(argv, '--dataset-list')) as f:
            files = f.read().splitlines()
        return OT.run(gt_type, files, opt(argv, '--dataset-dir'), cast(ck['disp.pth.tar']['state_dict']),
                      cast(ck[pose]['state_dict']) if pose else None, *SIZE, no_resize='--no-resize' in argv,
                      spatial_normalize='--spatial-normalize' in argv, max_depth=float(opt(argv, '--max-depth', 80)),
                      output='--output-dir' in argv)
    finally:
        os.chdir(cwd)


# ---- comparisons --------------------------------------------------------------------------------------------------------
_NUM = re.compile(r'-?(?:\d+\.\d+|inf|nan)')


def check_stdout(got, want, rtol=2e-3, atol=2e-4):
    """The same lines; the numbers of the result rows within the conv engine's tolerance (the words exactly)."""
    gl, wl = got.splitlines(), want.splitlines()
    assert len(gl) == len(wl), (got, want)
    for a, b in zip(gl, wl):
        if a == b:
            continue
        assert _NUM.sub('#', a) == _NUM.sub('#', b), (a, b)
        x, y = np.array([float(v) for v in _NUM.findall(a)]), np.array([float(v) for v in _NUM.findall(b)])
        assert np.array_equal(np.isfinite(x), np.isfinite(y)) and np.allclose(x, y, rtol=rtol, atol=atol,
                                                                              equal_nan=True), (a, b)


def check_errors(got, want, name, rtol=2e-3, atol=2e-4):
    """Per-sample errors [2,7,N] within the bound tests/depth_eval_cases.case_eval_batch holds depth_eval_batch to against
    the oracle nets, inf and NaN where the reference has them."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (name, got.shape, want.shape)
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(np.isinf(got), np.isinf(want)), (name, got, want)
    f = np.isfinite(want)
    assert np.allclose(got[f], want[f], rtol=rtol, atol=atol), (name, np.abs(got[f] - want[f]).max())


def check_images(images, want_images, predictions, run):
    """Every PNG equals the reference's, or is one bin apart at a bin edge within the conv tolerance (depth.png on the
    disparity 1/prediction; img.png exactly; gt.png exactly: its input does not depend on the nets)."""
    assert sorted(images) == sorted(want_images), (run, sorted(images), sorted(want_images))
    for name, want in want_images.items():
        got = images[name]
        assert got.shape == want.shape and got.dtype == np.uint8, (run, name, got.shape, want.shape)
        if name.endswith('depth.png'):
            disp = (1 / predictions[int(name[:4])]).astype(np.float32)
            check_image(got, want, disp, 'hot', None, False, 2 * disp_tolerance(disp), '%s %s' % (run, name))
        else:
            assert np.array_equal(got, want), (run, name, int((got != want).any(-1).sum()))


def fixture_images(d, run):
    names = [str(n) for n in d[run + '_image_names']] if run + '_image_names' in d else []
    return {n: d['%s_image_%d' % (run, k)] for k, n in enumerate(names)}


# ---- cases ------------------------------------------------------------------------------------------------------------
def case_hot_table(device=None):
    """The product's 'hot' table equals the oracle's and the one the fixture's stand-in made."""
    got = CE.colormap_table('hot')
    assert got.shape == (256, 3) and np.array_equal(got, OT.hot_table())
    assert np.array_equal(got, g()['table_hot'])


def run_main(tmp, run, device, workers=2, capsys=None, argv=None):
    """main() on a fresh copy of the work folder with RUNS[run] -> (result, stdout, work folder)."""
    write_work_dir(str(tmp))
    cwd = os.getcwd()
    os.chdir(str(tmp))
    try:
        res = TD.main(argv or RUNS[run], device=device, workers=workers)
    finally:
        os.chdir(cwd)
    out = capsys.readouterr().out if capsys is not None else None
    return res, out, str(tmp)


def read_outputs(root):
    """predictions.npy and the viz PNGs under root/out (None, {} without them)."""
    from PIL import Image
    out = os.path.join(root, 'out')
    if not os.path.isdir(out):
        return None, {}
    pred = np.load(os.path.join(out, 'predictions.npy'))
    viz = os.path.join(out, 'viz')
    return pred, {n: np.asarray(Image.open(os.path.join(viz, n))) for n in os.listdir(viz)}


def case_main(device, tmp, capsys, run, workers=2):
    """main() against the fixture: stdout, per-sample errors, predictions.npy and every PNG."""
    d = g()
    res, out, root = run_main(tmp, run, device, workers, capsys)
    check_stdout(out, str(d[run + '_stdout']))
    check_errors(res['errors'].transpose(1, 2, 0), d[run + '_errors'], run)
    pred, images = read_outputs(root)
    if '--output-dir' in RUNS[run]:
        want = d[run + '_predictions']
        assert pred.dtype == np.float64 and pred.shape == want.shape, (pred.shape, want.shape)
        assert np.allclose(pred, want, rtol=2e-3, atol=0), np.abs(pred - want).max()
        check_images(images, fixture_images(d, run), want, run)
    else:
        assert pred is None and not images
    return res, out, pred, images


def case_workers_identical(device, tmp, run='kitti_pose_out'):
    """One and three workers write the same stdout, errors, predictions and PNGs, bit for bit."""
    outs = []
    for w, sub in ((1, 'w1'), (3, 'w3')):
        os.makedirs(os.path.join(str(tmp), sub))
        buf = io.StringIO()
        import contextlib
        with contextlib.redirect_stdout(buf):
            res, _, root = run_main(os.path.join(str(tmp), sub), run, device, workers=w)
        outs.append((buf.getvalue(), res['errors'], *read_outputs(root)))
    (s1, e1, p1, i1), (s3, e3, p3, i3) = outs
    assert s1 == s3 and np.array_equal(e1, e3) and np.array_equal(p1, p3)
    assert sorted(i1) == sorted(i3) and all(np.array_equal(i1[n], i3[n]) for n in i1)


# ---- KITTI size -----------------------------------------------------------------------------------------------------------
KITTI_SIZE_DATES = {'2011_09_26': (375, 1242), '2011_09_30': (376, 1241)}
KITTI_SIZE_DRIVES = {('2011_09_26', '2011_09_26_drive_0001_sync'): (3, ('image_02',)),
                     ('2011_09_30', '2011_09_30_drive_0003_sync'): (3, ('image_02',))}
KITTI_SIZE_LIST = ['2011_09_26/2011_09_26_drive_0001_sync/image_02/data/0000000001.png',
                   '2011_09_26/2011_09_26_drive_0001_sync/image_02/data/0000000000.png',
                   '2011_09_30/2011_09_30_drive_0003_sync/image_02/data/0000000001.png']


def pose_checkpoint(name, nb=4, seed=31):
    from cc_b200 import models as M
    if name == 'PoseNetB6':
        return {'state_dict': ON.pose_params(nb, seed)}
    return {'state_dict': synth.seeded_fill(getattr(M, name)(nb_ref_imgs=nb), seed).state_dict()}


def kitti_size_case(device, tmp, posenet=None, n_points=100000):
    """1242x375 and 1241x376 frames with 100k-point sweeps (frame 0 has no reference frame before it) through main() at
    256x832: the per-sample errors within depth_eval_batch's bound against oracle.eval_disp on fp64 oracle nets
    (DispResNet6, and the pose net `posenet` at seq 5), and a second run gives the same bits."""
    root = str(tmp)
    write_kitti_tree(os.path.join(root, 'kitti'), n_points, KITTI_SIZE_DATES, KITTI_SIZE_DRIVES, seed=7)
    with open(os.path.join(root, 'list.txt'), 'w') as f:
        f.write('\n'.join(KITTI_SIZE_LIST) + '\n')
    disp = {'state_dict': ON.disp_params(DISP_SEED)}
    torch.save(disp, os.path.join(root, 'disp.pth.tar'))
    argv = ['--pretrained-dispnet', 'disp.pth.tar', '--dataset-dir', 'kitti', '--dataset-list', 'list.txt']
    pose = None
    if posenet is not None:
        pose = pose_checkpoint(posenet)
        torch.save(pose, os.path.join(root, 'pose.pth.tar'))
        argv += ['--pretrained-posenet', 'pose.pth.tar', '--posenet', posenet]
    cwd = os.getcwd()
    os.chdir(root)
    try:
        import contextlib
        with contextlib.redirect_stdout(io.StringIO()):
            first = TD.main(argv, device=device)['errors']
            again = TD.main(argv, device=device)['errors']
        d64 = lambda sd: {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}     # noqa: E731
        want = OT.run('KITTI', KITTI_SIZE_LIST, 'kitti', d64(disp['state_dict']),
                      d64(pose['state_dict']) if pose else None)['errors']
    finally:
        os.chdir(cwd)
    assert np.array_equal(first, again)
    check_errors(first.transpose(1, 2, 0), want, 'kitti size %s' % posenet)
    assert bool(first[:, 0].any()) == (posenet is not None)
    return first
