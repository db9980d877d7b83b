"""Cases of the depth evaluation on the device (cc_b200.evaluate.velodyne_depth / spline_zoom / depth_errors /
depth_eval_batch over ccb_velo_depth, ccb_spline_zoom and ccb_eigen_depth_errors), run on the CPU simulator build
(tests/test_depth_eval.py) and on the H100 (tests/test_gpu_depth_eval.py).

The references are tests/golden/depth_eval_small.npz (the reference's own generate_depth_map, both generate_masks and
test_disp.compute_errors, tests/golden/make_depth_eval.py), the oracle restatement (oracle/depth_eval.py) and scipy's zoom
itself.  The builders of the fixture's inputs live here so that the fixture maker and the tests write the same files."""
import os
import numpy as np
import torch
from scipy.ndimage import zoom
from cc_b200 import _lib, evaluate as CE, models as CM
from oracle import depth_eval as OD, nets as ON
from tests.util import golden

FIXTURE = 'depth_eval_small'
KITTI = (256, 832, 375, 1242)
ZOOM_SIZES = [(8, 26, 13, 39), (1, 26, 1, 39), (2, 26, 5, 39), (8, 1, 13, 3), (8, 2, 13, 2), (13, 39, 13, 39), (3, 4, 1, 1)]


# ---- inputs --------------------------------------------------------------------------------------

def kitti_calib(rs):
    """calib_cam_to_cam / calib_velo_to_cam values like KITTI's (cam 2), slightly perturbed."""
    R = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], np.float64) + rs.randn(3, 3) * 0.01
    T = np.array([-0.004, -0.076, -0.27]) + rs.randn(3) * 0.01
    R_rect = np.eye(3) + rs.randn(3, 3) * 0.005
    P_rect = np.array([[721.5377, 0, 609.5593, 44.85728], [0, 721.5377, 172.854, 0.2163791], [0, 0, 1, 0.002745884]])
    return dict(R=R.ravel(), T=T, R_rect_00=R_rect.ravel(), P_rect_02=P_rect.ravel())


def exact_calib():
    """A projection with exact arithmetic: X = y, Y = z, Z = x - 5 (identity rotation, rectification and translation)."""
    return dict(R=np.array([0, 1, 0, 0, 0, 1, 1, 0, 0], np.float64), T=np.zeros(3), R_rect_00=np.eye(3).ravel(),
                P_rect_02=np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, -5], np.float64))


def write_calib(calib_dir, c):
    """The two KITTI calibration files of the values `c` (repr round-trips every fp64)."""
    os.makedirs(calib_dir, exist_ok=True)
    line = lambda k: '%s: %s\n' % (k, ' '.join(repr(float(v)) for v in c[k]))      # noqa: E731
    with open(os.path.join(calib_dir, 'calib_cam_to_cam.txt'), 'w') as f:
        f.write('calib_time: 09-Jan-2012 13:57:47\n' + line('R_rect_00') + line('P_rect_02'))
    with open(os.path.join(calib_dir, 'calib_velo_to_cam.txt'), 'w') as f:
        f.write('calib_time: 15-Mar-2012 11:37:16\n' + line('R') + line('T'))


def kitti_sweep(rs, n):
    """n velodyne points around a car (x forward, y left, z up), a fifth of them behind it, on a 1/256 m grid (the sensor
    resolves about 2 cm; the grid keeps the fixture small)."""
    pts = np.stack([rs.uniform(-15, 60, n), rs.uniform(-25, 25, n), rs.uniform(-2.5, 1.5, n), rs.rand(n)], 1)
    return (np.round(pts * 256) / 256).astype(np.float32)


def quirk_sweep(W):
    """Points for exact_calib() in a 6 x W frame (Z = x - 5, u = round(y / Z) - 1, v = round(z / Z) - 1): several points
    on one pixel in both depth orders, the sub2ind collision of (v, W-1) with (v+1, 0) in both point orders, x < 0,
    off-frame points, negative Z in the frame, Z = 0 and Z ~ 1e-7, and .5 ties in u and v."""
    P = []
    add = lambda x, y, z: P.append((x, y, z, 0.3))      # noqa: E731
    add(6, 3, 2); add(7, 6, 4); add(6.5, 4.5, 3)          # (v, u) = (1, 2) three times, Z = 1, 2, 1.5
    add(8, 12, 9); add(6, 4, 3)                           # (2, 3): Z = 3, then 1 (last write = min)
    add(6, W, 1); add(6, 1, 2)                            # (0, W-1) then (1, 0): one key
    add(7, 2, 8); add(6, W, 3)                            # (3, 0) then (2, W-1): one key, the other order
    add(6.5, 1.5 * W, 1.5)                                # (0, W-1) again: a third point of the first key
    add(-1, -6, -6); add(-0.5, 3, 2)                      # x < 0: dropped before the projection
    add(6, W + 1, 2); add(6, 0, 2); add(6, 3, 7); add(6, 3, 0.4)      # u = W, u = -1, v = 6, v = -1: off the frame
    add(4, -3, -3); add(3, -4, -6)                        # Z = -1, -2 in the frame: (2, 2), (2, 1); depth < 0 -> 0
    add(4.5, -2, -1.5)                                    # Z = -0.5 on (2, 3) after positive points: the group min is < 0
    add(5, 1, 1); add(5, 0, 0)                            # Z = 0: inf and nan
    add(np.nextafter(np.float32(5), np.float32(6)), 1e-7, 1e-7)        # Z ~ 4.8e-7: u ~ 0.2 -> -1
    add(6, 2.5, 4.5); add(6, 3.5, 3.5)                    # ties: (3, 1), (3, 3) half to even
    add(6, 1.5, 0.5); add(6, 4.5, 5.5)                    # ties: (-1, 1) -> off, (5, 3)
    return np.array(P, np.float32)


def sparse(depth):
    idx = np.flatnonzero(depth)
    return idx.astype(np.int32), depth.ravel()[idx]


def dense(idx, val, shape):
    d = np.zeros(int(np.prod(shape)))
    d[idx] = val
    return d.reshape(shape)


def error_inputs(rs, H, W, fill=0.3, lo=1e-3, hi=80.0, n_exact=6):
    """(gt fp64 [H,W] sparse with values in (0, 90) and some exactly lo and hi, pred fp32 [H,W] in [lo, hi] near gt)."""
    gt = np.where(rs.rand(H, W) < fill, rs.uniform(0.5, 90, (H, W)), 0.0)
    ys, xs = rs.randint(H // 2, H, n_exact), rs.randint(0, W, n_exact)
    gt[ys[:n_exact // 2], xs[:n_exact // 2]] = lo
    gt[ys[n_exact // 2:], xs[n_exact // 2:]] = hi
    pred = np.clip(np.where(gt > 0, gt, 20.0) * rs.uniform(0.6, 1.6, (H, W)) * 0.37, lo, hi).astype(np.float32)
    return gt, pred


# ---- fixture --------------------------------------------------------------------------------------

def velo_cases():
    g = golden(FIXTURE)
    return [(str(c), g[c + '_points'], {k: g[c + '_calib_' + k] for k in ('R', 'T', 'R_rect_00', 'P_rect_02')},
             tuple(int(v) for v in g[c + '_shape']), dense(g[c + '_idx'], g[c + '_val'], tuple(g[c + '_shape'])))
            for c in g['velo_cases']]


def error_cases():
    g = golden(FIXTURE)
    out = []
    for c in g['error_cases']:
        shape = tuple(int(v) for v in g[c + '_shape'])
        poses = g[c + '_poses'] if c + '_poses' in g else None
        out.append(dict(name=str(c), gt=dense(g[c + '_gt_idx'], g[c + '_gt_val'], shape), pred=g[c + '_pred'],
                        crop=str(g[c + '_crop']), lo=float(g[c + '_lo']), hi=float(g[c + '_hi']),
                        mask=np.unpackbits(g[c + '_mask'])[:shape[0] * shape[1]].reshape(shape).astype(bool), poses=poses,
                        displacements=g[c + '_displacements'] if poses is not None else None, out=g[c + '_out']))
    return out


def crop_fractions(name):
    return {'eigen': OD.EIGEN, 'stillbox': OD.STILLBOX}[name]


# ---- cases ------------------------------------------------------------------------------------

def ulp_diff(a, b):
    """Largest distance in fp64 ulps between equal-shaped arrays of non-negative values."""
    return int(np.abs(np.asarray(a, np.float64).view(np.int64) - np.asarray(b, np.float64).view(np.int64)).max())


def run_velo(device, sweeps, Ps, H, W):
    pts = torch.from_numpy(np.concatenate(sweeps)).to(device)
    offs = torch.tensor(np.cumsum([0] + [len(s) for s in sweeps]), dtype=torch.int64, device=device)
    P = torch.from_numpy(np.stack(Ps)).to(device)
    return CE.velodyne_depth(pts, offs, P, H, W).cpu().numpy()


def case_velo_fixture(device, tmp_path, kitti=False):
    """velodyne_depth on the fixture's sweeps, the projection from kitti_velo_to_image on calibration files written from the
    fixture's values: the same pixels, the same zeros, values within one fp64 ulp (identical here: the kernel sums each
    row of the projection as the dgemm the fixture came from)."""
    seen = 0
    for name, points, calib, shape, want in velo_cases():
        if (shape[0] * shape[1] > 100000) != kitti:
            continue
        write_calib(str(tmp_path / name), calib)
        P = CE.kitti_velo_to_image(str(tmp_path / name), 2)
        got = run_velo(device, [points], [P], *shape)[0]
        assert np.array_equal(got != 0, want != 0), (name, int(((got != 0) != (want != 0)).sum()))
        assert ulp_diff(got, want) <= 1, name
        seen += 1
    assert seen >= 1


def case_velo_vs_oracle(device, B=2, H=40, W=130, n=6000, seed=3, reruns=0):
    """Random sweeps of different lengths in one batch against oracle.generate_depth_map per sample."""
    rs = np.random.RandomState(seed)
    sweeps = [kitti_sweep(rs, n + 777 * b) for b in range(B)]
    calib = kitti_calib(rs)
    P = OD_projection(calib)
    # a small frame: scale the intrinsics down so that the sweep covers it
    P = P * np.array([[W / 1242.0], [H / 375.0], [1.0]])
    got = run_velo(device, sweeps, [P] * B, H, W)
    for b in range(B):
        want = OD.generate_depth_map(sweeps[b], P, (H, W))
        assert np.array_equal(got[b] != 0, want != 0) and ulp_diff(got[b], want) <= 1, b
        assert (want > 0).mean() > 0.05
    for _ in range(reruns):
        assert np.array_equal(run_velo(device, sweeps, [P] * B, H, W), got)
    return got


def OD_projection(calib):
    """P_rect @ R_cam2rect @ velo2cam of calibration values, as kitti_velo_to_image builds it."""
    velo2cam = np.vstack((np.hstack((calib['R'].reshape(3, 3), calib['T'][:, None])), [0, 0, 0, 1.0]))
    R_cam2rect = np.eye(4)
    R_cam2rect[:3, :3] = calib['R_rect_00'].reshape(3, 3)
    return np.dot(np.dot(calib['P_rect_02'].reshape(3, 4), R_cam2rect), velo2cam)


def case_velo_batch_is_per_sample(device):
    """Three samples, one of them empty: the batch equals each sample run alone, bit for bit."""
    rs = np.random.RandomState(8)
    sweeps = [kitti_sweep(rs, 3000), kitti_sweep(rs, 0), quirk_sweep(9)]
    P = OD_projection(kitti_calib(rs)) * np.array([[40 / 1242.0], [6 / 375.0], [1.0]])
    Ps = [P, P, OD_projection(exact_calib())]
    got = run_velo(device, sweeps, Ps, 6, 9)
    for b in range(3):
        alone = run_velo(device, [sweeps[b]], [Ps[b]], 6, 9)[0]
        assert np.array_equal(got[b], alone), b
        assert np.array_equal(got[b], OD.generate_depth_map(sweeps[b], Ps[b], (6, 9))), b
    assert not got[1].any() and got[0].any()


def case_zoom_vs_scipy(device, sizes, N=2, seed=4):
    """spline_zoom within one fp32 ulp of scipy.ndimage.zoom(order=3), then the clip."""
    h, w, H, W = sizes
    rs = np.random.RandomState(seed)
    x = (1.0 / (rs.rand(N, h, w) * 0.3 + 0.01)).astype(np.float32)
    lo, hi = 1e-3, 60.0
    got = CE.spline_zoom(torch.from_numpy(x).to(device), H, W, lo, hi).cpu().numpy()
    want = np.stack([zoom(x[i], (H / h, W / w)).clip(lo, hi) for i in range(N)])
    assert got.shape == want.shape == (N, H, W)
    ulps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64)).max()
    assert ulps <= 1, (sizes, ulps)
    assert (want == np.float32(hi)).any() or H * W < 50


def run_errors(device, gt, pred, crop, lo, hi, poses=None, displacements=None):
    d = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(device)     # noqa: E731
    return CE.depth_errors(d(gt), d(pred), lo, hi, crop, d(poses), d(displacements)).cpu().numpy()


def check_errors(got, want, name=''):
    """a1..a3 exactly (they are counts over n), the rest within 1e-12 relative (inf and nan where the oracle has them)."""
    got, want = np.asarray(got), np.asarray(want)
    assert np.array_equal(got[..., 4:], want[..., 4:]), (name, got, want)
    assert np.array_equal(np.isfinite(got), np.isfinite(want)), (name, got, want)
    f = np.isfinite(want)
    assert np.all(np.abs(got[f] - want[f]) <= 1e-12 * np.abs(want[f])), (name, got, want)


def case_errors_fixture(device):
    """depth_errors on the fixture's samples against the numbers of the reference's compute_errors, both rows, both crops."""
    cases = error_cases()
    for c in cases:
        got = run_errors(device, c['gt'][None], c['pred'][None], c['crop'], c['lo'], c['hi'],
                         None if c['poses'] is None else c['poses'][None],
                         None if c['poses'] is None else c['displacements'][None])
        check_errors(got[0], c['out'], c['name'])
    assert {c['crop'] for c in cases} == {'eigen', 'stillbox'}


def case_errors_medians(device):
    """The medians exactly: a gt of one value and a prediction of another give scale = median ratio, so every prediction
    is scaled onto the ground truth: abs_rel 0 and a1 1 only if both medians (odd and even counts) are exact."""
    for n_valid in (7, 8):
        H, W = 10, 12
        gt = np.zeros((H, W))
        pred = np.full((H, W), 3.0, np.float32)
        ys, xs = np.unravel_index(np.arange(n_valid) + 60, (H, W))
        gt[ys, xs] = np.linspace(2.0, 9.0, n_valid)
        pred[ys, xs] = (gt[ys, xs] * 0.37).astype(np.float32)
        got = run_errors(device, gt[None], pred[None], (0, 1, 0, 1), 1e-3, 80.0)
        want = OD.sample_errors(gt, pred, crop=(0, 1, 0, 1))
        check_errors(got[0], want)


def case_errors_vs_oracle(device, B=2, H=60, W=200, seed=12, reruns=0, crop='eigen'):
    """Random samples with poses against oracle.sample_errors, per sample; reruns must give the same bits."""
    rs = np.random.RandomState(seed)
    ins = [error_inputs(rs, H, W) for _ in range(B)]
    gt, pred = np.stack([i[0] for i in ins]), np.stack([i[1] for i in ins])
    poses = rs.randn(B, 4, 6).astype(np.float32)
    disp = rs.uniform(-0.5, 2.0, (B, 4))
    disp[0, 1] = 0.0
    got = run_errors(device, gt, pred, crop, 1e-3, 80.0, poses, disp)
    for b in range(B):
        check_errors(got[b], OD.sample_errors(gt[b], pred[b], crop=crop_fractions(crop), poses=poses[b], displacements=disp[b]))
    for _ in range(reruns):
        assert np.array_equal(run_errors(device, gt, pred, crop, 1e-3, 80.0, poses, disp), got)
    return got


def case_errors_batch_is_per_sample(device):
    """A batch with poses equals its samples run alone, bit for bit; without poses row 0 is zeros and row 1 unchanged."""
    rs = np.random.RandomState(21)
    ins = [error_inputs(rs, 30, 70) for _ in range(3)]
    gt, pred = np.stack([i[0] for i in ins]), np.stack([i[1] for i in ins])
    poses, disp = rs.randn(3, 2, 6).astype(np.float32), rs.uniform(0.1, 2.0, (3, 2))
    disp[2] = -1.0                                          # no positive displacement: scale 0
    got = run_errors(device, gt, pred, 'stillbox', 1e-3, 80.0, poses, disp)
    for b in range(3):
        assert np.array_equal(run_errors(device, gt[b:b + 1], pred[b:b + 1], 'stillbox', 1e-3, 80.0, poses[b:b + 1],
                                         disp[b:b + 1])[0], got[b]), b
    plain = run_errors(device, gt, pred, 'stillbox', 1e-3, 80.0)
    assert not plain[:, 0].any() and np.array_equal(plain[:, 1], got[:, 1])
    assert got[2, 0, 0] == 1.0 and np.isinf(got[2, 0, 3]) and not got[2, 0, 4:].any()       # the zero-scale row


def case_arg_errors(device):
    """Null pointers, bad sizes, crop fractions outside [0, 1], poses without displacements and short workspaces return
    CCB_ERR_ARG and launch nothing (the outputs keep their contents)."""
    lib = _lib.lib()
    B, H, W = 1, 6, 9
    gt, pred = torch.ones(B, H, W, dtype=torch.float64, device=device), torch.ones(B, H, W, device=device)
    poses, disp = torch.ones(B, 2, 6, device=device), torch.ones(B, 2, dtype=torch.float64, device=device)
    nbytes = lib.ccb_eigen_depth_errors_workspace_bytes(B, H, W)
    work = torch.zeros(nbytes // 8 + 1, dtype=torch.int64, device=device)
    out = torch.full((B, 2, 7), -7.0, dtype=torch.float64, device=device)
    crop = (_lib.C.c_double * 4)(0, 1, 0, 1)
    bad_crop = (_lib.C.c_double * 4)(0, 1.5, 0, 1)
    good = dict(gt=gt.data_ptr(), pred=pred.data_ptr(), B=B, H=H, W=W, lo=_lib.C.c_double(1e-3), hi=_lib.C.c_double(80.0),
                crop=crop, poses=poses.data_ptr(), disp=disp.data_ptr(), R=2, work=work.data_ptr(), work_bytes=nbytes,
                out=out.data_ptr(), stream=_lib.stream(gt))
    before = lib.ccb_launch_count()
    for change in [dict(gt=None), dict(pred=None), dict(crop=None), dict(out=None), dict(work=None), dict(poses=None),
                   dict(disp=None), dict(B=0), dict(H=0), dict(W=-1), dict(R=0), dict(crop=bad_crop),
                   dict(work_bytes=nbytes - 1)]:
        assert lib.ccb_eigen_depth_errors(*dict(good, **change).values()) == -1, change
        assert lib.ccb_last_error_string().startswith(b'eigen_depth_errors')
    assert lib.ccb_eigen_depth_errors_workspace_bytes(1, 0, 3) == -1
    # ccb_velo_depth
    pts, offs = torch.ones(5, 4, device=device), torch.tensor([0, 5], dtype=torch.int64, device=device)
    P, depth = torch.ones(B, 3, 4, dtype=torch.float64, device=device), torch.full((B, H, W), -7.0, dtype=torch.float64, device=device)
    vbytes = lib.ccb_velo_depth_workspace_bytes(B, H, W)
    vwork = torch.zeros(vbytes // 8 + 1, dtype=torch.int64, device=device)
    vgood = dict(pts=pts.data_ptr(), offs=offs.data_ptr(), P=P.data_ptr(), total=_lib.C.c_longlong(5), B=B, H=H, W=W,
                 work=vwork.data_ptr(), work_bytes=_lib.C.c_longlong(vbytes), depth=depth.data_ptr(), stream=_lib.stream(gt))
    for change in [dict(pts=None), dict(offs=None), dict(P=None), dict(depth=None), dict(work=None), dict(B=0), dict(H=0),
                   dict(W=0), dict(total=_lib.C.c_longlong(-1)), dict(work_bytes=_lib.C.c_longlong(vbytes - 1))]:
        assert lib.ccb_velo_depth(*dict(vgood, **change).values()) == -1, change
        assert lib.ccb_last_error_string().startswith(b'velo_depth')
    assert lib.ccb_velo_depth_workspace_bytes(1, 6, 0) == -1
    # ccb_spline_zoom
    zbytes = lib.ccb_spline_zoom_workspace_bytes(B, H, W)
    zwork = torch.zeros(zbytes // 8 + 1, dtype=torch.int64, device=device)
    zout = torch.full((B, 4, 5), -7.0, device=device)
    zgood = dict(src=pred.data_ptr(), N=B, h=H, w=W, H=4, W=5, lo=_lib.C.c_float(0), hi=_lib.C.c_float(1),
                 work=zwork.data_ptr(), work_bytes=_lib.C.c_longlong(zbytes), dst=zout.data_ptr(), stream=_lib.stream(gt))
    for change in [dict(src=None), dict(dst=None), dict(work=None), dict(N=0), dict(h=0), dict(W=0),
                   dict(work_bytes=_lib.C.c_longlong(zbytes - 1))]:
        assert lib.ccb_spline_zoom(*dict(zgood, **change).values()) == -1, change
        assert lib.ccb_last_error_string().startswith(b'spline_zoom')
    assert lib.ccb_spline_zoom_workspace_bytes(0, 6, 9) == -1
    assert lib.ccb_launch_count() == before
    assert (out.cpu() == -7).all() and (depth.cpu() == -7).all() and (zout.cpu() == -7).all()
    assert lib.ccb_eigen_depth_errors(*good.values()) == 0 and lib.ccb_velo_depth(*vgood.values()) == 0
    assert lib.ccb_spline_zoom(*zgood.values()) == 0
    assert lib.ccb_launch_count() > before


ALL_CASES = [case_velo_vs_oracle, case_velo_batch_is_per_sample, case_errors_fixture, case_errors_medians,
             case_errors_vs_oracle, case_errors_batch_is_per_sample, case_arg_errors]


# ---- the whole sample with nets ---------------------------------------------------------------

def case_eval_batch(device, with_pose, B=2, h=64, w=128, Hg=94, Wg=300):
    """depth_eval_batch against the host depth_sample_errors on the same nets and frames (within 1e-6 relative, a* within
    one pixel over n) and against the oracle-net evaluation with the tolerances of tests/eval_cases.py."""
    from oracle import evaluate as OE
    from tests.eval_cases import _frames_u8
    from tests.net_cases import _load
    rs = np.random.RandomState(40 + with_pose)
    frames = [_frames_u8(5, h, w, seed=80 + b) for b in range(B)]
    gt = np.stack([error_inputs(rs, Hg, Wg, fill=0.4)[0] for _ in range(B)])
    disp = rs.uniform(0.2, 1.5, (B, 4))
    disp[0, 2] = 0.0
    disp_w, pose_w = ON.disp_params(), ON.pose_params()
    dnet = _load(CM.DispResNet6(), disp_w, device)
    pnet = _load(CM.PoseNetB6(nb_ref_imgs=4), pose_w, device) if with_pose else None
    tgt = torch.cat([CE._to_net_input(f[2], device) for f in frames])
    refs = [torch.cat([CE._to_net_input(f[k], device) for f in frames]) for k in (0, 1, 3, 4)]
    got = CE.depth_eval_batch(dnet, tgt, torch.from_numpy(gt).to(device), pose_net=pnet, refs=refs if with_pose else None,
                              displacements=torch.from_numpy(disp).to(device) if with_pose else None).cpu().numpy()
    assert got.shape == (B, 2, 7)
    for b in range(B):
        mask = OD.generate_mask(gt[b], 1e-3, 80.0)
        n = int(mask.sum())
        extra = (frames[b][2], gt[b], mask, 1e-3, 80.0)
        host = CE.depth_sample_errors(dnet, *extra, pnet, [frames[b][k] for k in (0, 1, 3, 4)] if with_pose else None,
                                      list(disp[b]) if with_pose else None, device=device)
        assert np.all(np.abs(got[b, :, :4] - host[:, :4]) <= 1e-6 * np.abs(host[:, :4]) + 1e-12), (b, got[b], host)
        assert np.all(np.abs(got[b, :, 4:] - host[:, 4:]) * n <= 1.0 + 1e-3), (b, got[b], host)
        want = OE.depth_sample_errors(disp_w, *extra, pose_w if with_pose else None,
                                      [frames[b][k] for k in (0, 1, 3, 4)] if with_pose else None,
                                      list(disp[b]) if with_pose else None)
        assert np.allclose(got[b], want, rtol=2e-3, atol=2e-4), (b, got[b], want)
        assert with_pose == bool(got[b, 0].any())
    return got
