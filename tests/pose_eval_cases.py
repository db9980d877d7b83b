"""Cases of the pose evaluation on the device (cc_b200.evaluate.pose_errors / pose_eval_batch over ccb_pose_errors), run on
the CPU simulator build (tests/test_pose_eval.py) and on the H100 (tests/test_gpu_pose_eval.py).

The references are tests/golden/pose_eval_small.npz (the reference's own frameworks, main-loop bodies, pose_vec2mat and
compute_pose_errors, tests/golden/make_pose_eval.py) and the oracle restatement (oracle/pose_eval.py).  The tree the
fixture's frameworks read is written here, so that the fixture maker and the tests write the same files.

Tolerances of the kernel against the oracle fed the same fp32 six-vectors: the kernel's sinf / cosf and torch's CPU sin /
cos may differ by an ulp or two (~1.2e-7 for the values of a rotation), which the fp64 algebra carries through a handful of
3x3 products and inverses of near-orthonormal matrices: rotation entries within 1e-6, translations within
1e-6 (1 + max|t|), ATE and RE within 1e-6 (1 + |v|).  The fp64 algebra alone (the oracle's compute_pose_error of the
kernel's own final poses against the kernel's errors) differs only by the rounding of a few dozen fp64 operations: 1e-12."""
import os
import numpy as np
import torch
from cc_b200 import _lib, evaluate as CE
from oracle import pose_eval as OP
from tests.util import golden

FIXTURE = 'pose_eval_small'
KITTI_PATTERNS = ['0*', '01']          # matches 00 and 01 (once), not 10
SINTEL_PATTERNS = ['alley_1']
KITTI_LENGTH, SINTEL_LENGTH = 5, 3
ALGEBRA = [(mode, L) for mode in ('euler', 'quat') for L in (3, 5)]


# ---- inputs --------------------------------------------------------------------------------------

def _rotation(rs, scale):
    a = scale * rs.randn(3)
    cx, sx, cy, sy, cz, sz = np.cos(a[0]), np.sin(a[0]), np.cos(a[1]), np.sin(a[1]), np.cos(a[2]), np.sin(a[2])
    return np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) @ \
        np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])


def trajectory(rs, n, scale=0.05):
    """n poses [n,3,4] fp64 of a camera driving forward and turning a little, rotations composed frame to frame."""
    R, t, out = _rotation(rs, 0.3), rs.randn(3), []
    for _ in range(n):
        out.append(np.concatenate([R, t[:, None]], 1))
        R = R @ _rotation(rs, scale)
        t = t + R @ np.array([0.05, 0.02, 1.0]) * (0.8 + 0.4 * rs.rand())
    return np.array(out)


def pose_vectors(rs, S, L, rotation_mode, zero_t=False):
    """[S,L-1,6] fp32 six-vectors like a pose net's: translations ~0.5, small rotations (euler angles / quaternion
    coefficients), the last snippet's rotations larger (up to ~0.8)."""
    p = np.concatenate([0.5 * rs.randn(S, L - 1, 3), 0.05 * rs.randn(S, L - 1, 3)], 2)
    p[-1, :, 3:] *= 16
    if zero_t:
        p[:, :, :3] = 0
    return p.astype(np.float32)


def write_frame(path, rs, H=6, W=10):
    from PIL import Image
    Image.fromarray(rs.randint(0, 256, (H, W, 3)).astype(np.uint8)).save(path, format='PNG')


def write_pose_tree(root, seed=7):
    """root/kitti: sequences 00 (7 frames), 01 (6) and 10 (5) with image_2/*.png (and a .jpg and a calib file that the
    framework skips) and poses/<seq>.txt in KITTI's 12 numbers per line; root/sintel: clean/alley_1 (6 frames) and
    camdata_left/alley_1/*.cam (tag 202021.25, 9 + 12 fp64), and clean/cave_2 that the patterns do not match."""
    rs = np.random.RandomState(seed)
    kitti = os.path.join(root, 'kitti')
    os.makedirs(os.path.join(kitti, 'poses'), exist_ok=True)
    for seq, n in (('00', 7), ('01', 6), ('10', 5)):
        d = os.path.join(kitti, 'sequences', seq, 'image_2')
        os.makedirs(d, exist_ok=True)
        for i in rs.permutation(n):
            write_frame(os.path.join(d, '%06d.png' % i), rs)
        write_frame(os.path.join(d, 'thumb.jpg'), rs)
        open(os.path.join(kitti, 'sequences', seq, 'calib.txt'), 'w').write('P0: 1 0 0 0\n')
        np.savetxt(os.path.join(kitti, 'poses', seq + '.txt'), trajectory(rs, n).reshape(n, 12), fmt='%.9e')
    sintel = os.path.join(root, 'sintel')
    for seq, n in (('alley_1', 6), ('cave_2', 4)):
        d, c = os.path.join(sintel, 'clean', seq), os.path.join(sintel, 'camdata_left', seq)
        os.makedirs(d, exist_ok=True)
        os.makedirs(c, exist_ok=True)
        K = np.array([[1120.0, 0, 511.5], [0, 1120.0, 217.5], [0, 0, 1]])
        for i, N in zip(rs.permutation(n), trajectory(rs, n, scale=0.1)):
            write_frame(os.path.join(d, 'frame_%04d.png' % (i + 1)), rs)
            with open(os.path.join(c, 'frame_%04d.cam' % (i + 1)), 'wb') as f:
                f.write(b'PIEH')
                f.write(K.astype(np.float64).tobytes())
                f.write(N.astype(np.float64).tobytes())
    return kitti, sintel


# ---- fixture --------------------------------------------------------------------------------------

def tree(kind):
    """The frozen framework of 'kitti' or 'sintel': n_rows, order (the reference's iteration order), and per sequence
    name: files (base names), snippets, gt, poses6 (the six-vectors fed), final, errors; imgs0 (the first snippet's
    frames) and the script's summary rows and predictions array in the reference's order."""
    g = golden(FIXTURE)
    seqs = {str(n): {k: g['%s_%s_%s' % (kind, n, k)] for k in ('files', 'snippets', 'gt', 'poses6', 'final', 'errors')}
            for n in g[kind + '_names']}
    return dict(n_rows=int(g[kind + '_n_rows']), order=[str(n) for n in g[kind + '_order']], seqs=seqs,
                imgs0=g[kind + '_imgs0'], summary=g[kind + '_summary'], predictions=g[kind + '_predictions'])


def algebra_cases():
    g = golden(FIXTURE)
    return [dict(name=str(c), mode=str(g[c + '_mode']), poses6=g[c + '_poses6'], gt=g[c + '_gt'], final=g[c + '_final'],
                 out=g[c + '_out']) for c in g['algebra_cases']]


# ---- checks ---------------------------------------------------------------------------------------

def _dev(a, device):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def check_final(got, want, name=''):
    """Rotation entries within 1e-6, translations within 1e-6 (1 + max|t|) of the snippet."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (name, got.shape, want.shape)
    assert np.all(np.abs(got[..., :3] - want[..., :3]) <= 1e-6), (name, np.abs(got[..., :3] - want[..., :3]).max())
    tmax = np.abs(want[..., 3]).max(axis=(-2, -1), keepdims=True)
    assert np.all(np.abs(got[..., 3] - want[..., 3]) <= 1e-6 * (1 + tmax)), (name, np.abs(got[..., 3] - want[..., 3]).max())


def check_errors(got, want, tol, name=''):
    """NaN where want has NaN, elsewhere within tol (1 + |v|)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (name, got, want)
    f = ~np.isnan(want)
    assert np.all(np.abs(got[f] - want[f]) <= tol * (1 + np.abs(want[f]))), (name, np.abs(got[f] - want[f]).max())


def check_kernel(device, poses6, gt, mode, sintel=False, want_final=None, want_out=None, name=''):
    """pose_errors on the device against the oracle fed the same six-vectors (and the frozen numbers where given), and the
    oracle's compute_pose_error of the kernel's own final poses against the kernel's errors."""
    out, final = CE.pose_errors(_dev(poses6, device), _dev(np.asarray(gt, np.float64), device), mode)
    out, final = out.cpu().numpy(), final.cpu().numpy()
    oracle_final = np.stack([OP.snippet_final(p, mode) for p in poses6])
    check_final(final, oracle_final, name)
    if want_final is not None:
        check_final(final, want_final, name)
    err = OP.sintel_pose_error if sintel else OP.pose_error
    col = slice(1, 2) if sintel else slice(0, 2)
    oracle_out = np.array([np.atleast_1d(err(g, f)) for g, f in zip(gt, oracle_final)])
    check_errors(out[:, col], oracle_out, 1e-6, name)
    if want_out is not None:
        check_errors(out[:, col], np.asarray(want_out).reshape(len(out), -1), 1e-6, name)
    own = np.array([np.atleast_1d(err(g, f)) for g, f in zip(gt, final)])
    check_errors(out[:, col], own, 1e-12, name)
    check_first_is_identity(final, poses6, name)
    return out, final


def check_first_is_identity(final, poses6, name=''):
    """final_0 = R_0 inv(R_0) [I | -t_0] + [0 | t_0] is [I|0] to fp64 rounding when inv is a true inverse; the transpose
    of the fp32-rounded R_0 (orthonormal to ~1e-7 only) leaves ~1e-7, which the 1e-6 bars above cannot see."""
    tmax = np.abs(poses6[..., :3]).max()
    assert np.abs(final[:, 0, :, :3] - np.eye(3)).max() <= 1e-12, (name, np.abs(final[:, 0, :, :3] - np.eye(3)).max())
    assert np.abs(final[:, 0, :, 3]).max() <= 1e-12 * (1 + tmax), (name, np.abs(final[:, 0, :, 3]).max())


# ---- cases ----------------------------------------------------------------------------------------

def case_algebra_fixture(device):
    """Each frozen case (euler and quat at L = 3 and 5, and all-zero translations: ATE NaN) against the reference."""
    cases = algebra_cases()
    for c in cases:
        check_kernel(device, c['poses6'], c['gt'], c['mode'], want_final=c['final'], want_out=c['out'], name=c['name'])
    assert any(np.isnan(c['out'][:, 0]).all() and np.isfinite(c['out'][:, 1]).all() for c in cases)


def case_tree_fixture(device):
    """The frozen frameworks' snippets: KITTI (ATE, RE) with its fp64 gt, Sintel (RE) with the fp64 upcast of its
    float32 gt."""
    for kind in ('kitti', 'sintel'):
        for name, s in tree(kind)['seqs'].items():
            mode = 'euler'
            check_kernel(device, s['poses6'], s['gt'], mode, sintel=kind == 'sintel', want_final=s['final'],
                         want_out=s['errors'], name=kind + name)


def case_vs_oracle(device, S=64, L=7, seed=3, reruns=0):
    """Random snippets of both rotation modes against the oracle; reruns give the same bits; without gt only the final
    poses are written, the same bits."""
    rs = np.random.RandomState(seed)
    for mode in ('euler', 'quat'):
        poses6 = pose_vectors(rs, S, L, mode)
        gt = np.stack([OP._compensated(trajectory(rs, L)) for _ in range(S)])
        out, final = check_kernel(device, poses6, gt, mode, name=mode)
        p = _dev(poses6, device)
        for _ in range(reruns):
            o2, f2 = CE.pose_errors(p, _dev(gt, device), mode)
            assert np.array_equal(o2.cpu().numpy(), out) and np.array_equal(f2.cpu().numpy(), final)
        none, f3 = CE.pose_errors(p, None, mode)
        assert none is None and np.array_equal(f3.cpu().numpy(), final)


def case_arg_errors(device):
    """Even, short or long snippets, no snippet, a bad rotation mode and NULL required pointers return CCB_ERR_ARG and
    launch nothing (outputs keep their contents)."""
    lib = _lib.lib()
    S, L = 2, 5
    poses = torch.zeros(S, L - 1, 6, device=device)
    gt = torch.zeros(S, L, 3, 4, dtype=torch.float64, device=device)
    final = torch.full((S, L, 3, 4), -7.0, dtype=torch.float64, device=device)
    out = torch.full((S, 2), -7.0, dtype=torch.float64, device=device)
    good = dict(poses=poses.data_ptr(), S=S, L=L, rot=_lib.ROT_EULER, gt=gt.data_ptr(), final=final.data_ptr(),
                out=out.data_ptr(), stream=_lib.stream(poses))
    before = lib.ccb_launch_count()
    for change in [dict(poses=None), dict(out=None), dict(gt=None), dict(gt=None, out=None, final=None), dict(S=0),
                   dict(L=4), dict(L=1), dict(L=17), dict(L=-3), dict(rot=2)]:
        assert lib.ccb_pose_errors(*dict(good, **change).values()) == -1, change
        assert lib.ccb_last_error_string().startswith(b'pose_errors'), change
    assert lib.ccb_launch_count() == before
    assert (out.cpu() == -7).all() and (final.cpu() == -7).all()
    long_poses = torch.zeros(1, 14, 6, device=device)                                          # the longest snippet
    long_final = torch.empty(1, 15, 3, 4, dtype=torch.float64, device=device)
    assert lib.ccb_pose_errors(*dict(good, poses=long_poses.data_ptr(), S=1, L=15, gt=None, final=long_final.data_ptr(),
                                     out=None).values()) == 0
    assert lib.ccb_pose_errors(*good.values()) == 0
    assert lib.ccb_launch_count() == before + 2
    # zero six-vectors: every final pose is [I|0]; a zero gt then gives 0/0 (ATE NaN) and tr(0) - 1 = -1 (RE = pi)
    eye = np.concatenate([np.eye(3), np.zeros((3, 1))], 1)
    assert np.array_equal(final.cpu().numpy(), np.broadcast_to(eye, (S, L, 3, 4)))
    o = out.cpu().numpy()
    assert np.isnan(o[:, 0]).all() and np.allclose(o[:, 1], np.pi, rtol=0, atol=1e-15)


ALL_CASES = [case_algebra_fixture, case_tree_fixture, case_vs_oracle, case_arg_errors]
