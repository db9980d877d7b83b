"""Cases of the Make3D evaluation on the device (cc_b200.evaluate.make3d_frames / make3d_depth_errors / make3d_eval_batch
over ccb_bytescale_u8, ccb_resize_u8, ccb_spline_zoom and ccb_make3d_depth_errors), run on the CPU simulator build
(tests/test_make3d_eval.py) and on the H100 (tests/test_gpu_make3d_eval.py).

The references are tests/golden/make3d_eval_small.npz (the reference's own test_framework, its main-loop body and
compute_errors around a restatement of scipy 1.1's imresize, tests/golden/make_make3d_eval.py) and the oracle restatement
(oracle/make3d_eval.py).  The builders of the fixture's inputs live here so that the fixture maker and the tests write
the same files."""
import os
import numpy as np
import torch
from cc_b200 import _lib, evaluate as CE, models as CM
from cc_b200.input_pipeline import bytescale_frames
from oracle import make3d_eval as OM, nets as ON
from tests.util import golden

FIXTURE = 'make3d_eval_small'
FRAMEWORK_INDICES = (0, 60, 61, 62)        # the first, the two either side of the popped file, the last


# ---- inputs --------------------------------------------------------------------------------------

def write_make3d_tree(root, n=64, seed=5):
    """A Make3D-like tree of n images (lossless PNG data under .jpg names: no libjpeg in the loop) and n laser grids.
    The numbers in the names are not zero-padded and the two lists are numbered differently, so sorting reorders both
    and pairs by index files of different numbers.  Images are 2272 rows (the full Make3D height) and 4..6 columns
    (never 3: scipy's toimage would take a width of 3 for the channel axis); grids are Position3DGrid [55,7,4] fp64 with
    depths at exactly 1e-3 and 70, beyond 70 and 0."""
    from PIL import Image
    from scipy import io
    rs = np.random.RandomState(seed)
    os.makedirs(os.path.join(root, 'Test134'), exist_ok=True)
    os.makedirs(os.path.join(root, 'Gridlaserdata'), exist_ok=True)
    img_ids, depth_ids = rs.permutation(n) * 7 + 1, rs.permutation(n) * 11 + 3
    for k in range(n):
        img = rs.randint(0, 256, (2272, 4 + k % 3, 3)).astype(np.uint8)
        Image.fromarray(img).save(os.path.join(root, 'Test134', 'img-%d.jpg' % img_ids[k]), format='PNG')
        grid = np.round(rs.uniform(-2, 85, (55, 7, 4)) * 256) / 256
        grid[rs.rand(55, 7) < 0.1, 3] = 0.0
        grid[20, 1, 3], grid[21, 2, 3], grid[25, 4, 3] = 1e-3, 70.0, 70.0
        io.savemat(os.path.join(root, 'Gridlaserdata', 'depth_sph_corr-%d.mat' % depth_ids[k]), {'Position3DGrid': grid})


def error_inputs(rs, fill=0.7, k=0.45, H=21, W=305, lo=1e-3, hi=70.0):
    """(gt fp64 [21,305] with zeros, values beyond hi and some exactly lo and hi, pred fp32 [21,305] clipped to [lo, hi]
    near k * gt: the median scale is about 1/k, so scaled predictions pass hi and the cap matters)."""
    gt = np.where(rs.rand(H, W) < fill, np.round(rs.uniform(0.5, 80, (H, W)) * 256) / 256, 0.0)
    gt[rs.randint(0, H, 3), rs.randint(0, W, 3)] = lo
    gt[rs.randint(0, H, 3), rs.randint(0, W, 3)] = hi
    pred = np.clip(np.where(gt > 0, gt, 20.0) * rs.uniform(0.6, 1.6, (H, W)) * k, lo, hi).astype(np.float32)
    pred[rs.randint(0, H, 4), rs.randint(0, W, 4)] = np.float32(lo)
    pred[rs.randint(0, H, 4), rs.randint(0, W, 4)] = np.float32(hi)
    return gt, pred


# ---- fixture --------------------------------------------------------------------------------------

def stretch_cases():
    g = golden(FIXTURE)
    return [dict(name=str(c), crop=g[c + '_crop'], size=tuple(int(v) for v in g[c + '_size']), resize=bool(g[c + '_resize']),
                 stretched=g.get(c + '_stretched'), out=g[c + '_out']) for c in g['stretch_cases']]


def error_cases():
    g = golden(FIXTURE)
    return [dict(name=str(c), gt=g[c + '_gt'], pred=g[c + '_pred'], lo=float(g[c + '_lo']), hi=float(g[c + '_hi']),
                 out=g[c + '_out']) for c in g['error_cases']]


def framework():
    g = golden(FIXTURE)
    return dict(length=int(g['framework_length']), img_files=[str(f) for f in g['framework_img_files']],
                depth_files=[str(f) for f in g['framework_depth_files']],
                samples={i: dict(tgt=g['framework_%d_tgt' % i], gt_depth=g['framework_%d_gt_depth' % i],
                                 mask=g['framework_%d_mask' % i]) for i in FRAMEWORK_INDICES})


# ---- cases ------------------------------------------------------------------------------------

def _dev(a, device):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def check_errors(got, want, name=''):
    """a1..a3 exactly (counts over n), the rest within 1e-12 relative, nan and inf where the oracle has them."""
    got, want = np.asarray(got), np.asarray(want)
    assert np.array_equal(got[..., 4:], want[..., 4:], equal_nan=True), (name, got, want)
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(np.isinf(got), np.isinf(want)), (name, got, want)
    f = np.isfinite(want)
    assert np.all(np.abs(got[f] - want[f]) <= 1e-12 * np.abs(want[f])), (name, got, want)


def case_stretch_fixture(device):
    """bytescale_frames and make3d_frames on the fixture's crops: the stretched bytes and the resized bytes equal the
    reference's, byte for byte, and the net input is their normalisation; where the reference neither stretches nor
    resizes (no resize, or a crop already at the size) the crop goes through as it is."""
    cases = stretch_cases()
    for c in cases:
        h, w = c['size']
        if c['stretched'] is not None:
            got = bytescale_frames(_dev(c['crop'][None], device)).cpu().numpy()[0]
            assert np.array_equal(got, c['stretched']), (c['name'], int((got != c['stretched']).sum()))
            assert np.array_equal(got, OM.bytescale(c['crop'].astype(np.float32))), c['name']
        x = CE.make3d_frames(_dev(c['crop'][None], device), h, w, c['resize']).cpu().numpy()
        want = OM.net_input(c['out'], *c['out'].shape[:2])
        assert x.shape == want.shape and np.array_equal(x, want), (c['name'], x.shape, want.shape)
        assert np.array_equal(want, OM.net_input(c['crop'], h, w, c['resize'])), c['name']
    assert {c['name'] for c in cases if c['stretched'] is None} >= {'same_size', 'no_resize'}


def case_stretch_batch_is_per_image(device):
    """One range per image: a batch of crops of different ranges equals each crop stretched alone, and the oracle."""
    rs = np.random.RandomState(31)
    crops = np.stack([np.clip(rs.randint(lo, hi + 1, (40, 52, 3)), 0, 255) for lo, hi in ((0, 202), (60, 61), (7, 7), (0, 255))])
    crops = crops.astype(np.uint8)
    got = bytescale_frames(_dev(crops, device)).cpu().numpy()
    for b in range(len(crops)):
        assert np.array_equal(got[b], bytescale_frames(_dev(crops[b:b + 1], device)).cpu().numpy()[0]), b
        assert np.array_equal(got[b], OM.bytescale(crops[b].astype(np.float32))), b
    fr = CE.make3d_frames(_dev(crops, device), 16, 20).cpu().numpy()
    for b in range(len(crops)):
        assert np.array_equal(fr[b:b + 1], OM.net_input(crops[b], 16, 20)), b


def run_errors(device, gt, pred, lo=1e-3, hi=70.0):
    return CE.make3d_depth_errors(_dev(gt, device), _dev(pred, device), lo, hi).cpu().numpy()


def case_errors_fixture(device):
    """make3d_depth_errors on the fixture's samples against the numbers of the reference's main-loop body and
    compute_errors: row 1, row 0 zeros, the empty mask a NaN row."""
    cases = error_cases()
    for c in cases:
        got = run_errors(device, c['gt'][None], c['pred'][None], c['lo'], c['hi'])
        check_errors(got[0], c['out'], c['name'])
        assert not got[0, 0].any()
    assert any(np.isnan(c['out'][1]).all() for c in cases)


def case_errors_vs_oracle(device, B=3, seed=12, reruns=0):
    """Random samples against oracle.sample_errors, per sample; reruns give the same bits."""
    rs = np.random.RandomState(seed)
    ins = [error_inputs(rs, fill=0.3 + 0.2 * b) for b in range(B)]
    gt, pred = np.stack([i[0] for i in ins]), np.stack([i[1] for i in ins])
    got = run_errors(device, gt, pred)
    for b in range(B):
        check_errors(got[b], OM.sample_errors(gt[b], pred[b]), b)
    for _ in range(reruns):
        assert np.array_equal(run_errors(device, gt, pred), got)
    return got


def case_errors_batch_is_per_sample(device):
    """A batch (one sample with an empty mask) equals its samples run alone, bit for bit."""
    rs = np.random.RandomState(21)
    ins = [error_inputs(rs) for _ in range(3)]
    gt, pred = np.stack([i[0] for i in ins]), np.stack([i[1] for i in ins])
    gt[1] = np.where(gt[1] > 0, 90.0, 0.0)
    got = run_errors(device, gt, pred)
    for b in range(3):
        assert np.array_equal(run_errors(device, gt[b:b + 1], pred[b:b + 1])[0], got[b], equal_nan=True), b
    assert np.isnan(got[1, 1]).all() and np.isfinite(got[[0, 2]]).all()


def case_arg_errors(device):
    """Null pointers, bad sizes and short workspaces return CCB_ERR_ARG and launch nothing (outputs keep their contents)."""
    lib = _lib.lib()
    B, H, W = 1, 6, 9
    gt, pred = torch.ones(B, H, W, dtype=torch.float64, device=device), torch.ones(B, H, W, device=device)
    nbytes = lib.ccb_make3d_depth_errors_workspace_bytes(B, H, W)
    work = torch.zeros(nbytes // 8 + 1, dtype=torch.int64, device=device)
    out = torch.full((B, 2, 7), -7.0, dtype=torch.float64, device=device)
    good = dict(gt=gt.data_ptr(), pred=pred.data_ptr(), B=B, H=H, W=W, lo=_lib.C.c_double(1e-3), hi=_lib.C.c_double(70.0),
                work=work.data_ptr(), work_bytes=_lib.C.c_longlong(nbytes), out=out.data_ptr(), stream=_lib.stream(gt))
    before = lib.ccb_launch_count()
    for change in [dict(gt=None), dict(pred=None), dict(out=None), dict(work=None), dict(B=0), dict(H=0), dict(W=-1),
                   dict(work_bytes=_lib.C.c_longlong(nbytes - 1))]:
        assert lib.ccb_make3d_depth_errors(*dict(good, **change).values()) == -1, change
        assert lib.ccb_last_error_string().startswith(b'make3d_depth_errors')
    assert lib.ccb_make3d_depth_errors_workspace_bytes(1, 0, 3) == -1
    src = torch.full((2, H, W, 3), 9, dtype=torch.uint8, device=device)
    dst = torch.full_like(src, 7)
    sbytes = lib.ccb_bytescale_u8_workspace_bytes(2, H, W)
    swork = torch.zeros(sbytes // 8 + 1, dtype=torch.int64, device=device)
    sgood = dict(src=src.data_ptr(), N=2, H=H, W=W, work=swork.data_ptr(), work_bytes=_lib.C.c_longlong(sbytes),
                 dst=dst.data_ptr(), stream=_lib.stream(gt))
    for change in [dict(src=None), dict(dst=None), dict(work=None), dict(N=0), dict(H=0), dict(W=-2),
                   dict(work_bytes=_lib.C.c_longlong(sbytes - 1))]:
        assert lib.ccb_bytescale_u8(*dict(sgood, **change).values()) == -1, change
        assert lib.ccb_last_error_string().startswith(b'bytescale_u8')
    assert lib.ccb_bytescale_u8_workspace_bytes(2, 6, 0) == -1
    assert lib.ccb_launch_count() == before
    assert (out.cpu() == -7).all() and (dst.cpu() == 7).all()
    assert lib.ccb_make3d_depth_errors(*good.values()) == 0 and lib.ccb_bytescale_u8(*sgood.values()) == 0
    assert lib.ccb_launch_count() > before
    assert (dst.cpu() == 0).all()                      # a constant image: (x - cmin) * 255 = 0


ALL_CASES = [case_stretch_fixture, case_stretch_batch_is_per_image, case_errors_fixture, case_errors_vs_oracle,
             case_errors_batch_is_per_sample, case_arg_errors]


def case_real_size(device, B=4, reruns=2, seed=50):
    """B crops of 852x1704 (Make3D's 1704-column images) -> 256x256, each of another range, byte-exact against the oracle's
    imresize; reruns give the same bits."""
    rs = np.random.RandomState(seed)
    crops = np.stack([np.clip(rs.randint(lo, hi + 1, (852, 1704, 3)) + (np.arange(1704) // 200)[None, :, None], 0, 255)
                      for lo, hi in ((0, 202), (3, 240), (20, 21), (0, 255))][:B]).astype(np.uint8)
    src = _dev(crops, device)
    stretched = bytescale_frames(src)
    got = CE.make3d_frames(src, 256, 256)
    s_np, g_np = stretched.cpu().numpy(), got.cpu().numpy()
    for b in range(B):
        assert np.array_equal(s_np[b], OM.bytescale(crops[b].astype(np.float32))), b
        assert np.array_equal(g_np[b:b + 1], OM.net_input(crops[b], 256, 256)), b
    for _ in range(reruns):
        assert torch.equal(bytescale_frames(src), stretched) and torch.equal(CE.make3d_frames(src, 256, 256), got)


# ---- the whole sample with nets ---------------------------------------------------------------

def _make3d_crops(rs, B, Hs, Ws):
    from tests.eval_cases import _frames_u8
    crops = []
    for b in range(B):
        f = _frames_u8(3, Hs, Ws, seed=90 + b)[1].astype(np.int32)
        crops.append(np.clip(f // (2 + b) + 9 * b, 0, 255).astype(np.uint8))     # ranges short of 0..255: the stretch matters
    return np.stack(crops)


def disp_net(name, device):
    """DispResNet6 with the oracle's weights (its oracle net exists), or another disparity net, seeded."""
    from cc_b200 import synth
    from tests.net_cases import _load
    if name == 'DispResNet6':
        return _load(CM.DispResNet6(), ON.disp_params(), device)
    return synth.seeded_fill(getattr(CM, name)(), 77).to(device)


def host_sample_errors(net, crop, gt, h, w, device, lo=1e-3, hi=70.0):
    """test_make3d.py:98-148 of one sample on the host around the same net: the historical imresize, scipy's zoom and the
    oracle's errors."""
    from scipy.ndimage import zoom
    with torch.no_grad():
        x = torch.from_numpy(OM.net_input(crop, h, w)).to(device)
        pred_disp = net(x)[0, 0].float().cpu().numpy()
    pred_depth = 1 / pred_disp
    z = zoom(pred_depth, (gt.shape[0] / pred_depth.shape[0], gt.shape[1] / pred_depth.shape[1])).clip(lo, hi)
    return OM.sample_errors(gt, z, lo, hi)


def case_eval_batch(device, name, B=2, Hs=96, Ws=192, h=64, w=128):
    """make3d_eval_batch against the host path on the same net (within 1e-6 relative, a* within one pixel over n) and, for
    DispResNet6, against the oracle net with the tolerances of tests/eval_cases.py."""
    rs = np.random.RandomState(44)
    crops = _make3d_crops(rs, B, Hs, Ws)
    gt = np.stack([error_inputs(rs, k=1.0)[0] for _ in range(B)])
    net = disp_net(name, device)
    got = CE.make3d_eval_batch(net, _dev(crops, device), _dev(gt, device), h, w).cpu().numpy()
    assert got.shape == (B, 2, 7) and not got[:, 0].any()
    for b in range(B):
        n = int(((gt[b] > 1e-3) & (gt[b] < 70.0)).sum())
        host = host_sample_errors(net, crops[b], gt[b], h, w, device)
        assert np.all(np.abs(got[b, 1, :4] - host[1, :4]) <= 1e-6 * np.abs(host[1, :4]) + 1e-12), (b, got[b], host)
        assert np.all(np.abs(got[b, 1, 4:] - host[1, 4:]) * n <= 1.0 + 1e-3), (b, got[b], host)
        if name == 'DispResNet6':
            with torch.no_grad():
                pd = ON.disp_forward(ON.disp_params(), torch.from_numpy(OM.net_input(crops[b], h, w)), training=False)
            pred_depth = 1 / pd.numpy()[0, 0]
            from scipy.ndimage import zoom
            z = zoom(pred_depth, (21 / h, 305 / w)).clip(1e-3, 70.0)
            want = OM.sample_errors(gt[b], z)
            assert np.allclose(got[b], want, rtol=2e-3, atol=2e-4), (b, got[b], want)
    return got
