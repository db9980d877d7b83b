"""Cases of the KITTI-2015 flow evaluation (cc_b200.evaluate.flow_eval / flow_eval_batch / back2future_eval_batch over
ccb_flow_eval), run on the CPU simulator build (tests/test_flow_eval.py) and on the H100 (tests/test_gpu_flow_eval.py).

The references are tests/golden/flow_eval_small.npz (the reference's own ValidationFlow, flow_io.flow_read_png,
compute_all_epes and test_flow.py's sample body, tests/golden/make_flow_eval.py) and the oracle restatement
(oracle/flow_eval.py).  The inputs and the tree the fixture's ValidationFlow reads are written here, so that the fixture
maker and the tests use the same data.

The combined mask is compared bit for bit.  The numbers are fp32 sums over the ground-truth grid: the kernel sums in fp64
block partials, torch in fp32 in its own order, so they agree within the bars of ccb_flow_metrics' tests: 1e-5 relative,
2e-5 at KITTI size."""
import os
import numpy as np
import torch
from cc_b200 import _lib, evaluate as CE
from oracle import flow_eval as OF
from tests.util import golden

FIXTURE = 'flow_eval_small'
# name: (h, w, Hg, Wg, THRESH, epe_thresh, kind); kind picks the masks: mixed, rigid (bare everywhere), census (cam = fwd)
CASES = {'mixed': (24, 64, 37, 97, 0.01, 0.5, 'mixed'), 'rigid': (16, 40, 25, 61, 0.01, 0.5, 'rigid'),
         'census': (16, 40, 25, 61, 0.01, 0.5, 'census'), 'thresholds': (24, 64, 37, 97, 0.05, 0.3, 'mixed'),
         'kitti': (256, 832, 375, 1242, 0.01, 0.5, 'mixed')}
STORED = ('mixed', 'rigid', 'census', 'thresholds')       # inputs frozen in the fixture; 'kitti' is regenerated from its seed
TREE_N = 4
TREE_SIZES = {0: (14, 40), 1: (14, 40), 2: (12, 44), 3: (14, 40)}     # sample 2 has no obj_map
# h, w of the seeded net outputs of the tree samples: odd against the even frame sizes, so that no ground-truth pixel takes
# bilinear weights of exactly 1/2, where torch's CPU upsample (the fixture's) and its CUDA upsample (the kernel's) round a
# blend of the 0/1 mask to either side of compute_all_epes' 0.5
TREE_NET = (7, 17)
BAR, BAR_KITTI = 1e-5, 2e-5


def q256(a):
    return (np.round(np.asarray(a, np.float64) * 256) / 256).astype(np.float32)


def obj_ids(rs, H, W):
    """An object map with instance ids 0..3: background 0 and three boxes."""
    obj = np.zeros((H, W), np.uint8)
    for k in (1, 2, 3):
        y, x = rs.randint(0, H - 3), rs.randint(0, W - 5)
        obj[y:y + max(3, H // 3), x:x + max(5, W // 4)] = k
    return obj


def gt_flow(rs, Hg, Wg):
    """[3,Hg,Wg] float32 on KITTI's 1/64 grid, valid 0/1 (about 70 % valid), some large outliers to come."""
    u = np.round(rs.randn(Hg, Wg) * 12 * 64) / 64
    v = np.round(rs.randn(Hg, Wg) * 4 * 64) / 64
    return np.stack([u, v, (rs.rand(Hg, Wg) < 0.7)]).astype(np.float32)


def net_outputs(rs, h, w, kind, Hg=None, Wg=None, gt=None):
    """emask [1,3,h,w], cam and fwd [1,2,h,w] like the nets' (values on a 1/256 grid).  mixed: a quarter of the pixels
    bare-rigid, about a third within the census; rigid: every pixel bare-rigid; census: fwd = cam."""
    emask = q256(rs.rand(1, 3, h, w) * (0.6 if kind != 'rigid' else 0.2) + (0.0 if kind != 'rigid' else 0.8))
    if kind == 'mixed':
        emask[:, 1:] = np.where(rs.rand(1, 1, h, w) < 0.25, emask[:, 1:] + 0.4, emask[:, 1:] * 0.5)
    cam = q256(rs.randn(1, 2, h, w) * 3)
    if gt is not None:      # predictions near the ground truth, so that EPE and Fl are not dominated by noise
        cam = q256(torch.nn.functional.interpolate(torch.from_numpy(gt[None, :2]), size=(h, w), mode='bilinear',
                                                   align_corners=False)[0].numpy() * np.array([w / Wg, h / Hg])[:, None, None]
                   + rs.randn(2, h, w) * 0.5)[None]
    fwd = cam + q256(rs.randn(1, 2, h, w) * 2)
    near = rs.rand(1, 1, h, w) < (0.35 if kind == 'mixed' else 0.0)
    fwd = np.where(near, cam + q256(rs.randint(-1, 2, size=(1, 2, h, w)) / 256.), fwd)
    if kind == 'census':
        fwd = cam.copy()
    return emask.astype(np.float32), cam.astype(np.float32), fwd.astype(np.float32)


def case_inputs(name, seed=None):
    """(emask, cam, fwd, gt [1,3,Hg,Wg], obj [1,Hg,Wg]) of a kernel case from its seed."""
    h, w, Hg, Wg, _, _, kind = CASES[name]
    rs = np.random.RandomState(seed if seed is not None else 100 + sorted(CASES).index(name))
    gt = gt_flow(rs, Hg, Wg)
    obj = obj_ids(rs, Hg, Wg).astype(np.float32)
    emask, cam, fwd = net_outputs(rs, h, w, kind, Hg, Wg, gt)
    return emask, cam, fwd, gt[None], obj[None]


def calib_text(rs):
    P = np.array([[721.5377, 0, 609.5593, 44.85728], [0, 721.5377, 172.854, 0.2163791], [0, 0, 1, 0.002745884]])
    P[:2, :3] *= 1 + 0.01 * rs.randn()
    row = lambda a: ' '.join('%e' % v for v in a.reshape(-1))       # noqa: E731
    return ('calib_time: 09-Jan-2012 13:57:47\ncorner_dist: 9.950000e-02\nP_rect_00: %s\nP_rect_02: %s\n'
            'R_rect_02: %s\n' % (row(P * 0.9), row(P), row(np.eye(3))))


def write_flow_tree(root, seed=11):
    """root/data_scene_flow_multiview/training/image_2/iiiiii_{08..12}.png (RGB), data_scene_flow/training/flow_occ and
    flow_noc/iiiiii_10.png (16-bit KITTI triplets), obj_map/iiiiii_10.png (8-bit ids 0..3; none for sample 2) and
    data_scene_flow_calib/training/calib_cam_to_cam/iiiiii.txt for TREE_N samples of TREE_SIZES -> {path: uint16
    [H,W,3]} of every flow PNG written, the rows a PNG reader yields."""
    from PIL import Image
    from cc_b200.flowutils import flow_io
    rs = np.random.RandomState(seed)
    d = lambda *p: os.path.join(root, *p)       # noqa: E731
    for sub in (('data_scene_flow_multiview', 'training', 'image_2'), ('data_scene_flow', 'training', 'flow_occ'),
                ('data_scene_flow', 'training', 'flow_noc'), ('data_scene_flow', 'training', 'obj_map'),
                ('data_scene_flow_calib', 'training', 'calib_cam_to_cam')):
        os.makedirs(d(*sub), exist_ok=True)
    rows = {}
    for i in range(TREE_N):
        H, W = TREE_SIZES[i]
        name = str(i).zfill(6)
        base = rs.randint(20, 220, (H, W, 3))
        for k in (8, 9, 10, 11, 12):
            img = np.clip(base + rs.randint(-20, 21, (H, W, 3)), 0, 255).astype(np.uint8)
            Image.fromarray(img).save(d('data_scene_flow_multiview', 'training', 'image_2', '%s_%02d.png' % (name, k)))
        for occ in ('flow_occ', 'flow_noc'):
            g = gt_flow(rs, H, W)
            png = np.stack([g[0] * 64 + 2 ** 15, g[1] * 64 + 2 ** 15, g[2]], -1).astype(np.uint16)
            p = d('data_scene_flow', 'training', occ, name + '_10.png')
            flow_io.write_png(p, png)
            rows[p] = png
        if i != 2:
            Image.fromarray(obj_ids(rs, H, W)).save(d('data_scene_flow', 'training', 'obj_map', name + '_10.png'))
        with open(d('data_scene_flow_calib', 'training', 'calib_cam_to_cam', name + '.txt'), 'w') as f:
            f.write(calib_text(rs))
    return rows


def tree_net_outputs(i):
    """The seeded emask, cam and fwd at TREE_NET that stand in for the nets on tree sample i."""
    return net_outputs(np.random.RandomState(200 + i), *TREE_NET, 'mixed')


def g():
    return golden(FIXTURE)


def to(device, a):
    return torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a).to(device)


def stored_inputs(name):
    d = g()
    return tuple(d[name + '_' + k] for k in ('emask', 'cam', 'fwd', 'gt', 'obj'))


def _close(got, want, bar, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.all(np.abs(got - want) <= bar * np.maximum(1.0, np.abs(want))), (what, got, want)


def check_case(device, name, inputs, want_out, want_mask, want_b2f):
    """flow_eval on one case (batch 1) and its flow-only mode against the frozen or oracle numbers."""
    h, w, Hg, Wg, T, ET, _ = CASES[name]
    emask, cam, fwd, gt, obj = (to(device, a) for a in inputs)
    out, mask = CE.flow_eval(emask, cam, fwd, gt, obj, T, ET, want_mask=True)
    assert np.array_equal(mask.cpu().numpy(), want_mask), '%s: %d mask pixels differ' % (name, (mask.cpu().numpy() != want_mask).sum())
    bar = BAR_KITTI if name == 'kitti' else BAR
    _close(out[0].cpu().numpy(), want_out, bar, name)
    _close(CE.flow_eval(None, None, fwd, gt, obj, epe_thresh=ET)[0].cpu().numpy(), want_b2f, bar, name + ' flow only')
    return out[0].cpu().numpy()


def case_fixture(device):
    """The stored cases against the numbers and masks frozen from the reference's compute_all_epes and script body."""
    d = g()
    for name in STORED:
        check_case(device, name, stored_inputs(name), d[name + '_out'], d[name + '_mask'], d[name + '_b2f'])


def case_thresholds_kept_apart(device):
    """THRESH (census, 0.05) and compute_all_epes' THRESH (0.3) swapped give other numbers than the frozen ones."""
    d = g()
    emask, cam, fwd, gt, obj = (to(device, a) for a in stored_inputs('thresholds'))
    swapped = CE.flow_eval(emask, cam, fwd, gt, obj, 0.3, 0.05)[0].cpu().numpy()
    assert np.abs(swapped - d['thresholds_out']).max() > 100 * BAR, (swapped, d['thresholds_out'])


def case_kitti_size(device):
    """256x832 predictions against a 375x1242 ground truth: the numbers and mask frozen from the reference."""
    d = g()
    want_mask = np.unpackbits(d['kitti_mask_bits'])[:256 * 832].reshape(1, 1, 256, 832).astype(np.float32)
    check_case(device, 'kitti', case_inputs('kitti'), d['kitti_out'], want_mask, d['kitti_b2f'])


def case_vs_oracle(device, B=3, seed=5, reruns=0):
    """B samples of one size in one call against the oracle sample by sample; each row equals that sample run alone
    bit for bit (the partials do not depend on B); reruns give the same bits."""
    name = 'mixed'
    h, w, Hg, Wg, T, ET, _ = CASES[name]
    ins = [case_inputs(name, seed + k) for k in range(B)]
    stacked = [np.concatenate(a) for a in zip(*ins)]
    emask, cam, fwd, gt, obj = (to(device, a) for a in stacked)
    out, mask = CE.flow_eval(emask, cam, fwd, gt, obj, T, ET, want_mask=True)
    out_np = out.cpu().numpy()
    for k, one in enumerate(ins):
        errs, comb = OF.sample_errors(*(torch.from_numpy(a) for a in one), THRESH=T, epe_thresh=ET)
        assert np.array_equal(mask[k:k + 1].cpu().numpy(), comb.numpy())
        _close(out_np[k], errs, BAR, 'sample %d' % k)
        alone = CE.flow_eval(*(to(device, a) for a in one), T, ET)[0].cpu().numpy()
        assert np.array_equal(alone, out_np[k]), (k, alone, out_np[k])
    for _ in range(reruns):
        assert np.array_equal(CE.flow_eval(emask, cam, fwd, gt, obj, T, ET).cpu().numpy(), out_np)


def case_refused(device):
    """Bad arguments return -1 with no launch: C < 3, non-positive sizes, missing pointers, a short workspace, emask
    without flow_cam and a combined mask without emask."""
    lib = _lib.lib()
    emask, cam, fwd, gt, obj = (to(device, a) for a in case_inputs('rigid'))
    h, w, Hg, Wg = CASES['rigid'][:4]
    nbytes = lib.ccb_flow_eval_workspace_bytes(1, h, w, Hg, Wg)
    work = torch.empty(nbytes, dtype=torch.uint8, device=device)
    out = torch.full((1, 8), -3.0, device=device)
    mask = torch.full((1, 1, h, w), -3.0, device=device)
    good = dict(emask=emask.data_ptr(), cam=cam.data_ptr(), fwd=fwd.data_ptr(), gt=gt.data_ptr(), obj=obj.data_ptr(), B=1,
                C=3, h=h, w=w, Hg=Hg, Wg=Wg, T=0.01, ET=0.5, t0=3.0, t1=0.05, mask=mask.data_ptr(), work=work.data_ptr(),
                nbytes=nbytes, out=out.data_ptr(), stream=_lib.stream(emask))
    before = lib.ccb_launch_count()
    for change in (dict(C=2), dict(B=0), dict(h=0), dict(Wg=-1), dict(fwd=None), dict(gt=None), dict(obj=None),
                   dict(out=None), dict(cam=None), dict(emask=None), dict(emask=None, cam=None), dict(nbytes=nbytes - 1),
                   dict(work=None)):
        rc = lib.ccb_flow_eval(*dict(good, **change).values())
        assert rc == -1, change
        assert lib.ccb_last_error_string().startswith(b'flow_eval'), change
    assert lib.ccb_launch_count() == before
    assert torch.all(out == -3.0) and torch.all(mask == -3.0)
    for args in ((0, h, w, Hg, Wg), (1, 0, w, Hg, Wg), (1, h, w, Hg, -1)):
        assert lib.ccb_flow_eval_workspace_bytes(*args) == -1
    assert lib.ccb_flow_eval(*good.values()) == 0


def _flow_eval_row(dev):
    CE.flow_eval(*(to(dev, a) for a in case_inputs('rigid')), want_mask=True)


ALL_CASES = [case_fixture, case_thresholds_kept_apart, case_kitti_size, case_vs_oracle, case_refused]
