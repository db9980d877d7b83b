"""Cases for the reference's remaining data transforms on the device (cc_b200.input_pipeline: RandomRotate, NormalizeLocally,
Scale), against the fixture frozen from the reference (tests/golden/make_augment.py), against the numpy restatements of
Pillow (tests/augment_oracle.py) and against oracle/make3d_eval.py's imresize.  Run by tests/test_augment.py on the CPU simulator and tests/test_gpu_augment.py on the
H100.  The rotate and resize kernels are bit-exact with Pillow, so their bytes are compared with np.array_equal."""
import random
import numpy as np
import torch
from cc_b200 import input_pipeline as CI
from tests import augment_oracle as AO
from tests.util import golden

FIXTURE = 'augment_small'


def _draw(g, case, **kw):
    s_random, s_np = (int(v) for v in g[case + '_seeds'])
    random.seed(s_random)
    np.random.seed(s_np)
    B, _, Hs, Ws, _ = g['frames'].shape
    return CI.draw_params(B, Hs, Ws, rotate=True, **kw)


def _check_decisions(p, angles):
    """draw_params(rotate=True) makes the reference's RandomRotate decisions: which samples rotate, and by which angle."""
    rotated = np.isfinite(angles)
    assert np.array_equal(p['rotate'], rotated), (p['rotate'], angles)
    assert np.array_equal(p['angle'][rotated], angles[rotated]), (p['angle'], angles)


def _stack(tgt, refs, t):
    """(tgt, refs) back into frame order [B,F,3,H,W] (numpy)."""
    return torch.stack(refs[:t] + [tgt] + refs[t:], 1).cpu().numpy()


def _kb(g, B):
    return np.broadcast_to(g['K'], (B, 3, 3)).copy()


def case_rotate_kernel_fixture(device):
    """ccb_rotate_frames_u8 equals the reference's imrotate byte for byte: the fixture's sampled angles (the identity for the
    samples that were not rotated), and one frame at fixed angles from 0.05 to 9.95 degrees."""
    g = golden(FIXTURE)
    frames = g['frames']
    B, F, Hs, Ws, _ = frames.shape
    p = dict(rotate=np.isfinite(g['rot_angle']), angle=np.nan_to_num(g['rot_angle']))
    got = CI.rotate_frames(torch.from_numpy(frames).to(device), CI.rotate_affines(p, B, Hs, Ws)).cpu().numpy()
    assert np.array_equal(got, g['rot_u8']), 'rotate: %d bytes differ' % (got != g['rot_u8']).sum()
    one, angles = g['angles_frame'], g['angles_deg']
    src = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(one, (len(angles), 1) + one.shape))).to(device)
    aff = np.array([CI.pil_rotate_affine(a, one.shape[1], one.shape[0]) for a in angles])
    got = CI.rotate_frames(src, aff).cpu().numpy()[:, 0]
    for i, a in enumerate(angles):
        assert np.array_equal(got[i], g['angles_u8'][i]), 'rotate by %g: %d bytes differ' % (a, (got[i] != g['angles_u8'][i]).sum())
        assert np.array_equal(AO.rotate_u8(one, aff[i]), g['angles_u8'][i]), 'oracle rotate by %g' % a


def case_resize_kernel_fixture(device):
    """ccb_resize_u8 equals the reference's imresize byte for byte, at a x0.68 downscale and at an upscale."""
    g = golden(FIXTURE)
    for name in ('down', 'up'):
        fr, want = g[name + '_frames'], g[name + '_u8']
        h, w = want.shape[2:4]
        got = CI.resize_frames(torch.from_numpy(fr).to(device), h, w).cpu().numpy()
        assert np.array_equal(got, want), '%s: %d bytes differ' % (name, (got != want).sum())
        assert np.array_equal(AO.resize_u8(fr[0, 0], h, w), want[0, 0]), 'oracle resize ' + name


def case_rotate_transform_golden(device):
    """(a) Compose([RandomRotate, RandomHorizontalFlip, ArrayToTensor, Normalize]): decisions from the same seeds, frames and
    intrinsics bit-exact."""
    g = golden(FIXTURE)
    frames = g['frames']
    B, F = frames.shape[:2]
    p = _draw(g, 'rot', scale_crop=False)
    _check_decisions(p, g['rot_angle'])
    tgt, refs, K, Kinv = CI.DeviceAugment(device, scale_crop=False, rotate=True)(torch.from_numpy(frames), _kb(g, B), params=p)
    out = _stack(tgt, refs, F // 2)
    assert np.array_equal(out, g['rot_out']), 'rotate + flip: max err %.3e' % np.abs(out - g['rot_out']).max()
    assert np.array_equal(K.cpu().numpy(), g['rot_K'])
    assert np.array_equal(Kinv.cpu().numpy(), np.linalg.inv(g['rot_K']))


def case_full_transform_golden(device):
    """(b) the flow-training transform with RandomScaleCrop: decisions and intrinsics exact; frames within the existing
    scale-crop bound (the lookup is not re-quantised to uint8 as the reference's resize is: one uint8 step per pass)."""
    g = golden(FIXTURE)
    frames = g['frames']
    B, F = frames.shape[:2]
    p = _draw(g, 'full')
    _check_decisions(p, g['full_angle'])
    tgt, refs, K, _ = CI.DeviceAugment(device, rotate=True)(torch.from_numpy(frames), _kb(g, B), params=p)
    out = _stack(tgt, refs, F // 2)
    assert np.abs(out - g['full_out']).max() <= 2 * (2 / 255) + 1e-6
    assert np.array_equal(K.cpu().numpy(), g['full_K'])


def case_local_transform_golden(device):
    """(c) (a) with NormalizeLocally: statistics within 2 fp32 ulp of the reference's (its fp32 sums against fp64 ones),
    frames within 1e-5."""
    g = golden(FIXTURE)
    frames = g['frames']
    B, F = frames.shape[:2]
    p = _draw(g, 'loc', scale_crop=False)
    _check_decisions(p, g['loc_angle'])
    aug = CI.DeviceAugment(device, scale_crop=False, rotate=True, normalization='local')
    tgt, refs, K, _ = aug(torch.from_numpy(frames), _kb(g, B), params=p)
    out = _stack(tgt, refs, F // 2)
    want_stats = g['loc_stats']
    stats = aug.stats.cpu().numpy()
    assert np.all(np.abs(stats - want_stats) <= 2 * np.spacing(np.abs(want_stats))), (stats, want_stats)
    assert np.abs(out - g['loc_out']).max() <= 1e-5, np.abs(out - g['loc_out']).max()
    assert np.array_equal(K.cpu().numpy(), g['loc_K'])


def case_scale_transform_golden(device):
    """(d) Compose([Scale(h, w), ArrayToTensor, Normalize]) at a downscale and an upscale: frames, K and K^-1 bit-exact."""
    g = golden(FIXTURE)
    for name in ('down', 'up'):
        fr, want = g[name + '_frames'], g[name + '_out']
        B, F = fr.shape[:2]
        h, w = want.shape[3:5]
        tgt, refs, K, Kinv = CI.DeviceScale(device, h=h, w=w)(torch.from_numpy(fr), _kb(g, B))
        out = _stack(tgt, refs, 0)
        assert np.array_equal(out, want), '%s: max err %.3e' % (name, np.abs(out - want).max())
        assert np.array_equal(K.cpu().numpy(), g[name + '_K'])
        assert np.array_equal(Kinv.cpu().numpy(), np.linalg.inv(g[name + '_K']))


class _Net(torch.nn.Module):
    """Stands in for one of flow_eval_batch's nets: records the inputs of each call and returns `out`."""

    def __init__(self, out):
        super().__init__()
        self.out, self.calls = out, []

    def forward(self, *args):
        self.calls.append(args)
        return self.out


def case_scale_low_contrast(device, B=2, F=5, Hs=80, Ws=200, h=64, w=192, seed=9):
    """(e) Scale on frames of 40..180, which imresize stretches to 0..255 before it resamples: DeviceScale's frames are
    the frames flow_eval_batch hands its nets, bit for bit, and equal the oracle's imresize, normalised."""
    from cc_b200 import evaluate as CE
    from oracle import make3d_eval as OM
    frames = np.random.RandomState(seed).randint(40, 181, size=(B, F, Hs, Ws, 3)).astype(np.uint8)
    K = np.tile(np.array([[120.0, 0, 100.0], [0, 120.0, 40.0], [0, 0, 1]], np.float32), (B, 1, 1))
    tgt, refs, _, _ = CI.DeviceScale(device, h, w)(torch.from_numpy(frames), K)
    out = _stack(tgt, refs, 0)
    pose = _Net(torch.zeros(B, F - 1, 6, device=device))
    nets = [_Net(torch.ones(B, 1, h, w, device=device)), pose, _Net(torch.ones(B, F - 1, h, w, device=device)),
            _Net(torch.zeros(B, 2, h, w, device=device))]
    gt, obj = torch.ones(B, 3, Hs, Ws, device=device), torch.ones(B, Hs, Ws, device=device)
    CE.flow_eval_batch(*nets, torch.from_numpy(frames).to(device), K, gt, obj, h=h, w=w)
    fed = _stack(*pose.calls[0], 0)
    assert np.array_equal(out, fed), 'DeviceScale against flow_eval_batch: max err %.3e' % np.abs(out - fed).max()
    want = np.stack([np.concatenate([OM.net_input(frames[b, f], h, w) for f in range(F)]) for b in range(B)])
    assert np.array_equal(out, want), 'DeviceScale against imresize: max err %.3e' % np.abs(out - want).max()


AUGMENT_CASES = [case_rotate_kernel_fixture, case_resize_kernel_fixture, case_rotate_transform_golden, case_full_transform_golden,
                 case_local_transform_golden, case_scale_transform_golden, case_scale_low_contrast]


# ---- full size, against the numpy restatements (no reference and no Pillow needed) -----------------------------------
def _unit(u8):
    """uint8 [..., H, W, 3] -> ArrayToTensor [..., 3, H, W] in fp32 (v / 255)."""
    return np.moveaxis(u8, -1, -3).astype(np.float32) / np.float32(255)


def case_rotate_fullsize(device, B=4, F=5, H=256, W=832, seed=7):
    """b4 x 5 frames at 256x832 with rotation: the rotated bytes equal the oracle's, the global transform (with scale-crop)
    is within the existing prep_frames bound of the float oracle, the local one (rotate + flip) matches the oracle's
    statistics within 2 ulp and its frames within 1e-5, and a repeat call gives the same bytes."""
    from oracle import transforms as OT
    rs = np.random.RandomState(seed)
    frames = rs.randint(0, 256, size=(B, F, H, W, 3)).astype(np.uint8)
    K = np.array([[483.3, 0, 408.3], [0, 492.6, 118.0], [0, 0, 1]], np.float32)
    Kb = np.broadcast_to(K, (B, 3, 3)).copy()
    random.seed(3)
    np.random.seed(4)
    p = CI.draw_params(B, H, W, rotate=True)
    pl = CI.draw_params(B, H, W, rotate=True, scale_crop=False)     # for the local run: rotate + flip only
    for q in (p, pl):
        q['rotate'][:] = [True, False, True, True]      # rotate most samples, keep one as it is
        q['angle'][:] = [0.37, 0.0, 9.91, 4.6]
        q['flip'][:] = p['flip']
    aff = CI.rotate_affines(p, B, H, W)
    dev_frames = torch.from_numpy(frames).to(device)
    rot = CI.rotate_frames(dev_frames, aff).cpu().numpy()
    want_rot = np.stack([np.stack([AO.rotate_u8(frames[b, f], aff[b]) for f in range(F)]) for b in range(B)])
    assert np.array_equal(rot, want_rot), 'rotate full size: %d bytes differ' % (rot != want_rot).sum()

    tgt, refs, Kd, _ = CI.DeviceAugment(device, rotate=True)(dev_frames, Kb, params=p)
    out = _stack(tgt, refs, F // 2)
    want, Kw = OT.apply(want_rot, K, p)
    bound = 2 * float(np.spacing(np.float32(max(p['scaled_w'].max(), p['scaled_h'].max())))) * 2.0   # as io_cases
    assert np.abs(out - want).max() <= bound, np.abs(out - want).max()
    assert np.array_equal(Kd.cpu().numpy(), Kw)

    runs = []
    for _ in range(2):
        aug = CI.DeviceAugment(device, scale_crop=False, rotate=True, normalization='local')
        tgt, refs, _, _ = aug(dev_frames, Kb, params=pl)
        runs.append((_stack(tgt, refs, F // 2), aug.stats.cpu().numpy()))
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1]), 'local normalisation is not repeatable'
    flipped = np.where(p['flip'][:, None, None, None, None] != 0, want_rot[:, :, :, ::-1], want_rot)
    for b in range(B):
        wo, wm, ws = AO.normalize_locally(_unit(flipped[b]))
        st = runs[0][1][b]
        assert np.all(np.abs(st[:, 0] - wm) <= 2 * np.spacing(np.abs(wm))), (st, wm)
        assert np.all(np.abs(st[:, 1] - ws) <= 2 * np.spacing(np.abs(ws))), (st, ws)
        assert np.abs(runs[0][0][b] - wo).max() <= 1e-5


def case_scale_fullsize(device, F=5, Hs=375, Ws=1242, h=256, w=832, seed=8):
    """One KITTI-2015-sized sample (5 x 375x1242) to 256x832: resized bytes equal the oracle's, the normalised frames are
    exactly (v/255 - .5)/.5 of them, and a repeat call gives the same bytes.  Scaled to its own size, the sample goes
    through unchanged: frames exactly (v/255 - .5)/.5 of the input, K as it was."""
    rs = np.random.RandomState(seed)
    frames = rs.randint(0, 256, size=(1, F, Hs, Ws, 3)).astype(np.uint8)
    src = torch.from_numpy(frames).to(device)
    got = CI.resize_frames(src, h, w).cpu().numpy()
    want = np.stack([AO.resize_u8(frames[0, f], h, w) for f in range(F)])[None]
    assert np.array_equal(got, want), 'resize full size: %d bytes differ' % (got != want).sum()
    assert np.array_equal(CI.resize_frames(src, h, w).cpu().numpy(), got)
    K = np.array([[721.5, 0, 609.6], [0, 721.5, 172.9], [0, 0, 1]], np.float32)[None]
    tgt, refs, Kd, Kinv = CI.DeviceScale(device, h, w)(src, K)
    out = _stack(tgt, refs, 0)
    assert np.array_equal(out, (_unit(want) - np.float32(0.5)) / np.float32(0.5))
    assert np.array_equal(Kd.cpu().numpy(), CI.scale_intrinsics(K, Hs, Ws, h, w))
    tgt, refs, Kd, _ = CI.DeviceScale(device, Hs, Ws)(src, K)
    out = _stack(tgt, refs, 0)
    assert np.array_equal(out, (_unit(frames) - np.float32(0.5)) / np.float32(0.5)), 'equal size is not the identity'
    assert np.array_equal(Kd.cpu().numpy(), K)
