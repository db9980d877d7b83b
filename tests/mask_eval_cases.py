"""Cases of the motion segmentation evaluation (cc_b200.evaluate.motion_mask_counts / mask_sample_errors over ccb_mask_iou),
run on the CPU simulator build (tests/test_mask_eval.py) and on the H100 (tests/test_gpu_mask_eval.py).

The references are tests/golden/mask_eval_small.npz (the reference's own mask_error, tests/golden/make_mask_eval.py), the
oracle restatement (oracle/evaluate_mask.py: mask_error on numpy and scipy's zoom, rigidity_masks in torch on the CPU) and scipy
itself for the index map of zoom(order=0).  Counts are integers and are compared exactly; the kernel forms the masks with
correctly rounded fp32 operations, so on equal inputs its masks equal the oracle's bit for bit (the oracle takes its square
root through fp64 for that reason, see oracle.evaluate_mask.rigidity_masks)."""
import numpy as np
import torch
from scipy.ndimage import zoom
from cc_b200 import _lib, evaluate as CE, models as CM, synth
from oracle import evaluate_mask as OE, nets as ON
from tests import flownetc6_cases as FC
from tests.util import golden

FIXTURE = 'mask_eval_small'
KITTI = (256, 832, 375, 1242)          # the script's network and ground-truth sizes
KITTI_AXES = [(2, 832, 2, 1242), (256, 2, 375, 2)]      # one axis of it each (the map is separable; 2 -> 2 is the identity)
ODD = (32, 96, 47, 150)


def fixture_cases():
    g = golden(FIXTURE)
    return [(str(c), g[str(c) + '_pred'], g[str(g[str(c) + '_gt']) + '_obj'], g[str(g[str(c) + '_gt']) + '_sem'], g[str(c) + '_out'])
            for c in g['cases']]


def inputs_for_masks(bare, census):
    """emask [1,3,h,w], flow_cam, flow [1,2,h,w] whose masks are the given 0/1 arrays at THRESH 0.5: channel 1 carries
    `bare` and channel 2 is 0; the flows differ by 0 where `census` is set and by (3, 4) elsewhere (soft = 1 and 0).
    `census` must leave at least one pixel unset (max(d) > 0)."""
    h, w = bare.shape
    assert not census.all()
    emask = torch.zeros(1, 3, h, w)
    emask[0, 0] = 0.9                                      # channel 0 is not read
    emask[0, 1] = torch.from_numpy(bare.astype(np.float32))
    flow = torch.from_numpy(np.random.RandomState(3).randn(1, 2, h, w).astype(np.float32))
    gap = torch.from_numpy((~census.astype(bool)).astype(np.float32))
    flow_cam = flow + torch.stack([3 * gap, 4 * gap])[None]
    return emask, flow_cam, flow


def run(device, emask, flow_cam, flow, obj, sem, THRESH, want_masks=True):
    d = lambda a: torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a).to(device)      # noqa: E731
    out = CE.motion_mask_counts(d(emask), d(flow_cam), d(flow), d(obj), d(sem), THRESH, want_masks=want_masks)
    return (out[0].cpu(), out[1].cpu()) if want_masks else out.cpu()


def oracle_counts(masks, obj, sem):
    """[3,6] from the oracle mask_error of combined, census, bare ([h,w] arrays)."""
    return np.array([OE.mask_error(np.asarray(obj), np.asarray(sem), np.asarray(m)) for m in masks], np.int64)


def case_fixture(device, full=False):
    """The fixture's small cases, or its KITTI-size ones.  Each fixture mask as the bare mask, the previous case's mask of that size (or its complement) as the census: counts
    equal the frozen reference numbers for bare and the oracle for all three; the returned masks are the inputs."""
    seen = 0
    for name, pred, obj, sem, out in fixture_cases():
        if name.startswith('full_') != full:
            continue
        bare = pred.astype(bool)
        census = np.roll(~bare, 5, axis=1) if bare.all() else np.roll(bare, 7, axis=0) ^ np.roll(bare, 3, axis=1)
        counts, masks = run(device, *inputs_for_masks(bare, census), obj[None], sem[None], 0.5)
        assert np.array_equal(masks[0, 2].numpy(), bare.astype(np.float32)), name
        assert np.array_equal(masks[0, 1].numpy(), census.astype(np.float32)), name
        assert np.array_equal(masks[0, 0].numpy(), (bare | census).astype(np.float32)), name
        assert np.array_equal(counts[0, 2].numpy(), out.astype(np.int64)), (name, counts[0, 2], out)
        want = oracle_counts([(bare | census).astype(np.float32), census, bare], obj, sem)
        assert np.array_equal(counts[0].numpy(), want), (name, counts[0], want)
        seen += 1
    assert seen >= 2


def case_fixture_full(device):
    case_fixture(device, full=True)


def random_sample(B, h, w, Hg, Wg, seed, flow_scale=None):
    rs = np.random.RandomState(seed)
    emask = torch.from_numpy(rs.rand(B, 4, h, w).astype(np.float32) * 0.75)
    flow_cam = torch.from_numpy(rs.randn(B, 2, h, w).astype(np.float32))
    flow = torch.from_numpy(rs.randn(B, 2, h, w).astype(np.float32))
    if flow_scale is not None:                              # a different max(d) per sample
        flow_cam = flow_cam * torch.tensor(flow_scale).view(B, 1, 1, 1)
    obj = (rs.randint(1, 6, size=(B, Hg, Wg)) * (rs.rand(B, Hg, Wg) > 0.6)).astype(np.float32)
    sem = np.where(rs.rand(B, Hg, Wg) < 0.35, 26, 7).astype(np.float32)
    return emask, flow_cam, flow, torch.from_numpy(obj), torch.from_numpy(sem)


def case_random_vs_oracle(device, B=1, sizes=(64, 128, 96, 200), THRESH=0.6, seed=17, reruns=0):
    """Random nets' outputs: per sample, masks bit-identical to oracle.rigidity_masks (torch on the CPU) and counts equal to
    the oracle mask_error of those masks; both census labels present.  reruns: further runs must be bit-identical."""
    h, w, Hg, Wg = sizes
    emask, flow_cam, flow, obj, sem = random_sample(B, h, w, Hg, Wg, seed, flow_scale=[1.0 + 0.5 * b for b in range(B)])
    counts, masks = run(device, emask, flow_cam, flow, obj, sem, THRESH)
    for b in range(B):
        bare, census, combined, soft = OE.rigidity_masks(emask[b:b + 1], flow_cam[b:b + 1], flow[b:b + 1], THRESH)
        assert 0.02 < census.float().mean() < 0.98 and 0.02 < bare.float().mean() < 0.98
        want_masks = torch.cat([combined, census.float(), bare.float(), soft], 1)[0]
        assert torch.equal(masks[b], want_masks), 'sample %d: %d mask values differ' % (b, (masks[b] != want_masks).sum())
        want = oracle_counts([combined[0, 0].numpy(), census[0, 0].numpy(), bare[0, 0].numpy()], obj[b].numpy(), sem[b].numpy())
        assert np.array_equal(counts[b].numpy(), want), (b, counts[b], want)
    for _ in range(reruns):
        c2, m2 = run(device, emask, flow_cam, flow, obj, sem, THRESH)
        assert torch.equal(c2, counts) and torch.equal(m2, masks), 'a second run differs'
    return counts


def scipy_index_map(h, w, Hg, Wg):
    """(rows [Hg,Wg], cols [Hg,Wg]) of the source pixel zoom(order=0) reads, from scipy itself."""
    idx = zoom(np.arange(h * w, dtype=np.float64).reshape(h, w), (float(Hg) / float(h), float(Wg) / float(w)), order=0)
    assert idx.shape == (Hg, Wg)
    idx = idx.astype(np.int64)
    return idx // w, idx % w


def case_index_map(device, sizes):
    """The kernel's nearest-source-index map equals scipy's: sample k of one batch carries bit k of the source column (then of
    the source row) as its bare mask, and the ground truth carries the complement of that bit at the pixel scipy reads, so a
    single pixel read elsewhere shows up off the diagonal of the confusion matrix."""
    h, w, Hg, Wg = sizes
    rows, cols = scipy_index_map(h, w, Hg, Wg)
    nx, ny = max(1, int(w - 1).bit_length()), max(1, int(h - 1).bit_length())
    B = nx + ny
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing='ij')
    emask = torch.zeros(B, 3, h, w)
    obj = np.zeros((B, Hg, Wg), np.float32)
    for k in range(B):
        src, at = ((xx >> k) & 1, (cols >> k) & 1) if k < nx else ((yy >> (k - nx)) & 1, (rows >> (k - nx)) & 1)
        emask[k, 1] = torch.from_numpy(src.astype(np.float32))
        obj[k] = 1 - at                                       # mask bit 1 -> class 0 -> ground truth 0
    flow = torch.zeros(B, 2, h, w)
    sem = np.full((B, Hg, Wg), 26, np.float32)
    counts = run(device, emask, flow, flow, obj, sem, 0.5, want_masks=False)
    bare = counts[:, 2].numpy()
    assert (bare[:, [1, 2, 4, 5]] == 0).all(), 'pixels read at another index than scipy: %s' % bare[:, [1, 2]].tolist()
    assert (bare[:, 0] + bare[:, 3] == Hg * Wg).all()


def case_half_rounding(device):
    """3 -> 5 rows and 5 -> 9 columns put every second output coordinate exactly on .5: scipy reads the upper neighbour."""
    rows, cols = scipy_index_map(3, 5, 5, 9)
    assert rows[:, 0].tolist() == [0, 1, 1, 2, 2] and cols[0].tolist() == [0, 1, 1, 2, 2, 3, 3, 4, 4]
    case_index_map(device, (3, 5, 5, 9))


def case_zero_max(device):
    """flow_cam == flow everywhere: max(d) = 0, soft = 0/0 = NaN, the census is empty and combined = bare, as in the reference."""
    h, w, Hg, Wg = 16, 24, 20, 36
    emask, _, flow, obj, sem = random_sample(1, h, w, Hg, Wg, seed=5)
    counts, masks = run(device, emask, flow, flow, obj, sem, 0.94)
    bare, census, combined, soft = OE.rigidity_masks(emask, flow, flow, 0.94)
    assert torch.isnan(soft).all() and not census.any()
    assert torch.isnan(masks[0, 3]).all() and not masks[0, 1].any() and torch.equal(masks[0, 0], masks[0, 2])
    assert torch.equal(masks[0, 2], bare[0, 0].float())
    want = oracle_counts([combined[0, 0].numpy(), census[0, 0].numpy(), bare[0, 0].numpy()], obj[0].numpy(), sem[0].numpy())
    assert np.array_equal(counts[0].numpy(), want)
    assert counts[0, 1, 0] == 0 and counts[0, 1, 1] == 0        # census: nothing is predicted rigid


def case_batch_is_per_sample(device):
    """Two samples whose max(d) differ by 3x: the batched call equals two calls at B = 1, without and with the masks."""
    emask, flow_cam, flow, obj, sem = random_sample(2, 24, 40, 30, 62, seed=9, flow_scale=[1.0, 3.0])
    gaps = (flow_cam - flow).pow(2).sum(1).sqrt().flatten(1).max(1)[0]
    assert gaps[1] > 1.5 * gaps[0]
    counts, masks = run(device, emask, flow_cam, flow, obj, sem, 0.7)
    plain = run(device, emask, flow_cam, flow, obj, sem, 0.7, want_masks=False)          # null `masks`: the same counts
    assert torch.equal(plain, counts)
    for b in range(2):
        c1, m1 = run(device, emask[b:b + 1], flow_cam[b:b + 1], flow[b:b + 1], obj[b:b + 1], sem[b:b + 1], 0.7)
        assert torch.equal(c1[0], counts[b]) and torch.equal(m1[0], masks[b])
    assert not torch.equal(counts[0], counts[1])


def case_arg_errors(device):
    """Null pointers, C < 3, non-positive sizes and a short workspace return CCB_ERR_ARG and launch nothing (the counts
    buffer keeps its contents)."""
    lib = _lib.lib()
    B, C, h, w, Hg, Wg = 1, 3, 8, 12, 10, 14
    emask, fc, ff = (torch.rand(B, n, h, w, device=device) for n in (C, 2, 2))
    obj, sem = torch.zeros(B, Hg, Wg, device=device), torch.full((B, Hg, Wg), 26.0, device=device)
    nbytes = lib.ccb_mask_iou_workspace_bytes(B, h, w, Hg, Wg)
    assert nbytes >= 8
    work = torch.zeros(nbytes // 8 + 1, dtype=torch.int64, device=device)
    counts = torch.full((B, 3, 4), -7, dtype=torch.int64, device=device)
    good = dict(emask=emask.data_ptr(), flow_cam=fc.data_ptr(), flow=ff.data_ptr(), obj=obj.data_ptr(), sem=sem.data_ptr(), B=B, C=C,
                h=h, w=w, Hg=Hg, Wg=Wg, thresh=0.94, car=26, masks=None, work=work.data_ptr(), work_bytes=nbytes,
                counts=counts.data_ptr(), stream=_lib.stream(emask))
    before = lib.ccb_launch_count()
    bad = [dict(emask=None), dict(flow_cam=None), dict(flow=None), dict(obj=None), dict(sem=None), dict(work=None), dict(counts=None),
           dict(C=2), dict(B=0), dict(h=0), dict(w=-1), dict(Hg=0), dict(Wg=0), dict(work_bytes=nbytes - 1)]
    for change in bad:
        rc = lib.ccb_mask_iou(*dict(good, **change).values())
        assert rc == -1, (change, rc)                          # CCB_ERR_ARG
        assert lib.ccb_last_error_string().startswith(b'mask_iou')
    assert lib.ccb_launch_count() == before
    assert lib.ccb_mask_iou_workspace_bytes(0, h, w, Hg, Wg) == -1
    assert (counts.cpu() == -7).all()
    assert lib.ccb_mask_iou(*good.values()) == 0
    assert counts.cpu().sum() == 3 * Hg * Wg                   # every pixel is a car pixel: each mask counts all of them


# (flow net, its weights, THRESH).  The script's default 0.94 leaves the census of nets with seeded random weights nearly
# empty (Back2Future's flows reach tens of pixels against a camera flow of hundredths), so each case takes a THRESH near the
# median of its soft census: about half of the pixels on either side.
SAMPLE_CASES = {'Back2Future': (ON.flow_params, 0.16), 'FlowNetC6': (FC.step_flow_params, 0.7)}


def sample_mask_params():
    """oracle.nets.mask_params with the full-resolution head's bias lowered by 0.88: the seeded weights give masks of
    0.5 +- 0.05, for which the bare mask 1 - (1-e1)(1-e2) > 0.5 is all ones; around 1 - sqrt(0.5) = 0.29 it has both labels."""
    p = ON.mask_params()
    p['pred_mask1.bias'] = p['pred_mask1.bias'] - 0.88
    return p


def case_sample_errors(device, flownet):
    """evaluate.mask_sample_errors with all four nets against the oracle evaluation on the CPU.  The nets' outputs agree to
    about 1e-4, so a pixel on a threshold may flip: each count within 1 % of the valid pixels, each IoU within 0.01."""
    H, W, Hg, Wg = 64, 128, 96, 200
    flow_params, THRESH = SAMPLE_CASES[flownet]
    tgt, refs = synth.frames(1, H, W, seed=74)
    K, Kinv = synth.intrinsics(1, H, W)
    _, _, _, obj, sem = random_sample(1, H, W, Hg, Wg, seed=23)
    P = dict(disp=ON.disp_params(), pose=ON.pose_params(), mask=sample_mask_params(), flow=flow_params())
    want = OE.mask_sample_errors(P, tgt, refs, K, Kinv, obj, sem, THRESH, flownet=flownet)
    valid = int((sem == 26).sum())
    gt_moving = int(((sem == 26) & (obj != 0)).sum())
    assert 0 < gt_moving < valid, 'both ground-truth classes must be present'
    for name, m in zip(('combined', 'census', 'bare'), want[3][:3]):
        assert 0.05 < m.mean().item() < 0.95, 'the oracle %s mask is one-sided: %.3f' % (name, m.mean().item())

    def load(net, p):
        net.load_state_dict({k: v.clone() for k, v in p.items()})
        return net.to(device)

    flow_net = CM.Back2Future(nlevels=6) if flownet == 'Back2Future' else CM.FlowNetC6()
    nets = (load(CM.DispResNet6(), P['disp']), load(CM.PoseNetB6(nb_ref_imgs=4), P['pose']),
            load(CM.MaskNet6(nb_ref_imgs=4, output_exp=True), P['mask']), load(flow_net, P['flow']))
    d = lambda t: t.to(device)      # noqa: E731
    got = CE.mask_sample_errors(*nets, d(tgt), [d(r) for r in refs], d(K), d(Kinv), d(obj), d(sem), THRESH)
    assert got[3].shape == (1, 4, H, W)
    for name, g, o in zip(('combined', 'census', 'bare'), got[:3], want[:3]):
        assert len(g) == 6 and all(isinstance(v, int) for v in g)
        assert g[0] + g[1] + g[2] + g[3] == valid, (name, g, valid)       # tp_0 + fp_0 + fn_0 + tp_1: every valid pixel once
        assert max(abs(a - b) for a, b in zip(g, o)) <= 0.01 * valid, (name, g, o)
        for a, b in zip(CE.mask_iou(g), CE.mask_iou(o)):
            assert abs(a - b) <= 0.01, (name, CE.mask_iou(g), CE.mask_iou(o))
    differ = (got[3][0, :3].cpu() != want[3][:3]).float().mean().item()
    assert differ <= 0.01, 'masks: %.2e of the pixels differ from the oracle' % differ


ALL_CASES = [case_fixture, case_random_vs_oracle, case_half_rounding, case_zero_max, case_batch_is_per_sample, case_arg_errors]
