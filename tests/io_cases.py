"""Parity cases for the rows either side of the step (SURVEY.md 8f): validation metrics (N2) and the on-device input
pipeline (N1).  Shared by the CPU-simulator tests and the real-GPU tests, like tests/kernel_cases.py."""
import random
import numpy as np
import torch
from tests.util import golden, T, assert_close
from cc_b200 import loss_functions as CL, input_pipeline as CI
from oracle import metrics as OM, transforms as OT


def case_flow_metrics_golden(device):
    g = golden('metrics_small')
    gt, pr, pn, mask = (T(g[k], device) for k in ('gt', 'pr', 'pn', 'mask'))
    assert_close(CL.flow_diff(gt, pr), g['flow_diff'], 1e-5, 'flow_diff')
    for got, want, nm in ((CL.compute_epe(gt, pr), g['epe3'], 'epe masked'), (CL.compute_epe(gt[:, :2].contiguous(), pr), g['epe2'], 'epe plain'),
                          (CL.outlier_err(gt, pr * 3), g['outlier'], 'outliers')):
        assert isinstance(got, float)
        assert abs(got - float(want)) <= 1e-5 * max(abs(float(want)), 1e-3), (nm, got, float(want))
    assert_close(torch.tensor(CL.compute_all_epes(gt, pr, pn, mask)), g['all_epes'], 1e-5, 'compute_all_epes')
    assert_close(torch.tensor(CL.compute_all_epes(gt, pr, pn, mask, THRESH=0.3)), g['all_epes_t3'], 1e-5, 'compute_all_epes T=.3')


def case_depth_errors_golden(device):
    g = golden('metrics_small')
    gt, pr = T(g['dgt'], device), T(g['dpr'], device)
    for crop, key in ((True, 'errors_crop'), (False, 'errors_nocrop')):
        got = torch.stack([v.detach().cpu() for v in CL.compute_errors(gt, pr, crop=crop)])
        assert_close(got, g[key], 1e-5, key)
        assert (got[3:] - T(g[key])[3:]).abs().max().item() <= 2e-7, 'a1..a3 are counts / n'


def case_depth_errors_medians(device):
    """compute_errors scales by torch.median, the LOWER middle value.  Even count: gt 1..8 against four 1s and four 2s
    scales by 4 / 1 (the upper middle values would give 5 / 2); odd count: one pixel fewer.  Against the oracle, each
    sample alone and both in one batch."""
    gt = torch.arange(1, 9, dtype=torch.float32).reshape(1, 2, 4).repeat(2, 1, 1)
    pred = torch.tensor([1., 2., 1., 2., 2., 1., 2., 1.]).reshape(1, 2, 4).repeat(2, 1, 1)
    gt[1, 1, 3] = 0.                                                    # 7 valid pixels
    for sl in (slice(0, 1), slice(1, 2), slice(0, 2)):
        want = torch.stack([torch.as_tensor(v) for v in OM.compute_errors(gt[sl], pred[sl], crop=False)])
        got = torch.stack([v.cpu() for v in CL.compute_errors(gt[sl].to(device), pred[sl].to(device), crop=False)])
        assert_close(got, want, 1e-6, 'compute_errors medians, samples %s' % sl)


def case_metrics_oracle_sizes(device, B=2, Hg=375, Wg=1242, hp=256, wp=832, seed=3):
    """KITTI-2015 ground-truth size against full-resolution predictions (validate_flow_with_gt, train.py:588-668), and a
    depth map pair with ties around the median."""
    g = torch.Generator().manual_seed(seed)
    gt = torch.cat((torch.randn(B, 2, Hg, Wg, generator=g) * 8, (torch.rand(B, 1, Hg, Wg, generator=g) > 0.8).float()), 1)
    pr, pn = torch.randn(B, 2, hp, wp, generator=g) * 3, torch.randn(B, 2, hp, wp, generator=g) * 3
    mask = torch.rand(B, 1, hp // 4, wp // 4, generator=g)
    want = OM.compute_all_epes(gt, pr, pn, mask)
    got = CL.compute_all_epes(gt.to(device), pr.to(device), pn.to(device), mask.to(device))
    assert_close(torch.tensor(got), torch.tensor(want), 2e-5, 'compute_all_epes at KITTI size')
    assert abs(CL.compute_epe(gt.to(device), pr.to(device)) - OM.compute_epe(gt, pr)) <= 2e-5 * OM.compute_epe(gt, pr)
    dgt = (torch.rand(B, 128, 416, generator=g) * 90 - 5).round()      # integer depths: many equal keys around the median
    dpr = torch.rand(B, 128, 416, generator=g) * 70 + 0.1
    want = torch.stack([torch.as_tensor(v) for v in OM.compute_errors(dgt, dpr)])
    got = torch.stack([v.cpu() for v in CL.compute_errors(dgt.to(device), dpr.to(device))])
    assert_close(got, want, 2e-5, 'compute_errors')


def _params_like_reference(g, key_random, seed_np, B, Hs, Ws, scale_crop):
    random.seed(int(g[key_random]))
    if seed_np is not None:
        np.random.seed(int(seed_np))
    return CI.draw_params(B, Hs, Ws, scale_crop=scale_crop)


def case_input_pipeline_golden(device):
    """ccb_prep_frames + intrinsics update against the reference's train transform run on uint8 frames (fixture)."""
    g = golden('transforms_small')
    frames, K = torch.from_numpy(g['frames']), g['K']
    B, F, Hs, Ws, _ = frames.shape
    Kb = np.broadcast_to(K, (B, 3, 3)).copy()
    aug = CI.DeviceAugment(device)
    p = _params_like_reference(g, 'seed_random', g['seed_np'], B, Hs, Ws, True)
    tgt, refs, Kd, Kinv = aug(frames, Kb, params=p)
    out = torch.stack(refs[:F // 2] + [tgt] + refs[F // 2:], 1).cpu().numpy()
    assert np.array_equal(Kd.cpu().numpy(), g['K_out'])
    assert np.allclose(Kinv.cpu().numpy() @ g['K_out'], np.eye(3), atol=1e-5)
    # within PIL's two uint8 re-quantisations of the reference's resize, and within fp32 rounding of the float oracle
    assert np.abs(out - g['out']).max() <= 2 * (2 / 255) + 1e-6
    want, _ = OT.apply(g['frames'], K, p)
    assert np.abs(out - want).max() <= 2e-5
    p2 = _params_like_reference(g, 'seed_flip', None, B, Hs, Ws, False)
    tgt, refs, Kd, _ = CI.DeviceAugment(device, scale_crop=False)(frames, Kb, params=p2)
    out2 = torch.stack(refs[:F // 2] + [tgt] + refs[F // 2:], 1).cpu().numpy()
    assert np.array_equal(out2, g['out_flip']), 'flip + normalise without resize must be exact'
    assert np.array_equal(Kd.cpu().numpy(), g['K_flip'])


def case_input_pipeline_fullsize(device, B=4, Hs=256, Ws=832):
    """BASELINE frame size: uint8 [4,5,256,832,3] -> five normalised frames; against the float oracle."""
    rs = np.random.RandomState(9)
    frames = rs.randint(0, 256, size=(B, 5, Hs, Ws, 3)).astype(np.uint8)
    K = np.array([[483.3, 0, 408.3], [0, 492.6, 118.0], [0, 0, 1]], np.float32)
    random.seed(1)
    np.random.seed(2)
    p = CI.draw_params(B, Hs, Ws)
    tgt, refs, Kd, Kinv = CI.DeviceAugment(device)(torch.from_numpy(frames), np.broadcast_to(K, (B, 3, 3)).copy(), params=p)
    want, Kw = OT.apply(frames, K, p)
    out = torch.stack(refs[:2] + [tgt] + refs[2:], 1).cpu().numpy()
    # uniform-noise frames: neighbouring pixels differ by up to 2.0 (normalised), so one ulp of an fp32 source coordinate
    # near x = 900 (6.1e-5) moves a bilinear sample by up to 1.2e-4 - the bound is 2 ulp(coordinate) x the pixel range
    # (measured 1.3e-4; the smooth golden fixture above holds 2e-5)
    bound = 2 * float(np.spacing(np.float32(max(p['scaled_w'].max(), p['scaled_h'].max())))) * 2.0
    err = float(np.abs(out - want).max())
    assert err <= bound, 'input pipeline full size: max err %.3e > %.3e' % (err, bound)
    assert np.array_equal(Kd.cpu().numpy(), Kw)
    assert tgt.shape == (B, 3, Hs, Ws) and len(refs) == 4 and out.min() >= -1 - 1e-6 and out.max() <= 1 + 1e-6


IO_CASES = [case_flow_metrics_golden, case_depth_errors_golden, case_depth_errors_medians, case_input_pipeline_golden]
