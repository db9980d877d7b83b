"""Cases for the small exports around the fused kernels (SURVEY.md 8a rows a1, a17, a22):
helper functions of loss_functions.py, the stand-alone geometry functions of inverse_warp.py, and PROPERTY tests of
the 9x9 cost volume - the one boundary whose third-party implementation (spatial-correlation-sampler) is not in the
reference tree: the kernel is pinned against (i) a brute-force loop over the published definition, with the channel
permutation tables frozen from the reference's own constructor (models/back2future.py:56-59), (ii) shift
equivariance, (iii) the f1 <-> f2 symmetry, (iv) the zero-displacement channel, (v) adjointness of the backward."""
import numpy as np
import torch
from tests.util import golden, T, assert_close
from tests import layer_audit as LA
from cc_b200 import synth, nn as cnn, loss_functions as CL, inverse_warp as CW
from oracle import geometry as OG


def case_loss_helpers_golden(device):
    g = golden('helpers_small')
    B, H, W, NL = int(g['B']), int(g['H']), int(g['W']), int(g['NL'])
    s = synth.sample(B, H, W, seed=33, nlevels=NL)
    s = {k: ([t.to(device) for t in v] if isinstance(v, list) else v.to(device)) for k, v in s.items()}
    assert_close(CL.spatial_normalize(s['depth'][0]), g['spatial_normalize'], 1e-6)
    x = s['flow_fwd'][0]
    assert_close(CL.robust_l1(x), g['robust_l1'], 1e-6)
    assert_close(CL.robust_l1(x, q=0.35, eps=1e-3), g['robust_l1_q'], 1e-6)
    assert_close(CL.robust_l1_per_pix(x), g['robust_l1_per_pix'], 1e-6)
    ob, of = CL.occlusion_masks(s['flow_bwd'][0] * 3, s['flow_fwd'][0] * 3)
    assert torch.equal(ob.cpu(), T(g['occ_bw'])) and torch.equal(of.cpu(), T(g['occ_fw']))
    assert 0.01 < float(ob.mean()) < 0.99
    occ = CL.depth_occlusion_masks(s['depth'][0], s['pose'], s['K'], s['Kinv'])
    assert torch.equal(occ.cpu(), T(g['depth_occ'])), 'depth_occlusion_masks must be bit-exact'
    assert_close(CL.gaussian_explainability_loss(s['emask']), g['gauss_expl'], 1e-6)
    assert_close(CL.logical_or(s['emask'][0][:, :2], s['emask'][0][:, 2:]), g['logical_or'], 1e-6)
    rig_f = [(a - b).abs() for a, b in zip(s['flow_fwd'], s['flow_bwd'])]
    rig_b = [(a + b).abs() * 0.5 for a, b in zip(s['flow_fwd'], s['flow_bwd'])]
    jm = CL.compute_joint_mask_for_depth(s['emask'], rig_b, rig_f, 0.5)
    for i in range(NL):
        assert torch.equal(jm[i].cpu(), T(g[f'joint{i}'])), f'joint mask level {i}'
        assert not jm[i].requires_grad
    tgt = (s['emask'][0] > 0.5).float()
    assert_close(CL.weighted_binary_cross_entropy(s['emask'][0], tgt, [0.3, 0.7]), g['wbce'], 1e-6)
    assert_close(CL.weighted_binary_cross_entropy(s['emask'][0], tgt), g['wbce_none'], 1e-6)


def case_geometry_shims(device):
    """pixel2cam / cam2pixel / set_id_grid (inverse_warp.py:13-79): vs the oracle, composed into the fused kernel's
    result, and the reference's own --DEBUG self-check (train.py:732-738): inverse_warp == flow_warp(pose2flow) in bounds."""
    s = synth.sample(2, 24, 40, seed=12, nlevels=1)
    s = {k: ([t.to(device) for t in v] if isinstance(v, list) else v.to(device)) for k, v in s.items()}
    depth, pose, K, Kinv, img = s['depth'][0][:, 0], s['pose'][:, 0], s['K'], s['Kinv'], s['refs'][0]
    cam = CW.pixel2cam(depth, Kinv)
    assert_close(cam, OG.pixel2cam(depth, Kinv), 1e-7, 'pixel2cam')
    assert CW.pixel_coords.shape == (1, 3, 24, 40) and float(CW.pixel_coords[0, 0, 3, 7]) == 7 and float(CW.pixel_coords[0, 1, 3, 7]) == 3
    P = K.bmm(CW.pose_vec2mat(pose))
    for pm in ('zeros', None):
        px = CW.cam2pixel(cam, P[:, :, :3], P[:, :, -1:], pm)
        assert_close(px, OG.cam2pixel(cam, P[:, :, :3], P[:, :, -1:], pm), 1e-7, 'cam2pixel')
    px = CW.cam2pixel(cam, P[:, :, :3], P[:, :, -1:], 'zeros')
    composed = torch.nn.functional.grid_sample(img, px, padding_mode='zeros', align_corners=False)
    fused = CW.inverse_warp(img, depth, pose, K, Kinv)
    assert_close(fused, composed, 1e-5, 'inverse_warp kernel vs pixel2cam->cam2pixel->grid_sample')
    # train.py:732-738
    flow = CW.pose2flow(depth, pose, K, Kinv)
    via_flow = CW.flow_warp(img, flow)
    inb = ~CW.flow2oob(flow)
    diff = ((fused - via_flow).abs() * inb.unsqueeze(1)).sum() / (inb.sum() * 3).clamp(min=1)
    assert float(diff) < 1e-5, float(diff)
    assert float(inb.float().mean()) > 0.5


def _brute_corr(f1, f2):
    """out[b, i*9+j, y, x] = (1/C) sum_c f1[b,c,y,x] * f2[b,c,y+i-4,x+j-4], zero outside (SURVEY.md A.8) - plain loops."""
    f1, f2 = f1.double().cpu().numpy(), f2.double().cpu().numpy()
    B, C, h, w = f1.shape
    out = np.zeros((B, 81, h, w))
    for i in range(9):
        for j in range(9):
            for y in range(h):
                yy = y + i - 4
                if yy < 0 or yy >= h:
                    continue
                for x in range(w):
                    xx = x + j - 4
                    if 0 <= xx < w:
                        out[:, i * 9 + j, y, x] = (f1[:, :, y, x] * f2[:, :, yy, xx]).sum(1) / C
    return out


def case_corr81_properties(device):
    g = golden('helpers_small')
    idx_f, idx_b = g['idx_fwd'].astype(np.int64), g['idx_bwd'].astype(np.int64)
    assert sorted(idx_f.tolist()) == list(range(81)) and idx_b.tolist() == idx_f[::-1].tolist()
    gen = torch.Generator().manual_seed(21)
    B, C, h, w = 2, 5, 11, 14
    f1, f2 = torch.randn(B, C, h, w, generator=gen).to(device), torch.randn(B, C, h, w, generator=gen).to(device)
    brute = _brute_corr(f1, f2)
    # (i) definition + the reference's permutation tables
    for rev, idx in ((False, idx_f), (True, idx_b)):
        got = cnn.corr81(f1, f2, rev).double().cpu().numpy()
        assert np.abs(got - brute[:, idx]).max() <= 1e-6, 'corr81 vs brute force (reversed=%s)' % rev
    nat = np.empty(81, np.int64)
    nat[idx_f] = np.arange(81)                      # natural channel (i*9+j) -> position in the permuted output
    fwd = cnn.corr81(f1, f2, False)
    # (ii) shift equivariance: f2 shifted by (dy,dx) moves displacement (i,j) to (i+dy, j+dx)
    for dy, dx in ((1, 0), (0, -2), (-3, 2)):
        f2s = torch.zeros_like(f2)
        ys, yd = (slice(0, h - dy), slice(dy, h)) if dy >= 0 else (slice(-dy, h), slice(0, h + dy))
        xs, xd = (slice(0, w - dx), slice(dx, w)) if dx >= 0 else (slice(-dx, w), slice(0, w + dx))
        f2s[:, :, yd, xd] = f2[:, :, ys, xs]
        sh = cnn.corr81(f1, f2s, False)
        for i in range(9):
            for j in range(9):
                i2, j2 = i + dy, j + dx
                if 0 <= i2 < 9 and 0 <= j2 < 9:
                    a, b_ = sh[:, nat[i2 * 9 + j2]], fwd[:, nat[i * 9 + j]]
                    # identical wherever the displaced source pixel survived the shift (zero fill elsewhere)
                    yy = torch.arange(h).view(h, 1) + i - 4
                    xx = torch.arange(w).view(1, w) + j - 4
                    ok = ((yy >= max(0, -dy)) & (yy < h - max(0, dy)) & (xx >= max(0, -dx)) & (xx < w - max(0, dx))).to(device)
                    assert float(((a - b_).abs() * ok).max()) <= 1e-6, ('shift', dy, dx, i, j)
    # (iii) symmetry: corr(f1,f2)[(i,j)](y,x) == corr(f2,f1)[(8-i,8-j)](y+i-4, x+j-4)
    swp = cnn.corr81(f2, f1, False)
    for i, j in ((0, 0), (2, 7), (4, 4), (8, 3)):
        a = fwd[:, nat[i * 9 + j]]
        b_ = swp[:, nat[(8 - i) * 9 + (8 - j)]]
        for y in range(h):
            for x in range(w):
                yy, xx = y + i - 4, x + j - 4
                if 0 <= yy < h and 0 <= xx < w:
                    assert abs(float(a[0, y, x]) - float(b_[0, yy, xx])) <= 1e-6
    # (iv) zero displacement = channel mean of the product; bwd table is the reversed fwd table
    assert_close(fwd[:, nat[40]], (f1 * f2).mean(1), 1e-6, 'centre channel')
    assert_close(cnn.corr81(f1, f2, True), fwd.flip(1), 1e-7, 'idx_bwd = reversed idx_fwd')
    # (v) adjointness: <corr(f1,f2), G> == <f1, d_f1> == <f2, d_f2> for the bilinear form
    f1r, f2r = f1.clone().requires_grad_(True), f2.clone().requires_grad_(True)
    G = torch.randn(B, 81, h, w, generator=gen).to(device)
    out = cnn.corr81(f1r, f2r, False)
    d1, d2 = torch.autograd.grad((out * G).sum(), [f1r, f2r])
    lhs = float((out.detach() * G).sum())
    assert abs(float((f1 * d1).sum()) - lhs) <= 1e-4 * max(1.0, abs(lhs)) and abs(float((f2 * d2).sum()) - lhs) <= 1e-4 * max(1.0, abs(lhs))
    # (vi) forward and both gradients held element by element to the layer audit's cost-volume bound, both tables: one
    # channel; 6 and 13 channels, not a multiple of the kernel's channel group (the last chunk is ragged); h and w one
    # past a multiple of the kernel's pixel tile
    for (B_, C_, h_, w_) in ((1, 1, 17, 17), (2, 6, 17, 33), (1, 13, 33, 17)):
        assert C_ == 1 or C_ % LA.CORR_CG
        assert h_ % LA.CORR_CT == 1 and w_ % LA.CORR_CT == 1
        a = torch.randn(B_, C_, h_, w_, generator=gen).to(device).requires_grad_(True)
        b = torch.randn(B_, C_, h_, w_, generator=gen).to(device).requires_grad_(True)
        G = torch.randn(B_, 81, h_, w_, generator=gen).to(device)
        with LA.LayerAudit(report=False) as audit:
            for rev in (False, True):
                torch.autograd.grad((cnn.corr81(a, b, rev) * G).sum(), [a, b])
        assert [(r['op'], r['phase']) for r in audit.rows] == [('corr81', 'fwd'), ('corr81', 'bwd')] * 2, audit.rows
        assert {c for r in audit.rows for c in r['checks']} == {'out', 'd_f1', 'd_f2'}, audit.rows


HELPER_CASES = [case_loss_helpers_golden, case_geometry_shims, case_corr81_properties]
