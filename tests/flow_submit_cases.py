"""Cases of the KITTI-2015 flow submission (cc_b200.evaluate.flow_submission / flow_colors / kitti_flow_errors over
ccb_flow_submit, ccb_flow_color and ccb_kitti_flow_errors), run on the CPU simulator build (tests/test_flow_submit.py) and
on the H100 (tests/test_gpu_flow_submit.py).

The references are tests/golden/flow_submit_small.npz (the reference's own flowlib / flow_io / compute_err,
tests/golden/make_flow_submit.py), the oracle restatement (oracle/flow_submit.py) and torch's CPU interpolate.  Every
comparison is exact: uint16 triplets, .flo bytes, uint8 levels and fp32 full-resolution flows bit for bit; the scores
within 1e-12 relative with equal outlier counts."""
import hashlib
import numpy as np
import torch
from cc_b200 import _lib, evaluate as CE, models as CM, synth
from cc_b200.flowutils import flow_io, flowlib
from oracle import flow_submit as OF, nets as ON
from tests import flownetc6_cases as FC
from tests.util import golden

FIXTURE = 'flow_submit_small'
KITTI = (256, 832, 375, 1242)
SUBMIT = {'small': (64, 128, 96, 200), 'odd': (32, 96, 47, 150)}
COLOR = ['wrap', 'unknown_nan', 'zero', 'stack3']


def g():
    return golden(FIXTURE)


def to(device, a):
    return torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a).to(device)


def flo_file(flo_hw2):
    return b'PIEH' + np.array([flo_hw2.shape[1], flo_hw2.shape[0]], np.int32).tobytes() + \
        np.ascontiguousarray(flo_hw2, np.float32).tobytes()


def check_submission(out, emask, cam, fwd, Hg, Wg, THRESH):
    """The kernel's dict against the oracle on the CPU (torch interpolate), bit for bit, sample by sample (the
    reference's bare-mask broadcast means what it says at batch 1 only) -> the oracle's (mask, cam, fwd, total)."""
    res = [OF.submit_flows(emask[k:k + 1], cam[k:k + 1], fwd[k:k + 1], Hg, Wg, THRESH) for k in range(emask.shape[0])]
    mask, cam_f, fwd_f, total_f = (torch.cat(t) for t in zip(*res))
    assert torch.equal(out['mask'].cpu(), mask)
    if 'full' in out:
        want = torch.stack([cam_f, fwd_f, total_f], 1)
        got = out['full'].cpu()
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), '%d full-resolution values differ' % (got != want).sum()
    for k in range(emask.shape[0]):
        png = OF.kitti_png_rows(total_f[k, 0].numpy(), total_f[k, 1].numpy())
        assert np.array_equal(out['png'][k].cpu().numpy(), png), 'sample %d: %d uint16 values differ' % (k, (out['png'][k].cpu().numpy() != png).sum())
        assert flo_file(out['flo'][k].cpu().numpy()) == OF.flo_bytes(total_f[k, 0].numpy(), total_f[k, 1].numpy())
    return mask, cam_f, fwd_f, total_f


def case_fixture_submit(device):
    """The small and odd fixture cases: mask, KITTI rows and .flo bytes equal the frozen reference outputs, the full
    flows and the row-2 colours equal oracle and fixture."""
    d = g()
    for name, (h, w, Hg, Wg) in SUBMIT.items():
        emask, cam, fwd = (torch.from_numpy(d[name + k]) for k in ('_emask', '_cam', '_fwd'))
        out = CE.flow_submission(to(device, emask), to(device, cam), to(device, fwd), Hg, Wg, 0.01, want_full=True)
        assert np.array_equal(out['mask'][0].cpu().numpy(), d[name + '_mask'])
        assert np.array_equal(out['png'][0].cpu().numpy(), d[name + '_png']), name
        b = flo_file(out['flo'][0].cpu().numpy())
        assert hashlib.sha256(b).hexdigest() == str(d[name + '_flo_sha256'])
        if name + '_flo' in d:
            assert b == d[name + '_flo'].tobytes()
        check_submission(out, emask, cam, fwd, Hg, Wg, 0.01)
        viz = CE.flow_colors(out['full'])[0].cpu().numpy()
        assert np.array_equal(viz, d[name + '_viz']), '%s: %d colour levels differ' % (name, (viz != d[name + '_viz']).sum())


def case_wrap_encoding(device):
    """Flows past +-512 px, on the truncation boundaries and past the int32 range: an identity-size call writes the flow
    as it is, and the triplet equals the reference's (numpy's cast: truncate, then wrap modulo 2^16)."""
    d = g()
    flow = torch.from_numpy(d['wrap_flow'])[None]
    _, h, w = d['wrap_flow'].shape
    emask = torch.zeros(1, 3, h, w)
    out = CE.flow_submission(to(device, emask), to(device, flow), to(device, flow), h, w, 0.01)
    assert np.array_equal(out['png'][0].cpu().numpy(), d['wrap_png'])
    # the kernel's identity resize keeps every value but the sign of a zero: fma(-0, 1, +0) = +0 (torch copies instead)
    assert np.array_equal(out['flo'][0].cpu().numpy(), np.frombuffer(d['wrap_flo'].tobytes()[12:], np.float32).reshape(h, w, 2))
    row = out['png'][0, 0, :6, 0].cpu().numpy().tolist()
    assert row[:2] == [65535, 0], row                                  # -1.5 -> 65535, -0.5 -> 0


def case_fixture_colors(device):
    """flow_colors equals the reference's flow_to_image: unknown and NaN pixels, zero flow, three panels, the wrap case."""
    d = g()
    for name in COLOR:
        flow = d[name + '_flow']
        panels = flow if flow.ndim == 4 else flow[None]
        got = CE.flow_colors(to(device, panels)[None])[0].cpu().numpy()
        assert np.array_equal(got, d[name + '_viz']), '%s: %d levels differ' % (name, (got != d[name + '_viz']).sum())
        want = OF.flow_to_image(np.hstack(list(panels)))
        assert np.array_equal(got / 255., want), name
    assert np.array_equal(flowlib.make_color_wheel(), d['wheel']) and np.array_equal(OF.make_color_wheel(), d['wheel'])


def case_flow_to_image_dropin(device):
    """flowlib.flow_to_image: numpy in -> the reference's float64 image, input untouched; tensor in -> uint8 on its device."""
    d = g()
    flow = d['unknown_nan_flow'].copy()
    img = flowlib.flow_to_image(flow)
    assert img.dtype == np.float64 and np.array_equal(img, d['unknown_nan_viz'] / 255.)
    assert np.array_equal(flow, d['unknown_nan_flow'], equal_nan=True)
    lv = flowlib.flow_to_image(to(device, d['stack3_flow'][1]))
    assert lv.dtype == torch.uint8 and lv.device.type == torch.device(device).type
    assert np.array_equal(lv.cpu().numpy(), np.round(OF.flow_to_image(d['stack3_flow'][1]) * 255).astype(np.uint8))


def case_random_colors(device, B=2, P=3, H=40, W=56, seed=5):
    """Random flows at several scales, per image one radius over its P panels: equal to the oracle's flow_to_image of the
    stacked panels, image by image (the batch does not mix radii)."""
    rs = np.random.RandomState(seed)
    flow = (rs.randn(B, P, 2, H, W) * rs.choice([0.3, 4.0, 60.0], size=(B, P, 1, 1, 1))).astype(np.float32)
    got = CE.flow_colors(to(device, flow)).cpu().numpy()
    for b in range(B):
        want = np.round(OF.flow_to_image(np.hstack(list(flow[b]))) * 255).astype(np.uint8)
        assert np.array_equal(got[b], want), 'image %d: %d levels differ' % (b, (got[b] != want).sum())


def random_submit_inputs(B, h, w, seed):
    rs = np.random.RandomState(seed)
    emask = torch.from_numpy((rs.rand(B, 4, h, w) * 0.6).astype(np.float32))
    cam = torch.from_numpy((rs.randn(B, 2, h, w) * 5).astype(np.float32))
    fwd = cam + torch.from_numpy((rs.randn(B, 2, h, w) * 3).astype(np.float32))
    near = torch.from_numpy(rs.rand(B, 1, h, w) < 0.4)
    fwd = torch.where(near, cam + torch.from_numpy((rs.rand(B, 2, h, w) * 0.018 - 0.009).astype(np.float32)), fwd)
    return emask, cam, fwd


def case_random_submit(device, B=1, sizes=(64, 128, 96, 200), seed=7, reruns=0, colors=True):
    """Random inputs with a third of the pixels in the census: every output equals the oracle bit for bit (the full
    flows against torch's CPU interpolate); reruns must give the same bits."""
    h, w, Hg, Wg = sizes
    emask, cam, fwd = random_submit_inputs(B, h, w, seed)
    out = CE.flow_submission(to(device, emask), to(device, cam), to(device, fwd), Hg, Wg, 0.01, want_full=True)
    assert 0.2 < out['mask'].float().mean().item() < 0.9
    _, cam_f, fwd_f, total_f = check_submission(out, emask, cam, fwd, Hg, Wg, 0.01)
    viz = CE.flow_colors(out['full']) if colors else None
    if colors:
        for b in range(B):
            want = np.round(OF.flow_to_image(np.hstack((cam_f[b].numpy(), fwd_f[b].numpy(), total_f[b].numpy()))) * 255)
            assert np.array_equal(viz[b].cpu().numpy(), want.astype(np.uint8)), 'image %d colours differ' % b
    for _ in range(reruns):
        again = CE.flow_submission(to(device, emask), to(device, cam), to(device, fwd), Hg, Wg, 0.01, want_full=True)
        assert all(torch.equal(again[k], out[k]) for k in out), 'a second run differs'
        if colors:
            assert torch.equal(CE.flow_colors(again['full']), viz)


def case_errors(device):
    """kitti_flow_errors equals the frozen compute_err and the oracle: fp64 within 1e-12 relative, outliers exact; the
    png codec's decoding equals flow_read_png's."""
    d = g()
    errs, counts = CE.kitti_flow_errors(to(device, d['err_gt']), to(device, d['err_pred']))
    errs, counts = errs.cpu().numpy()[0], counts.cpu().numpy()[0]
    assert np.allclose(errs, d['err_out'], rtol=1e-12, atol=0), (errs, d['err_out'])
    u_gt, v_gt, valid_gt = OF.decode_png_rows(d['err_gt'])
    u_p, v_p, _ = OF.decode_png_rows(d['err_pred'])
    want, n_err = OF.compute_err(u_gt, v_gt, valid_gt, u_p, v_p)
    assert want == d['err_out'].tolist()
    assert counts[0] == n_err and counts[1] == int(valid_gt.sum())


def case_errors_batch(device):
    """A batch of three: rows equal their images scored alone; an image without valid pixel gives NaN as numpy's 0/0."""
    d = g()
    gt = np.stack([d['err_gt'], d['err_pred'], d['err_gt']])
    pred = np.stack([d['err_pred'], d['err_gt'], d['err_pred']])
    gt[2, :, :, 2] = 0
    errs, counts = CE.kitti_flow_errors(to(device, gt), to(device, pred))
    for b in range(2):
        e1, c1 = CE.kitti_flow_errors(to(device, gt[b]), to(device, pred[b]))
        assert torch.equal(e1[0], errs[b]) and torch.equal(c1[0], counts[b])
    assert torch.isnan(errs[2]).all() and counts[2].tolist() == [0, 0]


def case_arg_errors(device):
    """Null pointers, C < 3, non-positive sizes and short workspaces return CCB_ERR_ARG and launch nothing."""
    lib = _lib.lib()
    B, C, h, w, Hg, Wg = 1, 3, 6, 8, 9, 12
    emask, cam, fwd = (torch.rand(B, n, h, w, device=device) for n in (C, 2, 2))
    mask = torch.zeros(B, 1, h, w, device=device)
    png = torch.zeros(B, Hg, Wg, 3, device=device, dtype=torch.uint16)
    flo = torch.zeros(B, Hg, Wg, 2, device=device)
    st = _lib.stream(emask)
    good = dict(emask=emask.data_ptr(), cam=cam.data_ptr(), fwd=fwd.data_ptr(), B=B, C=C, h=h, w=w, Hg=Hg, Wg=Wg, thresh=0.01,
                mask=mask.data_ptr(), full=None, png=png.data_ptr(), flo=flo.data_ptr(), stream=st)
    before = lib.ccb_launch_count()
    for change in [dict(emask=None), dict(cam=None), dict(fwd=None), dict(mask=None), dict(png=None), dict(flo=None), dict(C=2),
                   dict(B=0), dict(h=0), dict(w=-1), dict(Hg=0), dict(Wg=0)]:
        assert lib.ccb_flow_submit(*dict(good, **change).values()) == -1, change
        assert lib.ccb_last_error_string().startswith(b'flow_submit')
    flow = torch.rand(B, 1, 2, h, w, device=device)
    out = torch.zeros(B, 3, h, w, device=device, dtype=torch.uint8)
    nb = lib.ccb_flow_color_workspace_bytes(B, 1, h, w)
    work = torch.zeros(nb // 8 + 1, dtype=torch.int64, device=device)
    good = dict(flow=flow.data_ptr(), B=B, P=1, H=h, W=w, work=work.data_ptr(), nb=nb, out=out.data_ptr(), stream=st)
    for change in [dict(flow=None), dict(out=None), dict(work=None), dict(nb=nb - 1), dict(B=0), dict(P=0), dict(H=0), dict(W=0)]:
        assert lib.ccb_flow_color(*dict(good, **change).values()) == -1, change
        assert lib.ccb_last_error_string().startswith(b'flow_color')
    gt = torch.zeros(B, h, w, 3, device=device, dtype=torch.uint16)
    res = torch.zeros(B, 2, device=device, dtype=torch.float64)
    nb = lib.ccb_kitti_flow_errors_workspace_bytes(B, h, w)
    work = torch.zeros(nb // 8 + 1, dtype=torch.int64, device=device)
    good = dict(gt=gt.data_ptr(), pred=gt.data_ptr(), B=B, H=h, W=w, work=work.data_ptr(), nb=nb, out=res.data_ptr(), counts=None,
                stream=st)
    for change in [dict(gt=None), dict(pred=None), dict(work=None), dict(out=None), dict(nb=nb - 1), dict(B=0), dict(H=0), dict(W=-2)]:
        assert lib.ccb_kitti_flow_errors(*dict(good, **change).values()) == -1, change
        assert lib.ccb_last_error_string().startswith(b'kitti_flow_errors')
    assert lib.ccb_launch_count() == before
    for f, args in (('ccb_flow_color_workspace_bytes', (0, 1, h, w)), ('ccb_kitti_flow_errors_workspace_bytes', (B, 0, w))):
        assert getattr(lib, f)(*args) == -1
    assert (png.cpu() == 0).all() and (out.cpu() == 0).all() and (res.cpu() == 0).all()


ALL_CASES = [case_fixture_submit, case_wrap_encoding, case_fixture_colors, case_flow_to_image_dropin, case_random_colors,
             case_random_submit, case_errors, case_errors_batch, case_arg_errors]

# (flow net, its weights): the nets of tests/mask_eval_cases.py's sample cases
SAMPLE_NETS = {'Back2Future': ON.flow_params, 'FlowNetC6': FC.step_flow_params}


def case_submission_sample(device, flownet, tmpdir):
    """evaluate.flow_submission_sample with all four nets: the kernel's files equal the oracle's encoding of the product's
    own net outputs exactly; against the oracle pipeline (nets in fp64-faithful torch on the CPU) the decoded flows agree
    within the nets' tolerance plus 1/64 px; write_flow_submission writes the script's files and they read back."""
    import os
    H, W, Hg, Wg = 64, 128, 96, 200
    tgt, refs = synth.frames(1, H, W, seed=74)
    K, Kinv = synth.intrinsics(1, H, W)
    P = dict(disp=ON.disp_params(), pose=ON.pose_params(), mask=ON.mask_params(), flow=SAMPLE_NETS[flownet]())

    def load(net, p):
        net.load_state_dict({k: v.clone() for k, v in p.items()})
        return net.to(device)

    flow_net = CM.Back2Future(nlevels=6) if flownet == 'Back2Future' else CM.FlowNetC6()
    nets = (load(CM.DispResNet6(), P['disp']), load(CM.PoseNetB6(nb_ref_imgs=4), P['pose']),
            load(CM.MaskNet6(nb_ref_imgs=4, output_exp=True), P['mask']), load(flow_net, P['flow']))
    d = lambda t: t.to(device)      # noqa: E731
    dt, drefs, dK, dKinv = d(tgt), [d(r) for r in refs], d(K), d(Kinv)
    got = CE.flow_submission_sample(*nets, dt, drefs, dK, dKinv, Hg, Wg, 0.01, want_viz=True)
    assert got['viz'].shape == (1, 3, 3 * Hg, Wg) and got['png'].dtype == torch.uint16
    # the kernel against the oracle encoding of the product's own net outputs
    with torch.no_grad():
        for n in nets:
            n.eval()
        from cc_b200.inverse_warp import pose2flow
        emask = nets[2](dt, drefs)
        fwd = nets[3](dt, drefs[1:3])[0] if flownet == 'Back2Future' else nets[3](dt, drefs[2])
        cam = pose2flow((1 / nets[0](dt)).squeeze(1), nets[1](dt, drefs)[:, 2], dK, dKinv)
    _, cam_f, fwd_f, total_f = check_submission(got, emask.cpu(), cam.cpu(), fwd.cpu(), Hg, Wg, 0.01)
    want_viz = np.round(OF.flow_to_image(np.hstack((cam_f[0].numpy(), fwd_f[0].numpy(), total_f[0].numpy()))) * 255)
    assert np.array_equal(got['viz'][0].cpu().numpy(), want_viz.astype(np.uint8))
    # against the oracle pipeline: same composite where the masks agree, within tolerance + one PNG step
    (o_emask, o_cam, o_fwd), (o_mask, _, _, o_total), o_png, _ = OF.submission_sample(P, tgt, refs, K, Kinv, Hg, Wg, 0.01, flownet)
    u, v, _ = OF.decode_png_rows(got['png'][0].cpu().numpy())
    ou, ov, _ = OF.decode_png_rows(o_png)
    same = (got['mask'].cpu() == o_mask)[0, 0].numpy()
    assert same.mean() > 0.97, 'masks differ on %.3f of the pixels' % (1 - same.mean())
    scale = max(np.abs(ou).max(), np.abs(ov).max(), 1e-3)
    tol = 1e-3 * scale + 1 / 64 + 1e-12
    full_same = torch.nn.functional.interpolate(torch.from_numpy(same.astype(np.float32))[None, None], size=(Hg, Wg),
                                                mode='bilinear', align_corners=False)[0, 0].numpy() == 1
    assert np.abs(u - ou)[full_same].max() <= tol and np.abs(v - ov)[full_same].max() <= tol
    # the script's files
    CE.write_flow_submission(str(tmpdir), 0, got, dt)
    for rel in ('images/000.npy', 'mask/000.npy', 'testing/000000_10.png', 'testing_flo/000000_10.flo', 'viz/00002.png'):
        assert os.path.exists(os.path.join(str(tmpdir), rel)), rel
    u2, v2, valid = flow_io.flow_read_png(os.path.join(str(tmpdir), 'testing/000000_10.png'))
    assert np.array_equal(u2, u) and np.array_equal(v2, v) and (valid == 1).all()
    with open(os.path.join(str(tmpdir), 'testing_flo/000000_10.flo'), 'rb') as f:
        assert f.read() == OF.flo_bytes(total_f[0, 0].numpy(), total_f[0, 1].numpy())
    assert np.array_equal(flow_io.read_png(os.path.join(str(tmpdir), 'viz/00002.png')).transpose(2, 0, 1), got['viz'][0].cpu().numpy())
    assert np.load(os.path.join(str(tmpdir), 'mask/000.npy')).shape == (1, H, W)
