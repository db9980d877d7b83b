"""KITTI-2015 flow evaluation on the H100: the kernel cases of tests/flow_eval_cases.py on the sm_90a library, a batch of
samples against each sample alone with bit-identical reruns, flow_eval_batch against the host path flow_sample_errors on
the same uint8 frames and the same nets (Back2Future and FlowNetC6), back2future_eval_batch against the oracle, and the
frames, nets and kernel chain inside a CUDA graph."""
import numpy as np
import pytest
import torch
from cc_b200 import evaluate as CE, models as CM, synth
from oracle import flow_eval as OF, make3d_eval as OM
from tests import flow_eval_cases as FC
from tests.util import assert_graph_replays, device_lib      # noqa: F401  (module fixture: the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]
DEV = torch.device('cuda:0')


@pytest.mark.parametrize('case', FC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(DEV)


def test_batch_rows_equal_samples_alone():
    """16 samples in one call: each row equals its sample alone bit for bit and the oracle within the bar; reruns agree."""
    FC.case_vs_oracle(DEV, B=16, seed=40, reruns=2)


def _frames(B, F, H, W, seed):
    rs = np.random.RandomState(seed)
    base = rs.randint(20, 200, (B, 1, H, W, 3))
    return np.clip(base + rs.randint(-20, 21, (B, F, H, W, 3)), 0, 255).astype(np.uint8)


def _nets(flownet, seed=70):
    nets = [synth.seeded_fill(CM.DispResNet6(), seed), synth.seeded_fill(CM.PoseNetB6(nb_ref_imgs=4), seed + 1),
            synth.seeded_fill(CM.MaskNet6(nb_ref_imgs=4), seed + 2),
            synth.seeded_fill(CM.Back2Future(nlevels=6) if flownet == 'Back2Future' else CM.FlowNetC6(nlevels=6), seed + 3)]
    return [n.to(DEV).eval() for n in nets]


def _ground_truth(B, Hs, Ws, seed):
    rs = np.random.RandomState(seed)
    gt = np.stack([FC.gt_flow(rs, Hs, Ws) * np.float32(0.05) for _ in range(B)]).astype(np.float32)
    gt[:, 2] = np.round(gt[:, 2] * 20)
    obj = np.stack([FC.obj_ids(rs, Hs, Ws) for _ in range(B)]).astype(np.float32)
    return gt, obj


@pytest.mark.parametrize('flownet', ['Back2Future', 'FlowNetC6'])
def test_flow_eval_batch_against_host_path(flownet):
    """3 samples of 80x200 frames (stretched and resized to 64x192 as Scale does) through flow_eval_batch in one call,
    against flow_sample_errors at batch 1 on the oracle's imresize of the same frames and the same nets.  The nets at
    batch 3 and at batch 1 sum in other orders (fp32 convolutions), which moves flows by ~1e-5 relative and can flip a
    census pixel or an outlier near its threshold, so the bars are 1e-3 (1 + |v|) for EPE and 5e-3 for Fl (a few pixels
    of 16000).  Two calls give the same bits."""
    B, Hs, Ws, h, w = 3, 80, 200, 64, 192
    frames = _frames(B, 5, Hs, Ws, seed=8)
    K = np.tile(np.array([[120.0, 0, 100.0], [0, 120.0, 40.0], [0, 0, 1]], np.float32), (B, 1, 1))
    gt, obj = _ground_truth(B, Hs, Ws, seed=9)
    nets = _nets(flownet)
    out = CE.flow_eval_batch(*nets, frames, K, gt, obj, h=h, w=w).cpu().numpy()
    Ks, Kinv = CE.flow_intrinsics(K, Hs, Ws, h, w, DEV)
    for k in range(B):
        x = [torch.from_numpy(OM.imresize(f.astype(np.float32), (h, w))) for f in frames[k]]
        x = [((t.permute(2, 0, 1)[None].float() / 255 - 0.5) / 0.5).to(DEV) for t in x]
        errs, _ = CE.flow_sample_errors(*nets, x[0], x[1:], Ks[k:k + 1], Kinv[k:k + 1], torch.from_numpy(gt[k:k + 1]).to(DEV),
                                        torch.from_numpy(obj[k:k + 1]).to(DEV))
        errs = np.array(errs)
        for j in range(8):
            bar = 5e-3 if j % 4 == 3 else 1e-3 * (1 + abs(errs[j]))
            assert abs(out[k, j] - errs[j]) <= bar, (k, j, out[k], errs)
    assert np.array_equal(CE.flow_eval_batch(*nets, frames, K, gt, obj, h=h, w=w).cpu().numpy(), out)


def test_back2future_eval_batch_against_oracle():
    """back2future_eval_batch's rows against the oracle's compute_all_epes(gt, fwd, fwd, 1 - obj) of the same forward
    flows, sample by sample."""
    B, Hs, Ws, h, w = 4, 80, 200, 64, 192
    frames = _frames(B, 5, Hs, Ws, seed=12)
    gt, obj = _ground_truth(B, Hs, Ws, seed=13)
    net = _nets('Back2Future')[3]
    out = CE.back2future_eval_batch(net, frames, gt, obj, h, w).cpu().numpy()
    x = CE._flow_frames(frames, h, w)
    fwd = net(x[0], x[2:4])[0].cpu()
    for k in range(B):
        want = OF.back2future_errors(fwd[k:k + 1], torch.from_numpy(gt[k:k + 1]), torch.from_numpy(obj[k:k + 1]))
        FC._close(out[k], want, FC.BAR, k)


def test_chain_in_cuda_graph():
    """Stretch, resize, normalisation, the four nets at batch 2 and the kernel make no host round-trip: captured once,
    replayed on new frames, ground truth and object maps in the same buffers, equal to eager."""
    B, Hs, Ws, h, w = 2, 70, 150, 64, 128
    nets = _nets('Back2Future', seed=80)
    K = CE.flow_intrinsics(np.tile(np.array([[100.0, 0, 75.0], [0, 100.0, 35.0], [0, 0, 1]], np.float32), (B, 1, 1)),
                           Hs, Ws, h, w, DEV)

    def inputs(seed):
        gt, obj = _ground_truth(B, Hs, Ws, seed + 1)
        return [torch.from_numpy(a).to(DEV) for a in (_frames(B, 5, Hs, Ws, seed), gt, obj)]

    def chain(frames, gt, obj):
        return CE.flow_eval_batch(*nets, frames, K, gt, obj, h=h, w=w, want_mask=True)
    eager = assert_graph_replays(chain, inputs(1), inputs(2))
    assert not torch.equal(eager[0][0], eager[1][0])
