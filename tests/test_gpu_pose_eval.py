"""Pose evaluation on the H100: the kernel cases of tests/pose_eval_cases.py on the sm_90a library, a KITTI-09-sized batch
of snippets against the oracle with bit-identical reruns, pose_eval_batch against the host path pose_snippet_errors on the
same uint8 frames and the same nets (PoseNetB6 at L = 5 in both rotation modes, PoseNet6, PoseExpNet at L = 3), and the
frames, stretch, resize, gather and errors chain inside a CUDA graph."""
import numpy as np
import pytest
import torch
from cc_b200 import evaluate as CE, models as CM, synth
from oracle import make3d_eval as OM, pose_eval as OP
from tests import pose_eval_cases as PC
from tests.util import assert_graph_replays, device_lib      # noqa: F401  (module fixture: the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]
DEV = torch.device('cuda:0')


@pytest.mark.parametrize('case', PC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(DEV)


def test_many_snippets_exact_reruns():
    """1600 snippets of L = 5 (KITTI 09's count) in both modes against the oracle; two more runs give the same bits."""
    PC.case_vs_oracle(DEV, S=1600, L=5, seed=9, reruns=2)


def _frames(N, H, W, seed):
    rs = np.random.RandomState(seed)
    base = rs.randint(20, 200, (H, W, 3))
    return np.stack([np.clip(base + rs.randint(-20, 21, (H, W, 3)) + 3 * i, 0, 255) for i in range(N)]).astype(np.uint8)


@pytest.mark.parametrize('name,L,mode', [('PoseNetB6', 5, 'euler'), ('PoseNetB6', 5, 'quat'), ('PoseNet6', 5, 'euler'),
                                         ('PoseExpNet', 3, 'euler')])
def test_pose_eval_batch_against_host_path(name, L, mode):
    """Every snippet of 9 frames of 70x150 (stretched and resized to 64x128 as the script's imresize does) through
    pose_eval_batch in one call, against pose_snippet_errors at batch 1 on the oracle's imresize of the same frames and
    the same net.  The net at batch S and at batch 1 sums in other orders (fp32 convolutions), so the bars are those of
    the host path's own test against the oracle net: final poses within 1e-4 relative (1e-6 absolute), ATE and RE
    within 1e-4 (1 + |v|).  Two calls give the same bits."""
    h, w = 64, 128
    frames = _frames(9, 70, 150, seed=31)
    snippets = CE._snippet_indices(len(frames), L)
    rs = np.random.RandomState(4)
    gt = np.stack([OP._compensated(PC.trajectory(rs, L)) for _ in snippets])
    net = synth.seeded_fill(getattr(CM, name)(nb_ref_imgs=L - 1), 60 + L).to(DEV)
    out, final = CE.pose_eval_batch(net, frames, snippets, gt, mode, h, w)
    out, final = out.cpu().numpy(), final.cpu().numpy()
    resized = [OM.imresize(f.astype(np.float32), (h, w)) for f in frames]
    for k, s in enumerate(snippets):
        ate, re, want = CE.pose_snippet_errors(net, [resized[i] for i in s], gt[k], mode, device=DEV)
        assert np.allclose(final[k], want, rtol=1e-4, atol=1e-6), (k, np.abs(final[k] - want).max())
        assert abs(out[k, 0] - ate) <= 1e-4 * (1 + abs(ate)) and abs(out[k, 1] - re) <= 1e-4 * (1 + abs(re)), (k, out[k], ate, re)
    out2, final2 = CE.pose_eval_batch(net, frames, snippets, gt, mode, h, w)
    assert np.array_equal(out2.cpu().numpy(), out) and np.array_equal(final2.cpu().numpy(), final)


def test_chain_in_cuda_graph():
    """Stretch, resize, normalisation, the snippet gather, a stand-in for the pose net (the same shapes) and the errors
    make no host round-trip: captured once, replayed on new frames and ground truth in the same buffers, equal to eager."""
    N, Hs, Ws, h, w, L = 7, 40, 90, 16, 48, 5
    snippets = torch.from_numpy(CE._snippet_indices(N, L)).to(DEV)

    def inputs(seed):
        rs = np.random.RandomState(seed)
        gt = np.stack([OP._compensated(PC.trajectory(rs, L)) for _ in range(len(snippets))])
        return [torch.from_numpy(_frames(N, Hs, Ws, seed)).to(DEV), torch.from_numpy(gt).to(DEV)]

    def stand_in(tgt, refs):
        return torch.stack([0.1 * torch.cat([(tgt - r).mean((2, 3)), (tgt * r).mean((2, 3))], 1) for r in refs], 1)

    def chain(frames, gt):
        return CE.pose_eval_batch(stand_in, frames, snippets, gt, 'euler', h, w)
    stand_in.eval = lambda: None
    eager = assert_graph_replays(chain, inputs(1), inputs(2))
    assert not torch.equal(eager[0][0], eager[1][0])
