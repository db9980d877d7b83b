"""Motion segmentation evaluation on the H100: the kernel cases of tests/mask_eval_cases.py on the sm_90a library, the
KITTI sizes at B = 1 and B = 4 with bit-identical reruns, mask_sample_errors with all four nets against the oracle
evaluation, and motion_mask_counts inside a CUDA graph."""
import pytest
import torch
from cc_b200 import evaluate as CE
from tests import mask_eval_cases as MC
from tests.util import assert_graph_replays, device_lib      # noqa: F401  (module fixture: the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]
DEV = torch.device('cuda:0')


@pytest.mark.parametrize('case', MC.ALL_CASES + [MC.case_fixture_full], ids=lambda f: f.__name__)
def test_case(case):
    case(DEV)


@pytest.mark.parametrize('sizes', [MC.KITTI, MC.ODD] + MC.KITTI_AXES, ids=lambda s: '%dx%d-%dx%d' % s)
def test_index_map_equals_scipy(sizes):
    MC.case_index_map(DEV, sizes)


@pytest.mark.parametrize('B', [1, 4])
def test_kitti_size_exact_and_repeatable(B):
    """256x832 -> 375x1242: masks and counts equal the CPU oracle's exactly, per sample, and two more runs give the same bits."""
    MC.case_random_vs_oracle(DEV, B=B, sizes=MC.KITTI, THRESH=0.6, seed=31 + B, reruns=2)


@pytest.mark.parametrize('flownet', sorted(MC.SAMPLE_CASES))
def test_mask_sample_errors_vs_oracle(flownet):
    MC.case_sample_errors(DEV, flownet)


def test_motion_mask_counts_in_cuda_graph():
    """The call makes no host round-trip: captured once, replayed on new inputs in the same buffers."""
    first = [t.to(DEV) for t in MC.random_sample(2, 64, 128, 96, 200, seed=51, flow_scale=[1.0, 2.0])]
    second = [t.to(DEV) for t in MC.random_sample(2, 64, 128, 96, 200, seed=52, flow_scale=[2.0, 1.0])]
    eager = assert_graph_replays(lambda *ins: CE.motion_mask_counts(*ins, THRESH=0.6, want_masks=True), first, second)
    assert not torch.equal(eager[0][0], eager[1][0])
