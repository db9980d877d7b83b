"""KITTI-2015 flow submission on the H100: the kernel cases of tests/flow_submit_cases.py on the sm_90a library, the KITTI
size at B = 1 and 4 equal to the oracle bit for bit and over reruns, flow_submission_sample with all four nets, and
ccb_flow_submit + ccb_flow_color inside a CUDA graph."""
import pytest
import torch
from cc_b200 import evaluate as CE
from tests import flow_submit_cases as SC
from tests.util import assert_graph_replays, device_lib      # noqa: F401  (module fixture: the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]
DEV = torch.device('cuda:0')


@pytest.mark.parametrize('case', SC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(DEV)


@pytest.mark.parametrize('B', [1, 4])
def test_kitti_size_exact_and_repeatable(B):
    SC.case_random_submit(DEV, B=B, sizes=SC.KITTI, seed=31 + B, reruns=2)


@pytest.mark.parametrize('flownet', sorted(SC.SAMPLE_NETS))
def test_flow_submission_sample_vs_oracle(flownet, tmp_path):
    SC.case_submission_sample(DEV, flownet, tmp_path)


def test_submit_and_colors_in_cuda_graph():
    """No host round-trip: flow_submission + flow_colors captured once and replayed on new inputs in the same buffers."""
    first = [t.to(DEV) for t in SC.random_submit_inputs(2, 64, 128, seed=51)]
    second = [t.to(DEV) for t in SC.random_submit_inputs(2, 64, 128, seed=52)]

    def run(*ins):
        out = CE.flow_submission(*ins, 96, 200, 0.01, want_full=True)
        out['viz'] = CE.flow_colors(out['full'])
        return out

    eager = assert_graph_replays(run, first, second)
    assert not torch.equal(eager[0]['png'], eager[1]['png'])
