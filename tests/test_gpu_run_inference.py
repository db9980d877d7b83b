"""run_inference on the H100: the cases of tests/run_inference_cases.py and the command on the sm_90a library,
KITTI-size frames through infer() with DispNetS and DispResNet6 against the oracle's fp64 nets, and the colorize calls
inside a CUDA graph."""
import numpy as np
import pytest
import torch
from cc_b200 import evaluate as CE
from tests import run_inference_cases as RC
from tests.util import assert_graph_replays, device_lib      # noqa: F401  (module fixture: the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]
DEV = torch.device('cuda:0')


@pytest.mark.parametrize('case', RC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(DEV)


@pytest.mark.parametrize('run', sorted(RC.RUNS))
def test_main(run, tmp_path, capsys):
    RC.case_main(DEV, tmp_path, capsys, run)


@pytest.mark.parametrize('mode', ['RGBA', 'L'])
def test_refusal(mode, tmp_path, capsys):
    RC.case_refusal(DEV, tmp_path, capsys, mode)


@pytest.mark.parametrize('target', [(128, 416), (256, 832)])
@pytest.mark.parametrize('name', ['DispNetS', 'DispResNet6'])
def test_kitti_size_vs_fp64_oracle(name, target):
    RC.kitti_case(DEV, name, target=target, n=2 if target == (128, 416) else 1)


def test_colorize_in_cuda_graph():
    """Both colorize calls of a batch make no host round-trip: captured once, replayed on new maps in the same buffers."""
    def maps(seed):
        rs = np.random.RandomState(seed)
        return [torch.from_numpy(rs.uniform(0.01, 10, (3, 48, 80)).astype(np.float32)).to(DEV)]

    def chain(disp):
        return CE.colorize(disp, 'bone'), CE.colorize(disp, 'rainbow', 10, invert=True)
    eager = assert_graph_replays(chain, maps(1), maps(2))
    assert not torch.equal(eager[0][0], eager[1][0]) and not torch.equal(eager[0][1], eager[1][1])
