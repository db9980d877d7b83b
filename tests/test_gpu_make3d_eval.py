"""Make3D evaluation on the H100: the kernel cases of tests/make3d_eval_cases.py and the workspace rows on the sm_90a
library, Make3D-sized crops byte-exact with bit-identical reruns, make3d_eval_batch against the host path and the oracle
net, and the stretch, resize, normalisation, zoom and errors chain inside a CUDA graph."""
import numpy as np
import pytest
import torch
from cc_b200 import evaluate as CE
from tests import make3d_eval_cases as MC, workspace_cases as WC
from tests.test_make3d_eval import ROWS
from tests.util import assert_graph_replays, device_lib      # noqa: F401  (module fixture: the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]
DEV = torch.device('cuda:0')


@pytest.mark.parametrize('case', MC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(DEV)


@pytest.mark.parametrize('row', ROWS, ids=[r.entry for r in ROWS])
def test_workspace_row(row, monkeypatch):
    WC.check_row(DEV, row, monkeypatch)


def test_real_size_exact_and_repeatable():
    """Four 852x1704 crops -> 256x256 byte-exact against the oracle; two more runs give the same bits."""
    MC.case_real_size(DEV, B=4, reruns=2)
    MC.case_errors_vs_oracle(DEV, B=4, seed=80, reruns=2)


@pytest.mark.parametrize('name', ['DispResNet6', 'DispNetS6'])
def test_make3d_eval_batch(name):
    MC.case_eval_batch(DEV, name)


def test_chain_in_cuda_graph():
    """Stretch, resize, normalisation, the net-free zoom and the errors make no host round-trip: captured once, replayed
    on new inputs in the same buffers."""
    B, Hs, Ws, h, w = 2, 60, 90, 32, 48

    def inputs(seed):
        rs = np.random.RandomState(seed)
        crops = np.stack([rs.randint(10 * b, 200 + 20 * b, (Hs, Ws, 3)) for b in range(B)]).astype(np.uint8)
        gt = np.stack([MC.error_inputs(rs)[0] for _ in range(B)])
        return [torch.from_numpy(crops).to(DEV), torch.from_numpy(gt).to(DEV)]

    def chain(crops, gt):
        x = CE.make3d_frames(crops, h, w)
        disp = 0.05 + 0.02 * (x[:, 0] + x[:, 1] * x[:, 2])          # a stand-in for the net's disparity, same shape
        pred = CE.spline_zoom(1 / disp, 21, 305, 1e-3, 70.0)
        return CE.make3d_depth_errors(gt, pred, 1e-3, 70.0)
    eager = assert_graph_replays(chain, inputs(1), inputs(2))
    assert not torch.equal(eager[0], eager[1])
