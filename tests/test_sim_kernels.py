"""The product kernel sources, compiled by g++ against the CPU execution-model simulator
(tests/sim), checked against the oracle and the golden fixtures - so that indexing / reduction /
derivation bugs are caught in the GPU-less container.  The same cases run on the real H100 in
tests/test_gpu_parity.py."""
import os
import sys
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'sim'))


@pytest.fixture(scope='module', autouse=True)
def sim_lib():
    import build_sim
    from cc_b200 import _lib, pyramid
    prev = (_lib._lib, _lib._is_sim)
    _lib.use_library(build_sim.build())
    assert _lib.is_simulator()
    pyramid.clear()
    yield
    _lib._lib, _lib._is_sim = prev
    pyramid.clear()


from tests import kernel_cases as KC   # noqa: E402


@pytest.mark.parametrize('case', KC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(torch.device('cpu'))


from tests import net_cases as NC   # noqa: E402


@pytest.mark.parametrize('case', NC.NET_CASES, ids=lambda f: f.__name__)
def test_net_case(case):
    case(torch.device('cpu'))


from tests import step_cases as SC   # noqa: E402


@pytest.mark.parametrize('case', SC.STEP_CASES_SIM, ids=lambda f: f.__name__)
def test_step_case(case):
    case(torch.device('cpu'))


from tests import io_cases as IC   # noqa: E402


@pytest.mark.parametrize('case', IC.IO_CASES, ids=lambda f: f.__name__)
def test_io_case(case):
    case(torch.device('cpu'))


def test_metrics_other_sizes():
    IC.case_metrics_oracle_sizes(torch.device('cpu'), B=1, Hg=47, Wg=150, hp=32, wp=96)


from tests import helper_cases as HC   # noqa: E402


@pytest.mark.parametrize('case', HC.HELPER_CASES, ids=lambda f: f.__name__)
def test_helper_case(case):
    case(torch.device('cpu'))


from tests import eval_cases as EC   # noqa: E402


@pytest.mark.parametrize('case', [EC.case_eval_pose], ids=lambda f: f.__name__)      # depth / flow cores: GPU suite (CPU suite time)
def test_eval_case(case):
    case(torch.device('cpu'))
