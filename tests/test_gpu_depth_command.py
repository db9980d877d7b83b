"""The depth-evaluation command on the H100: the fixture's runs and the worker counts of tests/depth_command_cases.py on
the sm_90a library, and KITTI-size trees (1242x375 and 1241x376 frames, 100k-point sweeps, a missing reference frame)
against fp64 oracle nets for DispResNet6 alone and with PoseNetB6 and PoseExpNet, with bit-identical reruns."""
import pytest
import torch
from tests import depth_command_cases as DC
from tests.util import device_lib      # noqa: F401  (module fixture: the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]
DEV = torch.device('cuda:0')


def test_hot_table():
    DC.case_hot_table(DEV)


@pytest.mark.parametrize('run', sorted(DC.RUNS))
def test_main(run, tmp_path, capsys):
    DC.case_main(DEV, tmp_path, capsys, run)


def test_workers_identical(tmp_path):
    DC.case_workers_identical(DEV, tmp_path)


@pytest.mark.parametrize('posenet', [None, 'PoseNetB6', 'PoseExpNet'])
def test_kitti_size_vs_fp64_oracle(posenet, tmp_path):
    DC.kitti_size_case(DEV, tmp_path, posenet)
