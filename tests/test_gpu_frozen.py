"""Training with fixed networks on the H100: the README's canonical step (cfg3 with MaskNet6 and Back2Future fixed)
against the oracle, its CUDA-graph replay, phase switches with checkpoints, a fixed DispResNet6's BatchNorm statistics
and the photometric loss's value-only paths at full size."""
import pytest
import torch
from tests import frozen_cases as FC, step_cases as SC
from tests.util import device_lib      # noqa: F401  (module fixture: the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]
DEV = torch.device('cuda:0')


def test_canonical_step_vs_oracle():
    FC.case_canonical_vs_oracle(DEV)


@pytest.mark.parametrize('size', [(2, 64, 128), (4, 256, 832)], ids=lambda s: 'b%d_%dx%d' % s)
def test_canonical_graph_replay(size):
    """capture() + three replay()s of the canonical step equal three eager steps bit for bit; replay() refuses after
    set_fixed()."""
    B, H, W = size
    SC.case_step_graph_vs_eager(DEV, 'cfg3', B, H, W, fixed=('mask', 'flow'))


def test_phase_switch_and_checkpoints():
    FC.case_phase_switch(DEV)


def test_fixed_dispnet_batchnorm_statistics():
    FC.case_fixed_dispnet_batchnorm(DEV)


def test_photo_value_only_full_size():
    FC.case_photo_value_only(DEV, B=4, H=256, W=832, NL=6)


def test_adam_ranges_on_device():
    FC.case_adam_ranges_fp64(DEV)
