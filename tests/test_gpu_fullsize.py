"""-m gpu: the production path (IMPL_AUTO: wgmma conv kernels + fused loss kernels) at the BASELINE.json
configurations (b4, 256x832, 6 levels) against the CPU oracle, per tensor; and against the step fixture frozen
from the reference's real train() body; the layer and loss audits of the timed step and the layer audit of the
evaluation forwards at B = 1.  See tests/fullsize_cases.py for the bars."""
import pytest
import torch
from tests import fullsize_cases as FC
from tests.util import device_lib      # noqa: F401  (module fixture: the sm_90a library; the noise-floor run needs TF32 off)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]


@pytest.fixture(scope='module', autouse=True)
def production_dispatch(device_lib):
    from cc_b200 import _lib, nn as cnn
    assert cnn.CONV_IMPL == _lib.IMPL_AUTO, 'full-size parity is defined on the production dispatch'


@pytest.mark.parametrize('cfg', ['cfg1', 'cfg2', 'cfg3'])
def test_step_fullsize_vs_cpu_oracle(cfg):
    FC.run(cfg, torch.device('cuda:0'), B=4, H=256, W=832)


def test_layer_audit_cfg3_second_step():
    """Every layer call of the timed step (cfg3 b4 256x832, committed weight cache) against fp64, element by element."""
    FC.audit_step(torch.device('cuda:0'))


def test_loss_audit_cfg3_second_step():
    """Every loss-layer call of the timed step (cfg3 b4 256x832, committed weight cache) against fp64, element by element."""
    FC.loss_audit_step(torch.device('cuda:0'))


@pytest.mark.parametrize('flownet', ['Back2Future', 'FlowNetC6'])
def test_layer_audit_eval_forwards(flownet):
    """Every layer call of evaluate._flow_nets (the four nets in eval mode, B = 1, 256x832) against fp64, element by
    element, with every BatchNorm's running statistics seeded far from the defaults (fullsize_cases.audit_eval_forwards)."""
    FC.audit_eval_forwards(torch.device('cuda:0'), flownet)


def test_step_vs_reference_fixture():
    """step_small.npz (reference train.py:454-509 on the reference modules) vs the CUDA step, per-parameter gradients."""
    rows = FC.golden_step_small(torch.device('cuda:0'))
    bad = []
    print()
    for name, err, floor, bar in rows:
        ok = err <= bar or (floor is not None and err <= FC.FLOOR_FACTOR * floor)
        if not ok and 'disp' in name and err <= FC.CHAOS_L2:
            ok = True          # DispResNet6 gradients are chaotic (fullsize_cases docstring): held to the chaos cap, floor printed beside
        print('   %-40s err %.2e  floor %s  bar %.0e %s' % (name, err, 'n/a' if floor is None else '%.2e' % floor, bar, '' if ok else 'FAIL'))
        if not ok:
            bad.append(name)
    assert not bad, 'tensors over their bar: %s' % bad
