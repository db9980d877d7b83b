"""-m gpu: the production path (IMPL_AUTO: wgmma conv kernels + fused loss kernels) at the BASELINE.json
configurations (b4, 256x832, 6 levels) against the CPU oracle, per tensor; and against the step fixture frozen
from the reference's real train() body.  See tests/fullsize_cases.py for the bars."""
import pytest
import torch
from tests import fullsize_cases as FC

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def cuda_lib():
    from cc_b200 import _lib, pyramid, nn as cnn
    _lib._lib = None
    assert not _lib.is_simulator(), 'GPU tests must run on the sm_90a library'
    assert cnn.CONV_IMPL == _lib.IMPL_AUTO, 'full-size parity is defined on the production dispatch'
    pyramid.clear()
    torch.backends.cudnn.allow_tf32 = False       # the noise-floor run (oracle on the GPU) must be fp32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


@pytest.mark.parametrize('cfg', ['cfg1', 'cfg2', 'cfg3'])
def test_step_fullsize_vs_cpu_oracle(cfg):
    FC.run(cfg, torch.device('cuda:0'), B=4, H=256, W=832)


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
