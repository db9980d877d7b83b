"""Motion segmentation evaluation without a GPU: the oracle mask_error against the numbers frozen from the reference's own
function, then ccb_mask_iou compiled by g++ against the CPU execution-model simulator (tests/sim) against the fixture,
the oracle and scipy's zoom.  The same cases run on the H100 in tests/test_gpu_mask_eval.py."""
import math
import numpy as np
import pytest
import torch
from cc_b200 import evaluate as CE
from oracle import evaluate_mask as OE
from tests import mask_eval_cases as MC
from tests.util import sim_lib      # noqa: F401  (module fixture: the simulator library)

CPU = torch.device('cpu')


@pytest.mark.parametrize('case', MC.fixture_cases(), ids=lambda c: c[0])
def test_oracle_mask_error_equals_reference(case):
    name, pred, obj, sem, out = case
    obj_before = obj.copy()
    got = OE.mask_error(obj, sem, pred)
    assert got == out.tolist(), (name, got, out)
    assert np.array_equal(obj, obj_before), 'the oracle must not relabel its argument'
    if name == 'nocar_bool':
        assert not any(got)


def test_oracle_mask_error_on_relabelled_ground_truth():
    """The script hands mask_error the array its previous call relabelled (0 / 1 / 255): the same numbers."""
    name, pred, obj, sem, out = MC.fixture_cases()[1]
    relabelled = np.where(sem != 26, 255, (obj != 0).astype(obj.dtype))
    assert OE.mask_error(relabelled, sem, pred) == out.tolist()


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('case', MC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(CPU)


@pytest.mark.usefixtures('sim_lib')
def test_fixture_kitti_size():
    """256x832 -> 375x1242 through the simulator (a thread per ground-truth pixel: about 20 s)."""
    MC.case_fixture_full(CPU)


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('sizes', MC.KITTI_AXES + [MC.ODD, (5, 7, 1, 1), (1, 1, 4, 6)], ids=lambda s: '%dx%d-%dx%d' % s)
def test_index_map_equals_scipy(sizes):
    """The KITTI map one axis at a time (the full 2-D map runs on the GPU; here it is covered by test_fixture_kitti_size)."""
    MC.case_index_map(CPU, sizes)


def test_mask_iou():
    avg, bg, fg = CE.mask_iou([6, 1, 1, 3, 1, 1])
    assert bg == 6 / 8 and fg == 3 / 5 and avg == (6 / 8 + 3 / 5) / 2
    summed = np.array([10, 2, 3, 0, 3, 2]) + np.array([5, 0, 0, 4, 0, 0])       # counts accumulate over a dataset
    assert CE.mask_iou(summed) == ((15 / 20 + 4 / 9) / 2, 15 / 20, 4 / 9)
    avg, bg, fg = CE.mask_iou(torch.tensor([4, 0, 0, 0, 0, 0]))                  # no moving pixel at all: 0/0
    assert bg == 1.0 and math.isnan(fg) and math.isnan(avg)
