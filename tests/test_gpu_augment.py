"""The reference's remaining data transforms (RandomRotate, NormalizeLocally, Scale) on the H100: the fixture cases of
tests/augment_cases.py and full-size runs against the numpy restatements of Pillow (tests/augment_oracle.py)."""
import pytest
import torch
from tests import augment_cases as AC
from tests.util import device_lib      # noqa: F401  (module fixture: the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]
DEV = torch.device('cuda:0')


@pytest.mark.parametrize('case', AC.AUGMENT_CASES, ids=lambda f: f.__name__)
def test_augment_case(case):
    case(DEV)


def test_rotate_train_transform_full_size():
    AC.case_rotate_fullsize(DEV)


def test_scale_kitti_full_size():
    AC.case_scale_fullsize(DEV)
