"""The workspace contract of include/ccb200.h on the H100: the cases of tests/workspace_cases.py on the sm_90a library.
Every short buffer is refused on the host before any launch, so no kernel ever sees one."""
import pytest
import torch
from tests import workspace_cases as WC
from tests.util import device_lib      # noqa: F401  (module fixture: the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]
DEV = torch.device('cuda:0')


@pytest.mark.parametrize('row', WC.ROWS, ids=WC.IDS)
def test_row(row, monkeypatch):
    WC.check_row(DEV, row, monkeypatch)


def test_null_where_nothing_is_needed():
    WC.check_zero_need(DEV)
    torch.cuda.synchronize()
