"""Make3D evaluation without a GPU: the oracle (oracle/make3d_eval.py) against the numbers frozen from the reference's own
test_framework and compute_errors (tests/golden/make3d_eval_small.npz), make3d_files / load_make3d against the frozen
framework on the same tree, then ccb_bytescale_u8 and ccb_make3d_depth_errors compiled by g++ against the CPU
execution-model simulator (tests/sim) against the fixture and the oracle, and their workspace contract.  The same kernel
cases run on the H100 in tests/test_gpu_make3d_eval.py."""
import numpy as np
import pytest
import torch
from cc_b200 import evaluate as CE
from oracle import make3d_eval as OM
from tests import make3d_eval_cases as MC, workspace_cases as WC
from tests.util import sim_lib      # noqa: F401  (module fixture: the simulator library)

CPU = torch.device('cpu')


@pytest.mark.parametrize('case', MC.stretch_cases(), ids=lambda c: c['name'])
def test_oracle_stretch_equals_reference(case):
    c = case
    h, w = c['size']
    if c['stretched'] is not None:
        assert np.array_equal(OM.bytescale(c['crop'].astype(np.float32)), c['stretched'])
        assert np.array_equal(OM.imresize(c['crop'].astype(np.float32), (h, w)), c['out'])
    else:
        assert np.array_equal(c['out'], c['crop'])
    assert np.array_equal(OM.net_input(c['crop'], h, w, c['resize']), OM.net_input(c['out'], *c['out'].shape[:2], False))


def test_oracle_stretch_rounds_each_step():
    """The pinned tie: (101 - 0) * float32(255 / 202) = 127.49999237 in float32, + 0.5 -> 127; exact arithmetic gives 128."""
    x = np.zeros((4, 5, 3), np.float32)
    x[0, 0, 0], x[1, 1, 1] = 202, 101
    assert OM.bytescale(x)[1, 1, 1] == 127 and OM.bytescale(x)[0, 0, 0] == 255


@pytest.mark.parametrize('case', MC.error_cases(), ids=lambda c: c['name'])
def test_oracle_errors_equal_reference(case):
    c = case
    got = OM.sample_errors(c['gt'], c['pred'], c['lo'], c['hi'])
    assert np.array_equal(got, c['out'], equal_nan=True), (c['name'], got, c['out'])


def test_summary_is_the_printed_row():
    outs = [c['out'] for c in MC.error_cases() if not np.isnan(c['out'][1]).any()]
    got = CE.depth_summary(np.stack(outs))
    assert got.dtype == np.float32 and not got[0].any()
    assert np.array_equal(got[1], MC.golden(MC.FIXTURE)['summary'])


def test_make3d_files_and_samples(tmp_path):
    """The same tree rebuilt: the sorted lists without element 61, paired by index, and the samples at the frozen indices."""
    want = MC.framework()
    MC.write_make3d_tree(str(tmp_path))
    img_files, depth_files = CE.make3d_files(str(tmp_path))
    assert len(img_files) == len(depth_files) == want['length']
    assert [f.split('/')[-1] for f in img_files] == want['img_files']
    assert [f.split('/')[-1] for f in depth_files] == want['depth_files']
    for i, s in want['samples'].items():
        got = CE.load_make3d(img_files[i], depth_files[i], 1e-3, 70.0)
        assert got['tgt'].dtype == np.uint8 and np.array_equal(got['tgt'], s['tgt']), i
        assert got['gt_depth'].dtype == np.float64 and np.array_equal(got['gt_depth'], s['gt_depth']), i
        assert np.array_equal(got['mask'], s['mask']), i
    assert want['samples'][61]['mask'].any() and not want['samples'][61]['mask'].all()


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('case', MC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(CPU)


def _bytescale_row(dev):
    CE.make3d_frames((WC._rand(dev, 2, 9, 13, 3, seed=60, lo=20, hi=200)).to(torch.uint8), 6, 17)


def _make3d_errors_row(dev):
    CE.make3d_depth_errors(WC._rand(dev, 2, 12, 20, seed=61, lo=0.5, hi=90).double(), WC._rand(dev, 2, 12, 20, seed=62, lo=0.5, hi=70))


ROWS = [WC.Row('bytescale_u8', 4, 5, [6], _bytescale_row, ('ccb_bytescale_u8_workspace_bytes', (2, 0, 13))),
        WC.Row('make3d_depth_errors', 7, 8, [9], _make3d_errors_row, ('ccb_make3d_depth_errors_workspace_bytes', (2, 12, 0)))]


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('row', ROWS, ids=[r.entry for r in ROWS])
def test_workspace_row(row, monkeypatch):
    WC.check_row(CPU, row, monkeypatch)
