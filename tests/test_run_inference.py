"""run_inference without a GPU: the oracle (oracle/run_inference.py) against the arrays frozen from the reference's own
run_inference.main() (tests/golden/run_inference_small.npz), the bone table against OpenCV, then ccb_colorize,
ccb_prep_frames_inference and the command compiled by g++ against the CPU execution-model simulator (tests/sim).  The same
cases run on the H100 in tests/test_gpu_run_inference.py."""
import numpy as np
import pytest
import torch
from cc_b200 import evaluate as CE, run_inference as RI
from oracle import run_inference as ORI
from tests import run_inference_cases as RC
from tests.util import sim_lib      # noqa: F401  (module fixture: the simulator library)

CPU = torch.device('cpu')


@pytest.mark.parametrize('run', ['glob', 'list', 'noresize_depth'])
def test_oracle_equals_reference(run):
    """The oracle's images of the fixture's disparity maps equal the reference's imsave arrays."""
    d = RC.g()
    argv = RC.RUNS[run]
    kinds = [k for k in ('disp', 'depth') if '--output-' + k in argv]
    names = [str(n) for n in d[run + '_saved_names']]
    for k in range(len(names)):
        disp = torch.from_numpy(d['%s_disp_%d' % (run, k // len(kinds))][0])
        img = ORI.images(disp)[('disp', 'depth').index(kinds[k % len(kinds)])]
        assert np.array_equal(img, d['%s_saved_%d' % (run, k)].transpose(1, 2, 0)), (run, names[k])


def test_oracle_net_equals_reference():
    """The oracle's DispNetS forward and net input, on the fixture's photos and checkpoint, give the reference's
    disparity maps."""
    d = RC.g()
    p = RC.checkpoint()['state_dict']
    for k, name in enumerate(('a.png', 'b.png')):              # the 'glob' run's first two photos, in listdir order
        h, w, seed = RC.PHOTOS[name]
        x = ORI.net_input(RC.photo(h, w, seed), *RC.SIZE)
        with torch.no_grad():
            got = ORI.dispnets_forward(p, x)
        names = [str(n) for n in d['glob_saved_names']]
        i = [n.split('_disp')[0] for n in names[::2]].index(name[0])
        want = d['glob_disp_%d' % i]
        assert np.abs(got.numpy() - want).max() <= 1e-5 * np.abs(want).max(), name


def test_bone_against_opencv():
    """Bone at 256 points within 2 levels of OpenCV's COLORMAP_BONE (an independent implementation of the same map)."""
    cv2 = pytest.importorskip('cv2', reason='OpenCV is not installed: the bone table is not checked against it')
    ramp = np.arange(256, dtype=np.uint8).reshape(1, 256)
    cv = cv2.applyColorMap(ramp, cv2.COLORMAP_BONE)[0, :, ::-1].astype(np.int32)
    table = CE.colormap_table('bone').astype(np.int32)
    ours = table[np.minimum((np.arange(256) / 255.0 * 10000).astype(int), 9999)]
    assert np.abs(ours - cv).max() <= 2, np.abs(ours - cv).max()


def test_must_output_one_value(capsys, tmp_path):
    assert RI.main(['--pretrained', 'missing.pth', '--output-dir', str(tmp_path / 'o')]) is None
    assert capsys.readouterr().out == 'You must at least output one value !\n'
    assert not (tmp_path / 'o').exists()


def test_unknown_colormap():
    with pytest.raises(ValueError, match='magma'):
        CE.colorize(torch.zeros(1, 2, 2), 'magma')


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('case', RC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(CPU)


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('run', sorted(RC.RUNS))
def test_main(run, tmp_path, capsys):
    RC.case_main(CPU, tmp_path, capsys, run)


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('mode', ['RGBA', 'L'])
def test_refusal(mode, tmp_path, capsys):
    RC.case_refusal(CPU, tmp_path, capsys, mode)
