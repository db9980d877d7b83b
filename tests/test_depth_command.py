"""The depth-evaluation command without a GPU: the oracle (oracle/eval_disp.py) against what the reference's own
test_disp.main() printed, computed and wrote (tests/golden/test_disp_small.npz), the 'hot' table, then cc_b200.test_disp
end to end with the kernels compiled by g++ against the CPU execution-model simulator (tests/sim): the fixture's runs,
worker counts, refusals and errors.  The same command runs on the H100 in tests/test_gpu_depth_command.py."""
import os
import numpy as np
import pytest
import torch
from cc_b200 import evaluate as CE, test_disp as TD
from tests import depth_command_cases as DC
from tests.util import sim_lib      # noqa: F401  (module fixture: the simulator library)

CPU = torch.device('cpu')


@pytest.fixture(scope='module')
def work(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('depth_command'))
    DC.write_work_dir(root)
    return root


@pytest.mark.parametrize('run', sorted(DC.RUNS))
def test_oracle_equals_reference(run, work):
    """The oracle on the fixture's trees prints the reference's stdout and computes its errors, predictions and PNGs."""
    d = DC.g()
    r = DC.oracle_run(work, run)
    assert r['stdout'] == str(d[run + '_stdout'])
    DC.check_errors(r['errors'], d[run + '_errors'], run, rtol=1e-6, atol=1e-7)
    if '--output-dir' in DC.RUNS[run]:
        assert np.allclose(r['predictions'], d[run + '_predictions'], rtol=1e-6, atol=0)
        DC.check_images(r['images'], DC.fixture_images(d, run), d[run + '_predictions'], run)


def test_hot_table():
    DC.case_hot_table()


def test_frameworks(work, capsys):
    """The frameworks' files, shifts and displacements: edges, the missing target, the zero-speed frame, camera 03."""
    kitti = CE.kitti_depth_framework(os.path.join(work, 'kitti'), DC.KITTI_LIST, 5)
    out = capsys.readouterr().out
    assert out == 'getting test metadata ... \n%s missing\n' % os.path.join(work, 'kitti', DC.KITTI_LIST[2])
    assert [os.path.relpath(s['path'], os.path.join(work, 'kitti')) for s in kitti] == DC.KITTI_LIST[:2] + DC.KITTI_LIST[3:]
    edge = kitti[1]                                         # frame 0: the frames -2 and -1 are the target itself
    assert edge['refs'][:2] == [edge['path']] * 2 and edge['displacements'][:2] == [0.0, 0.0]
    assert all(v > 0 for v in edge['displacements'][2:])
    assert not any(v > 0 for v in kitti[2]['displacements'])            # zero speed
    assert kitti[3]['cam'] == 3 and kitti[3]['displacements'][2:] == [0.0, 0.0]
    still = CE.stillbox_depth_framework(os.path.join(work, 'stillbox'), DC.STILLBOX_LIST, 3)
    assert len(still) == 4 and still[0]['displacements'][0] == 0 and still[0]['refs'][0] == still[0]['path']
    assert still[3]['displacements'][1] == 0 and still[3]['refs'][1] == still[3]['path']        # the scene's last frame
    assert CE.kitti_depth_framework(os.path.join(work, 'kitti'), DC.KITTI_LIST[:1], 0)[0]['refs'] == []


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('run', sorted(DC.RUNS))
def test_main(run, tmp_path, capsys):
    DC.case_main(CPU, tmp_path, capsys, run)


@pytest.mark.usefixtures('sim_lib')
def test_workers_identical(tmp_path):
    DC.case_workers_identical(CPU, tmp_path)


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('argv,match', [
    (['--gt-type', 'npy'], '--gt-type npy'),
    (['--gt-type', 'png'], '--gt-type png'),
    (['--no-resize', '--output-dir', 'out'], '--no-resize with --output-dir'),
])
def test_refusals(argv, match, tmp_path, capsys):
    """--gt-type npy|png and --no-resize with --output-dir on frames of two sizes: parser errors that name the flag."""
    with pytest.raises(SystemExit):
        DC.run_main(tmp_path, None, CPU, argv=DC.RUNS['kitti_sn'] + argv)
    assert match in capsys.readouterr().err
    assert not os.path.exists(os.path.join(str(tmp_path), 'out', 'predictions.npy'))


@pytest.mark.usefixtures('sim_lib')
def test_bad_frame_is_named(tmp_path):
    """A greyscale frame is refused, and the error names the file."""
    from PIL import Image
    DC.write_work_dir(str(tmp_path))
    name = os.path.join(str(tmp_path), 'kitti', DC.KITTI_LIST[0])
    Image.fromarray(np.asarray(Image.open(name))[:, :, 0]).save(name)
    cwd = os.getcwd()
    os.chdir(str(tmp_path))
    try:
        with pytest.raises(ValueError, match=DC.KITTI_LIST[0]):
            TD.main(DC.RUNS['kitti_sn'], device=CPU, workers=1)
    finally:
        os.chdir(cwd)


def test_min_depth_is_a_float():
    args = TD.build_parser().parse_args(['--pretrained-dispnet', 'x', '--min-depth', '0.5'])
    assert args.min_depth == 0.5 and TD.build_parser().parse_args(['--pretrained-dispnet', 'x']).min_depth == 1e-3


def test_bare_file_names_are_refused(tmp_path):
    with pytest.raises(ValueError, match='a.png'):
        CE.kitti_depth_framework(str(tmp_path), ['a.png'], 3)
    with pytest.raises(ValueError, match='a.png'):
        CE.stillbox_depth_framework(str(tmp_path), ['a.png'], 3)
