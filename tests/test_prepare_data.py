"""Training-data preparation (cc_b200.prepare_train_data) without a GPU, the kernels on the CPU simulator build: the
oracle and the module against what the reference's prepare_train_data.py wrote (tests/golden/prepare_small.npz) for a
KITTI raw tree (by speed and with a static-frames list, velodyne depth) and a Cityscapes tree; the same dump for any
--num-threads; the argument errors; and cc_b200.train's samples on the written dump."""
import multiprocessing
import os
import shutil
import numpy as np
import pytest
import torch

from cc_b200 import prepare_train_data as PT, train as T
from oracle import prepare as OP
from tests import prepare_cases as PC, prepare_data_checks as PD
from tests.util import sim_lib      # noqa: F401  (module fixture: the kernels on the CPU simulator)

CPU = torch.device('cpu')


def _in(d, fn):
    cwd = os.getcwd()
    os.chdir(d)
    try:
        return fn()
    finally:
        os.chdir(cwd)


def oracle_run(d, run):
    a = PC.RUNS[run]
    opt = lambda k: a[a.index(k) + 1] if k in a else None            # noqa: E731
    return _in(d, lambda: OP.prepare('raw', a[a.index('--dataset-format') + 1], 'dump', int(opt('--height')),
                                     int(opt('--width')), opt('--static-frames'), '--with-gt' in a, opt('--test-scenes')))


def product_run(d, run, device, extra=(), presplit=False, monkeypatch=None):
    """main() on the run's arguments in d; presplit: with the split left out (every depth map stays)."""
    if presplit:
        monkeypatch.setattr(PT, 'split', lambda root: ([n for n in os.listdir(root)
                                                        if os.path.isdir(os.path.join(root, n))], [], []))
    return _in(d, lambda: PT.main(list(PC.RUNS[run]) + list(extra), device=device))


@pytest.mark.parametrize('run', list(PC.RUNS))
def test_oracle_equals_fixture(tmp_path, run):
    PD.check_fixture_consistent(run)
    d = PD.write_run_dir(str(tmp_path), run)
    rec = oracle_run(d, run)
    PD.check_oracle_record(run, rec, os.path.join(d, 'dump'))


@pytest.mark.parametrize('run', list(PC.RUNS))
def test_main_equals_fixture(tmp_path, monkeypatch, sim_lib, run):       # noqa: F811
    d = PD.write_run_dir(str(tmp_path), run)
    out = product_run(d, run, CPU, presplit=True, monkeypatch=monkeypatch)
    dump = os.path.join(d, 'dump')
    PD.check_dump(run, dump, out['order'], presplit=True)
    monkeypatch.undo()
    order, train, val = PT.split(dump)
    assert (train, val) == PD.split_rule(order)
    PD.check_dump(run, dump, order)
    assert not multiprocessing.active_children()


def test_num_threads_same_dump(tmp_path, sim_lib):        # noqa: F811
    """--num-threads 1 and 3 write the same files, byte for byte; every worker is joined."""
    got = {}
    for n in (1, 3):
        d = PD.write_run_dir(str(tmp_path / ('t%d' % n)), 'kitti_static')
        out = product_run(d, 'kitti_static', CPU, ['--num-threads', str(n)])
        PD.check_dump('kitti_static', os.path.join(d, 'dump'), out['order'])
        got[n] = PD.hashes(os.path.join(d, 'dump'))
        assert not multiprocessing.active_children()
    assert got[1] == got[3]


def test_argument_errors(tmp_path, capsys, sim_lib):        # noqa: F811
    d = PD.write_run_dir(str(tmp_path), 'kitti_static')
    a = list(PC.RUNS['kitti_static'])
    k = a.index('--test-scenes')
    for argv, needle in ((a[:k] + a[k + 2:], '--test-scenes is required'),
                         (a + ['--height', '0'], '--height and --width must be positive'),
                         (a + ['--width', '-4'], '--height and --width must be positive'),
                         (a + ['--num-threads', '0'], '--num-threads must be at least 1')):
        with pytest.raises(SystemExit):
            _in(d, lambda: PT.main(argv, device=CPU))
        assert needle in capsys.readouterr().err
    shutil.rmtree(os.path.join(d, 'raw', '2011_09_28'))
    with pytest.raises(FileNotFoundError, match='KITTI date folder not found: raw/2011_09_28'):
        _in(d, lambda: PT.main(a, device=CPU))
    os.makedirs(os.path.join(d, 'raw', '2011_09_28'))
    missing = os.path.join('raw', '2011_09_30', '2011_09_30_drive_0005_sync', 'velodyne_points', 'data', '0000000004.bin')
    os.remove(os.path.join(d, missing))
    with pytest.raises(FileNotFoundError, match='velodyne file not found: ' + missing):
        _in(d, lambda: PT.main(a + ['--num-threads', '2'], device=CPU))
    assert not multiprocessing.active_children()
    _in(d, lambda: PT.main([x for x in a if x != '--with-gt'], device=CPU))      # without --with-gt no sweep is read


def test_train_samples_on_dump(tmp_path, sim_lib):        # noqa: F811
    """cc_b200.train's sequence_samples (train and val) and validation_samples on the module's dump equal those on the
    oracle's dump."""
    d = PD.write_run_dir(str(tmp_path / 'product'), 'kitti_static')
    product_run(d, 'kitti_static', CPU)
    o = PD.write_run_dir(str(tmp_path / 'oracle'), 'kitti_static')
    oracle_run(o, 'kitti_static')
    roots = [os.path.join(x, 'dump') for x in (d, o)]
    rel = lambda root, paths: [os.path.relpath(p, root) for p in paths]        # noqa: E731
    for train in (True, False):
        got, want = (T.sequence_samples(r, 3, train=train) for r in roots)
        assert len(got) > 0 and [rel(roots[0], s['frames']) for s in got] == [rel(roots[1], s['frames']) for s in want]
        assert all(np.array_equal(a['K'], b['K']) for a, b in zip(got, want))
    got, want = (T.validation_samples(r) for r in roots)
    assert len(got) > 0 and [rel(roots[0], p) for p in got] == [rel(roots[1], p) for p in want]
