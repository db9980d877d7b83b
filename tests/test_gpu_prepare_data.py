"""Training-data preparation (cc_b200.prepare_train_data) on the H100: the fixture parity of tests/test_prepare_data.py
on the sm_90a build, a KITTI-size case against the oracle (1242x375 and 1241x376 frames resized to 832x256, sweeps of
about 100k points with duplicate pixels: frames byte-equal, depth bit-equal), and a prepared dump trained on by
cc_b200.train.main."""
import io
import multiprocessing
import os
import numpy as np
import pytest
import torch
from PIL import Image

from cc_b200 import prepare_train_data as PT, train as T
from oracle import prepare as OP
from tests import prepare_cases as PC, prepare_data_checks as PD
from tests.test_prepare_data import product_run, _in
from tests.util import device_lib      # noqa: F401  (module fixture: the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]
DEV = torch.device('cuda:0')


@pytest.mark.parametrize('run', list(PC.RUNS))
def test_main_equals_fixture(tmp_path, monkeypatch, run):
    d = PD.write_run_dir(str(tmp_path), run)
    out = product_run(d, run, DEV, ['--num-threads', '4'], presplit=True, monkeypatch=monkeypatch)
    dump = os.path.join(d, 'dump')
    PD.check_dump(run, dump, out['order'], presplit=True)
    monkeypatch.undo()
    order, _, _ = PT.split(dump)
    PD.check_dump(run, dump, order)
    assert not multiprocessing.active_children()


def test_kitti_size_against_oracle(tmp_path, monkeypatch):
    """Two drives of KITTI's frame sizes, both cameras, --with-gt at 256x832 with a static-frames list: each jpg is
    Pillow's encoding of the oracle's uint8 frame, each .npy the oracle's float32 depth bit for bit (the split is left
    out, so that every depth map stays)."""
    d = PC.write_kitti_tree(str(tmp_path), drives=PC.kitti_size_drives(frames=4), out_hw=(256, 832), points=100000)
    PC.write_files(d, {'static.txt': PC.STATIC, 'test_scenes.txt': PC.TEST_SCENES})
    argv = ['raw', '--dataset-format', 'kitti', '--dump-root', 'dump', '--with-gt', '--height', '256', '--width', '832',
            '--num-threads', '4', '--test-scenes', 'test_scenes.txt', '--static-frames', 'static.txt']
    monkeypatch.setattr(PT, 'split', lambda root: ([], [], []))
    _in(d, lambda: PT.main(argv, device=DEV))
    rec = _in(d, lambda: OP.prepare('raw', 'kitti', 'oracle_dump', 256, 832, 'static.txt', True, 'test_scenes.txt'))
    dump = os.path.join(d, 'dump')
    assert len(rec['frames']) >= 12 and sorted(rec['depth']) == sorted(f for f in PC.dump_files(dump) if f.endswith('.npy'))
    assert sorted(rec['frames']) == sorted(f for f in PC.dump_files(dump) if f.endswith('.jpg'))
    filled = 0
    for k, a in rec['frames'].items():
        b = io.BytesIO()
        Image.fromarray(a).save(b, format='JPEG')
        with open(os.path.join(dump, k), 'rb') as f:
            assert f.read() == b.getvalue(), k
    for k, a in rec['depth'].items():
        got = np.load(os.path.join(dump, k))
        assert got.dtype == np.float32 and got.tobytes() == a.tobytes(), k
        filled += int((a > 0).sum())
    assert filled > 0
    assert not multiprocessing.active_children()


def test_prepare_then_train(tmp_path):
    """A raw tree prepared with --with-gt at 64x128 and cc_b200.train.main on the dump with --with-depth-gt: one epoch of
    two steps, depth validation, the checkpoints and logs.  The disp net trains and the pose, mask and flow nets are
    fixed: with the README's --fix-masknet --fix-flownet alone the best model is chosen by --with-flow-gt, which needs
    KITTI-2015."""
    d = PD.write_run_dir(str(tmp_path), 'kitti_static')
    argv = ['raw', '--dataset-format', 'kitti', '--dump-root', 'dump', '--with-gt', '--height', '64', '--width', '128',
            '--num-threads', '2', '--test-scenes', 'test_scenes.txt', '--static-frames', 'static.txt']
    prep = _in(d, lambda: PT.main(argv, device=DEV))
    assert prep['val'] and prep['train']
    out = _in(d, lambda: T.main(['dump', '--name', 'prep', '-b', '2', '--epochs', '1', '--epoch-size', '2',
                                 '--workers', '2', '--with-depth-gt', '--fix-posenet', '--fix-masknet', '--fix-flownet',
                                 '-m0.1', '-pf', '0.5', '-pc', '1.0', '-s0.1', '-c0.3', '--smoothness-type', 'edgeaware'],
                                device=DEV))
    assert len(out['train_losses']) == 1 and np.isfinite(out['train_losses'][0])
    assert len(out['decisive_errors']) == 1 and np.isfinite(float(out['decisive_errors'][0]))
    save = os.path.join(d, out['save_path'])
    for prefix in T.CKPT_PREFIXES:
        for kind in ('checkpoint', 'model_best'):
            assert os.path.isfile(os.path.join(save, '%s_%s.pth.tar' % (prefix, kind))), (prefix, kind)
    for log in ('progress_log_summary.csv', 'progress_log_full.csv'):
        with open(os.path.join(save, log)) as f:
            assert len(f.read().splitlines()) == (2 if 'summary' in log else 3), log
