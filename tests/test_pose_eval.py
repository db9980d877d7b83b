"""Pose evaluation without a GPU: the oracle (oracle/pose_eval.py) against the numbers frozen from the reference's own
frameworks, main-loop bodies and compute_pose_errors (tests/golden/pose_eval_small.npz), the loaders of cc_b200.evaluate
against the frozen frameworks on the same tree, the printed rows and the predictions file, then ccb_pose_errors compiled
by g++ against the CPU execution-model simulator (tests/sim) against the fixture and the oracle.  The same kernel cases
run on the H100 in tests/test_gpu_pose_eval.py."""
import os
import numpy as np
import pytest
import torch
from cc_b200 import evaluate as CE
from oracle import pose_eval as OP
from tests import pose_eval_cases as PC
from tests.util import sim_lib      # noqa: F401  (module fixture: the simulator library)

CPU = torch.device('cpu')


@pytest.mark.parametrize('case', PC.algebra_cases(), ids=lambda c: c['name'])
def test_oracle_algebra_equals_reference(case):
    c = case
    final = np.stack([OP.snippet_final(p, c['mode']) for p in c['poses6']])
    assert np.array_equal(final, c['final'])
    out = np.array([OP.pose_error(g, f) for g, f in zip(c['gt'], final)])
    assert np.array_equal(out, c['out'], equal_nan=True), (out, c['out'])
    PC.check_first_is_identity(c['final'], c['poses6'], c['name'])        # the reference's own numbers hold the bar


@pytest.mark.parametrize('kind', ['kitti', 'sintel'])
def test_oracle_snippets_equal_reference(kind):
    for name, s in PC.tree(kind)['seqs'].items():
        final = np.stack([OP.snippet_final(p, 'euler') for p in s['poses6']])
        assert np.array_equal(final, s['final']), name
        err = [OP.sintel_pose_error(g, f) for g, f in zip(s['gt'], final)] if kind == 'sintel' else \
            [OP.pose_error(g, f) for g, f in zip(s['gt'], final)]
        assert np.array_equal(np.array(err).reshape(s['errors'].shape), s['errors']), name


@pytest.fixture(scope='module')
def written_tree(tmp_path_factory):
    return PC.write_pose_tree(str(tmp_path_factory.mktemp('pose_tree')))


@pytest.mark.parametrize('kind', ['kitti', 'sintel'])
@pytest.mark.parametrize('loader', ['cc_b200', 'oracle'])
def test_frameworks_rebuild_the_reference(kind, loader, written_tree):
    """The same tree read again: the matched sequences in sorted order, their sorted files, the snippets and the
    compensated ground truth, bit for bit and in the reference's dtype, and n_rows = len(framework)."""
    want = PC.tree(kind)
    root = written_tree[0] if kind == 'kitti' else written_tree[1]
    patterns, L = (PC.KITTI_PATTERNS, PC.KITTI_LENGTH) if kind == 'kitti' else (PC.SINTEL_PATTERNS, PC.SINTEL_LENGTH)
    if loader == 'oracle':
        seqs, n_rows = OP.framework(root, patterns, L, sintel=kind == 'sintel')
    else:
        seqs, n_rows = (CE.kitti_pose_framework if kind == 'kitti' else CE.sintel_pose_framework)(root, patterns, L)
    assert n_rows == want['n_rows'] and [s['name'] for s in seqs] == sorted(want['seqs'])
    for s in seqs:
        w = want['seqs'][s['name']]
        assert [os.path.basename(f) for f in s['files']] == list(w['files'])
        assert s['snippets'].dtype == np.int64 and np.array_equal(s['snippets'], w['snippets'])
        assert s['gt'].dtype == w['gt'].dtype and np.array_equal(s['gt'], w['gt']), s['name']
    first = next(s for s in seqs if s['name'] == want['order'][0])
    assert np.array_equal(CE.load_pose_frames([first['files'][i] for i in first['snippets'][0]]), want['imgs0'])


def test_compensation_keeps_the_aliased_subtraction():
    """Every row loses the ORIGINAL first translation (row 0 ends at zero), and the rotation is the first pose's."""
    for s in PC.tree('kitti')['seqs'].values():
        assert not s['gt'][:, 0, :, 3].any()
        assert np.allclose(s['gt'][:, 0, :, :3], np.eye(3), atol=1e-12)
        assert np.abs(s['gt'][:, 1:, :, 3]).min() > 0


def test_sintel_cam_read(tmp_path):
    N = np.arange(12, dtype=np.float64).reshape(3, 4) / 7
    p = str(tmp_path / 'a.cam')
    with open(p, 'wb') as f:
        f.write(b'PIEH' + np.eye(3).tobytes() + N.tobytes())
    assert np.array_equal(CE.sintel_cam_read(p), N) and np.array_equal(OP.cam_read(p), N)
    with open(p, 'wb') as f:
        f.write(b'PIEG' + np.eye(3).tobytes() + N.tobytes())
    with pytest.raises(AssertionError, match='wrong tag'):
        CE.sintel_cam_read(p)


def _in_reference_order(kind, key):
    t = PC.tree(kind)
    return np.concatenate([t['seqs'][n][key] for n in t['order']])


@pytest.mark.parametrize('kind', ['kitti', 'sintel'])
def test_summary_is_the_printed_rows(kind):
    """pose_summary of the per-snippet errors in the reference's order equals its printed float32 rows bit for bit, zero
    rows included; in sorted sequence order it agrees within float32 rounding."""
    t = PC.tree(kind)
    sintel = kind == 'sintel'
    per = _in_reference_order(kind, 'errors')
    per = np.concatenate([np.zeros_like(per), per], 1) if sintel else per
    got = CE.pose_summary(per, t['n_rows'], sintel)
    assert got.dtype == np.float32 and got.shape == ((2, 1) if sintel else (2, 2))
    assert np.array_equal(got, t['summary']) and np.array_equal(OP.summary(per, t['n_rows'], sintel), t['summary'])
    unpadded = np.stack([per[:, 1:].mean(0), per[:, 1:].std(0)]) if sintel else np.stack([per.mean(0), per.std(0)])
    assert not np.allclose(got, unpadded, rtol=1e-3), 'the zero rows must count'
    per_sorted = np.concatenate([t['seqs'][n]['errors'] for n in sorted(t['seqs'])])
    per_sorted = np.concatenate([np.zeros_like(per_sorted), per_sorted], 1) if sintel else per_sorted
    assert np.allclose(CE.pose_summary(per_sorted, t['n_rows'], sintel), t['summary'], rtol=4e-7, atol=0)


def test_predictions_file(tmp_path):
    t = PC.tree('kitti')
    CE.write_pose_predictions(str(tmp_path / 'out'), _in_reference_order('kitti', 'final'), t['n_rows'])
    got = np.load(str(tmp_path / 'out' / 'predictions.npy'))
    assert got.dtype == np.float64 and np.array_equal(got, t['predictions'])


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('case', PC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(CPU)


@pytest.mark.parametrize('name,nb', [('PoseNetB6', 4), ('PoseNet6', 4), ('PoseExpNet', 2)])
def test_load_pose_net(name, nb, tmp_path):
    """seq_length from conv1.0.weight's input channels, the net built for seq_length - 1 references, loaded with
    strict=False: a checkpoint with keys the net lacks (the mask decoder of a PoseExpNet trained with output_exp) loads."""
    from cc_b200 import models as CM, synth
    src = synth.seeded_fill(getattr(CM, name)(nb_ref_imgs=nb, **({'output_exp': True} if name == 'PoseExpNet' else {})), 8)
    p = str(tmp_path / 'posenet.pth.tar')
    torch.save({'state_dict': src.state_dict(), 'epoch': 3}, p)
    net, seq_length = CE.load_pose_net(p, name, CPU)
    assert seq_length == nb + 1 and type(net).__name__ == name and net.nb_ref_imgs == nb
    sd = net.state_dict()
    assert sd and all(torch.equal(v, src.state_dict()[k]) for k, v in sd.items())
    if name == 'PoseExpNet':
        assert set(src.state_dict()) - set(sd)
