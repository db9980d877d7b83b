"""Checks of a prepared dump against tests/golden/prepare_small.npz (what the reference's prepare_train_data.py wrote for
the trees of tests/prepare_cases.py), shared by the CPU simulator tests and the H100 tests.

The split depends on the order os.listdir gives the dump's folders, which differs between file systems, so the expected
files are derived from the order the run itself saw: draw k of RandomState(8964) decides folder k."""
import hashlib
import io
import os
import numpy as np
from PIL import Image

from tests import prepare_cases as PC
from tests.util import golden

FIXTURE = 'prepare_small'


def fixture():
    return golden(FIXTURE)


def named(g, run, kind):
    """{relative path: array} of the fixture's recorded jpg frames or npy depth maps of a run."""
    return {str(n): g['%s_%s_%d' % (run, kind, i)] for i, n in enumerate(g['%s_%s_names' % (run, kind)])}


def split_rule(order, seed=8964):
    rs = np.random.RandomState(seed)
    draws = [rs.random_sample() for _ in order]
    return [n for n, r in zip(order, draws) if r >= 0.1], [n for n, r in zip(order, draws) if r < 0.1]


def expected_files(g, run, order, presplit=False):
    """The dump's files after the run when the split saw `order` (presplit: every folder keeps its depth maps and no
    list is written)."""
    train, _ = split_rule(order)
    files = [str(f) for f in g[run + '_cam_names']] + list(named(g, run, 'jpg'))
    files += [f for f in named(g, run, 'npy') if presplit or f.split('/')[0] not in train]
    return sorted(files + ([] if presplit else ['train.txt', 'val.txt']))


def write_run_dir(root, run):
    """The run's working directory rebuilt from the fixture's tree bytes."""
    g = fixture()
    return PC.write_run_dir(root, PC.tree_from_fixture(g, PC.RUN_TREE[run]))


def check_fixture_consistent(run):
    g = fixture()
    order = [str(n) for n in g[run + '_order']]
    train, val = split_rule(order)
    assert [str(n) for n in g[run + '_train']] == train and [str(n) for n in g[run + '_val']] == val
    assert [str(f) for f in g[run + '_files']] == expected_files(g, run, order)


def check_dump(run, dump, order, presplit=False):
    """The dump at `dump` equals the fixture: the file set for the split order `order`, cam.txt text, each jpg's bytes
    (Pillow encoding the fixture's uint8 frame here, so the check does not depend on the Pillow that made the fixture),
    each .npy bit for bit (its bytes those of np.save of the fixture's array), train.txt and val.txt."""
    g = fixture()
    listed = [n for n in os.listdir(dump) if os.path.isdir(os.path.join(dump, n))]
    assert order == listed and sorted(order) == sorted(str(n) for n in g[run + '_order']), (order, listed)
    assert PC.dump_files(dump) == expected_files(g, run, order, presplit)
    for name, text in zip(g[run + '_cam_names'], g[run + '_cam_text']):
        with open(os.path.join(dump, str(name))) as f:
            assert f.read() == str(text), name
    for name, a in named(g, run, 'jpg').items():
        b = io.BytesIO()
        Image.fromarray(a).save(b, format='JPEG')
        with open(os.path.join(dump, name), 'rb') as f:
            assert f.read() == b.getvalue(), name
    for name, a in named(g, run, 'npy').items():
        p = os.path.join(dump, name)
        if not os.path.exists(p):
            continue                                      # a train folder's depth, removed by the split
        got = np.load(p)
        assert got.dtype == np.float32 and got.tobytes() == a.tobytes(), name
        b = io.BytesIO()
        np.save(b, a)
        with open(p, 'rb') as f:
            assert f.read() == b.getvalue(), name
    if not presplit:
        train, val = split_rule(order)
        for name, names in (('train.txt', train), ('val.txt', val)):
            with open(os.path.join(dump, name)) as f:
                assert f.read() == ''.join(n + '\n' for n in names), name


def check_oracle_record(run, rec, dump):
    """oracle.prepare's record and dump equal the fixture: the pre-encode uint8 frames and float32 depth maps bit for
    bit, and the dump's files for the order its split saw."""
    g = fixture()
    want = named(g, run, 'jpg')
    assert sorted(rec['frames']) == sorted(want)
    for k, a in want.items():
        assert rec['frames'][k].dtype == np.uint8 and np.array_equal(rec['frames'][k], a), k
    want = named(g, run, 'npy')
    assert sorted(rec['depth']) == sorted(want)
    for k, a in want.items():
        assert rec['depth'][k].dtype == np.float32 and rec['depth'][k].tobytes() == a.tobytes(), k
    assert (rec['train'], rec['val']) == split_rule(rec['order'])
    check_dump(run, dump, rec['order'])


def hashes(root):
    out = {}
    for f in PC.dump_files(root):
        with open(os.path.join(root, f), 'rb') as fh:
            out[f] = hashlib.sha256(fh.read()).hexdigest()
    return out
