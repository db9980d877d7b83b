"""The workspace contract of include/ccb200.h without a GPU: the cases of tests/workspace_cases.py on the CPU simulator
build, and a check of the headers that every scratch buffer is followed by its size.  The same cases run on the H100 in
tests/test_gpu_workspace_contract.py."""
import re
import pytest
import torch
from tests import workspace_cases as WC
from tests.test_cabi_symbols import _ctype, _header_source
from tests.util import sim_lib      # noqa: F401  (module fixture: the simulator library)

CPU = torch.device('cpu')
SCRATCH = re.compile(r'(?:work|partials|\w+_partials)$')
SUFFIX = {'float*': '_floats', 'unsigned long long*': '_words', 'void*': '_bytes'}


@pytest.mark.usefixtures('sim_lib')
@pytest.mark.parametrize('row', WC.ROWS, ids=WC.IDS)
def test_row(row, monkeypatch):
    WC.check_row(CPU, row, monkeypatch)


@pytest.mark.usefixtures('sim_lib')
def test_null_where_nothing_is_needed():
    WC.check_zero_need(CPU)


def scratch_violations(src):
    """Every parameter or descriptor field named work, partials or *_partials of the C source `src` (comments removed)
    that is not followed directly by a `long long` named after it with the suffix of its pointer type."""
    src = re.sub(r'^\s*#.*$', '', src, flags=re.M)
    lists = [m.group(1).split(',') for m in re.finditer(r'\bccb_\w+\s*\(([^()]*)\)\s*;', src)]
    lists += [body.split(';') for body in re.findall(r'typedef\s+struct\s+\w+\s*\{(.*?)\}\s*\w+\s*;', src, flags=re.S)]
    bad = []
    for decls in lists:
        decls = [(_ctype(t[:-1]), t[-1]) for t in (re.findall(r'\w+|\*', re.sub(r'\[\w*\]', '', d)) for d in decls) if t]
        for i, (ctype, name) in enumerate(decls):
            if SCRATCH.match(name):
                want = ('long long', name + SUFFIX.get(ctype, '?'))
                got = decls[i + 1] if i + 1 < len(decls) else None
                if got != want:
                    bad.append('%s %s: followed by %s, not %s %s' % (ctype, name, got, *want))
    return bad


def test_every_scratch_buffer_has_its_size():
    src = _header_source()
    assert len(re.findall(r'\b(?:work|partials|pose_partials)\b', src)) >= 20
    assert scratch_violations(src) == []


def test_scratch_check_reports_planted_violations():
    """The check is not vacuous: a dropped size, a size in the wrong unit and a size moved away from its buffer are each
    reported."""
    src = _header_source()
    planted = re.sub(r'(int ccb_ssim_bwd\([^;]*?float\* work), long long work_floats', r'\1', src)
    planted = re.sub(r'(int ccb_featwarp_bwd\([^;]*?)work_words', r'\1work_floats', planted)
    planted = re.sub(r'(typedef struct ccb_smooth_desc \{.*?float\* partials;)\s*long long partials_floats;(\s*float\* loss;)',
                     r'\1\2 long long partials_floats;', planted, flags=re.S)
    assert planted.count('work_floats') == src.count('work_floats')
    assert sorted(scratch_violations(planted)) == [
        "float* partials: followed by ('float*', 'loss'), not long long partials_floats",
        "float* work: followed by ('ccb_stream_t', 'stream'), not long long work_floats",
        "unsigned long long* work: followed by ('long long', 'work_floats'), not long long work_words",
    ]
