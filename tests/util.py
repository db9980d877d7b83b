"""Shared helpers for the parity tests, and the fixtures that bind a build of the library for a test module."""
import contextlib
import os
import sys
import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, 'golden')
SIM = os.path.join(HERE, 'sim')
_cache = {}


@contextlib.contextmanager
def _bound(path):
    """libccb200 at `path` (None: the in-tree sm_90a build) bound for the block, the pyramid memo cleared on both sides
    (it holds tensors of the other build's calls); the previous binding is restored afterwards."""
    from cc_b200 import _lib, pyramid
    prev = (_lib._lib, _lib._is_sim)
    if path is None:
        _lib._lib = None
        _lib.lib()
    else:
        _lib.use_library(path)
    pyramid.clear()
    try:
        yield _lib
    finally:
        _lib._lib, _lib._is_sim = prev
        pyramid.clear()


@pytest.fixture(scope='module')
def sim_lib():
    """The product kernels compiled by g++ against the CPU simulator (tests/sim)."""
    if SIM not in sys.path:
        sys.path.insert(0, SIM)
    import build_sim
    with _bound(build_sim.build()) as lib:
        assert lib.is_simulator()
        yield


@pytest.fixture(scope='module')
def device_lib():
    """The sm_90a library, with torch's TF32 off (torch computes some of the checks on the device in fp32)."""
    with _bound(None) as lib:
        assert not lib.is_simulator(), 'GPU tests must run on the sm_90a library'
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        yield


@contextlib.contextmanager
def conv_impl(impl):
    """cc_b200.nn's convolutions dispatched to `impl` (cc_b200._lib.IMPL_*) inside the block."""
    from cc_b200 import nn as cnn
    saved = cnn.CONV_IMPL
    cnn.CONV_IMPL = impl
    try:
        yield
    finally:
        cnn.CONV_IMPL = saved


def golden(name):
    """The arrays of tests/golden/<name>.npz, or merged from <name>.part<i>.npz when the set is split (files < 1 MB)."""
    if name not in _cache:
        whole = os.path.join(GOLDEN, name + '.npz')
        parts = [whole] if os.path.exists(whole) else \
            sorted(os.path.join(GOLDEN, f) for f in os.listdir(GOLDEN) if f.startswith(name + '.part') and f.endswith('.npz'))
        assert parts, 'golden fixture %s is missing' % name
        d = {}
        for p in parts:
            with np.load(p) as z:
                d.update({k: z[k] for k in z.files})
        _cache[name] = d
    return _cache[name]


def _assert_equal(got, want, where):
    """torch.equal on every tensor of `want`, through tuples, lists and dicts."""
    if isinstance(want, dict):
        assert got.keys() == want.keys(), where
        for k in want:
            _assert_equal(got[k], want[k], '%s[%r]' % (where, k))
    elif isinstance(want, (tuple, list)):
        assert len(got) == len(want), where
        for i, (g, w) in enumerate(zip(got, want)):
            _assert_equal(g, w, '%s[%d]' % (where, i))
    else:
        assert torch.equal(got, want), where


def assert_graph_replays(chain, first, second):
    """`chain(*inputs)` makes no host round-trip: captured once in a CUDA graph on a clone of `first` (after a warm-up on a
    side stream), then replayed with `first`, `second` and `first` again copied into the captured buffers, each replay
    equal bit for bit to the eager run on the same inputs.  Returns the two eager results: the caller asserts that they
    differ, on the output it cares about, so that the replays cannot pass vacuously."""
    eager = [chain(*ins) for ins in (first, second)]
    static = [t.clone() for t in first]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        chain(*static)                          # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = chain(*static)
    for i, (ins, want) in enumerate(zip((first, second, first), eager + eager[:1])):
        for dst, src in zip(static, ins):
            dst.copy_(src)
        graph.replay()
        _assert_equal(out, want, 'replay %d' % i)
    return eager


def T(a, device='cpu'):
    return torch.from_numpy(np.asarray(a)).to(device)


def rel_err(a, b):
    """max |a-b| / max(|b|_inf, tiny): the '1e-4 relative in fp32' bar of BASELINE.json is read as
    error relative to the tensor's scale (per-element relative error is meaningless at zero crossings)."""
    a = torch.as_tensor(a, dtype=torch.float64).cpu()
    b = torch.as_tensor(b, dtype=torch.float64).cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    scale = max(b.abs().max().item(), 1e-30)
    return (a - b).abs().max().item() / scale


def assert_close(a, b, tol=1e-4, what=''):
    e = rel_err(a, b)
    assert e <= tol, f'{what}: rel err {e:.3e} > {tol:.1e}'


def key_with_stride(d, prefix):
    """Golden grads of big tensors are stored as flat[::stride] under 'name@stride'."""
    for k in d:
        if k == prefix:
            return k, None
        if k.startswith(prefix + '@'):
            return k, int(k.split('@')[1])
    raise KeyError(prefix)


def pick(g, stride):
    return g if stride is None else g.flatten()[::stride]


def assert_close_robust(a, b, tol=1e-4, max_outlier_frac=2e-4, what=''):
    """Full-size variant: the gradient of a bilinear sample is discontinuous where a coordinate lands on
    an integer pixel, so 1-ulp coordinate differences flip a handful of pixels' gradients - the oracle
    run on CPU and on GPU disagree with EACH OTHER at ~1e-4 of the level-0 pixels (tools/diag_masks.py
    log).  Require <= tol everywhere except a vanishing fraction."""
    a = torch.as_tensor(a, dtype=torch.float64).cpu()
    b = torch.as_tensor(b, dtype=torch.float64).cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    scale = max(b.abs().max().item(), 1e-30)
    err = (a - b).abs() / scale
    n_bad = int((err > tol).sum().item())
    allowed = max(2, int(max_outlier_frac * err.numel()))
    assert n_bad <= allowed, f'{what}: {n_bad} of {err.numel()} elements exceed {tol:.1e} (max {err.max().item():.2e}), allowed {allowed}'
