"""Host-side tile geometry of the wgmma convolution kernels (conv_tc.cu), no GPU: for every output-channel count the
wgmma N covers the channel tile, the pipeline has 2-4 stages, and the stages plus the barrier / 1 KB alignment slack fit
the 227 KB of shared memory an H100 block may use.  And the plan edges the ring tests reach: every shape of
tests/test_gpu_conv_ring.py's EDGE_SHAPES mapped to the cells of the stage ring it runs, every cell covered."""
import ctypes as C
import pytest

SMEM_MAX = 227 * 1024
A_TILE = 128 * 32 * 4          # one A operand copy of one stage: 128 rows x 32 fp32


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    from cc_b200 import _lib
    lib = C.CDLL(ge.build())
    _lib._bind(lib)
    return lib


def test_tc_plan_fits_shared_memory(lib):
    out = (C.c_int * 4)()
    for n in list(range(1, 300)) + [512, 1024, 4096]:
        assert lib.ccb_debug_tc_plan(n, out) == 0
        nt, b_bytes, stages, smem = list(out)
        tile = min(n, 128)
        assert nt in (16, 32, 64, 128) and nt >= tile and (nt == 16 or nt // 2 < tile), (n, nt)
        assert b_bytes == nt * 128, (n, b_bytes)
        assert 2 <= stages <= 4, (n, stages)
        stage = 2 * A_TILE + 2 * b_bytes            # A hi + lo, B hi + lo
        assert smem - stages * stage >= 1023 + 2 * 4 * 8, (n, smem)    # alignment slack + full / empty barriers
        assert smem <= SMEM_MAX, (n, smem)
        assert smem + stage > SMEM_MAX or stages == 4, (n, stages)      # as many stages as fit
    assert lib.ccb_debug_tc_plan(0, out) != 0


# ---- the plan edges of the ring tests --------------------------------------------------------------------------------
# The planner's public arithmetic (conv_tc.cu): 128-pixel M tiles, 128-channel N tiles, k-tiles of 32, at most 32 splits
# of a fprop / data gradient, and NUM_SMS = 132 (ccb_common.cuh).  The persistent grid itself is sized from the card's
# real SM count (tc_persistent_grid), which is 132 on the H100 SXM: the units-per-CTA cells below assume that card.
TC_M, TC_NMAX, TC_K, TC_MAX_SPLITS, NUM_SMS = 128, 128, 32, 32, 132
PATHS = ('ffma', 'tc', 'tc_padded')        # ccb_debug_conv_plan's path codes


def cdiv(a, b):
    return -(-a // b)


def tc_kp(ntaps, cc):
    """conv_tc.cu tc_kp: the k extent of `ntaps` taps of cc channels padded to 4, in whole k-tiles; a parity class
    without taps still runs one all-zero k-tile."""
    return cdiv(ntaps * cdiv(cc, 4) * 4, TC_K) * TC_K if ntaps > 0 else TC_K


def _plan(lib, shape, op):
    from cc_b200 import _lib
    B, Ci, H, W, Co, k, s, p = shape
    d = _lib.ConvDesc()
    d.B, d.Ci, d.Hi, d.Wi, d.Co = B, Ci, H, W, Co
    d.Ho, d.Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    d.kh = d.kw = k
    d.stride, d.pad, d.act, d.slope, d.impl, d.wcache = s, p, _lib.ACT_NONE, 0.0, _lib.IMPL_TC, None
    out = (C.c_int * 2)()
    assert lib.ccb_debug_conv_plan(C.byref(d), op, out) == 0, shape
    return PATHS[out[0]], out[1]


def _geometry(lib, n):
    out = (C.c_int * 4)()
    assert lib.ccb_debug_tc_plan(n, out) == 0
    return out[0], out[2]                   # wgmma N, ring depth


def _launch_cells(kernel, depth, M, N, ktiles, splits):
    """Cells of one launch of `kernel` (conv_tc or conv_tc_wgrad): k-tiles per unit modulo the ring depth, units per
    CTA, the M / N tiles and the split-K edges."""
    cells = set()
    kps = cdiv(ktiles, splits)
    nkt = [max(0, min(ktiles, z * kps + kps) - z * kps) for z in range(splits)]
    cells |= {(kernel, 'k-tiles per unit mod depth %d' % depth, n % depth) for n in nkt if n > 0}
    units = cdiv(M, TC_M) * cdiv(N, TC_NMAX) * splits
    if units <= NUM_SMS:
        cells.add((kernel, 'units per CTA', '1'))
    elif units % NUM_SMS:
        cells.add((kernel, 'units per CTA', '>= 2, ragged last wave'))
    if splits > 1:
        cells.add((kernel, 'splits', 2 if splits == 2 else 'many'))
        if nkt[-1] in (0, 1):
            cells.add((kernel, 'last split', ('empty', 'one k-tile')[nkt[-1]]))
    if M < TC_M:
        cells.add((kernel, 'M', '< 128'))
    elif M % TC_M:
        cells.add((kernel, 'M', 'ragged last tile'))
    if N > TC_NMAX and N % TC_NMAX:
        cells.add((kernel, 'N', 'ragged above 128'))
    return cells


def ring_cells(lib, shape, epilogues):
    """{call: cells}: the cells the fprop, the data gradient (dgrad) and the weight gradient (wgrad) of one conv shape
    reach on the tensor-core path."""
    from cc_b200 import _lib
    B, Ci, H, W, Co, k, s, p = shape
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    out = {}
    out['fprop'] = cells = set()
    # fprop: M = output pixels, N = Co, K = k^2 taps of Ci channels
    path, splits = _plan(lib, shape, _lib.CONV_FPROP)
    assert path == 'tc', (shape, path)
    nt, depth = _geometry(lib, Co)
    cells |= {('fprop', 'wgmma N', nt), ('conv_tc', 'depth', depth)}
    cells |= _launch_cells('conv_tc', depth, B * Ho * Wo, Co, tc_kp(k * k, Ci) // TC_K, splits)
    if splits == TC_MAX_SPLITS:
        cells.add(('conv_tc', 'splits', 'most'))
    if splits > 1:
        cells |= {('fprop epilogue under split-K', 'bias + residual', act) for act in epilogues}
    # data gradient: one launch per stride parity class (py, px), M = the class's pixels, N = Ci, K = its taps of Co
    out['dgrad'] = cells = set()
    path, splits = _plan(lib, shape, _lib.CONV_DGRAD)
    assert path == 'tc', (shape, path)
    nt, depth = _geometry(lib, Ci)
    cells.add(('dgrad', 'wgmma N', nt))
    for py in range(min(s, H)):
        for px in range(min(s, W)):
            ky0, kx0 = (py + p) % s, (px + p) % s
            ntaps = (cdiv(k - ky0, s) if k > ky0 else 0) * (cdiv(k - kx0, s) if k > kx0 else 0)
            if ntaps == 0:
                cells.add(('dgrad stride %d' % s, 'class without taps', True))
            cells |= _launch_cells('conv_tc', depth, B * cdiv(H - py, s) * cdiv(W - px, s), Ci, tc_kp(ntaps, Co) // TC_K, splits)
    if splits == TC_MAX_SPLITS:
        cells.add(('conv_tc', 'splits', 'most'))
    if s > 1 and (H % 2 or W % 2):
        cells.add(('dgrad stride %d' % s, 'odd Hi or Wi, k', k))
    # weight gradient: M = k^2 taps of Ci padded to 4, N = Co, K = output pixels (rows padded to 4 on the padded path)
    out['wgrad'] = cells = set()
    path, splits = _plan(lib, shape, _lib.CONV_WGRAD)
    if path != 'ffma':
        nt, depth = _geometry(lib, Co)
        P = B * Ho * (cdiv(Wo, 4) * 4)
        cells |= {('wgrad', 'wgmma N', nt), ('wgrad', 'path', path), ('wgrad', 'splits', 1 if splits == 1 else 'many')}
        if P % TC_K:
            cells.add(('wgrad', 'pixels', 'not a multiple of 32'))
        cells |= _launch_cells('conv_tc_wgrad', depth, k * k * cdiv(Ci, 4) * 4, Co, cdiv(P, TC_K), splits)
    return out


def required_cells():
    from tests.net_cases import EPILOGUES
    req = {(op, 'wgmma N', n) for op in ('fprop', 'dgrad', 'wgrad') for n in (16, 32, 64, 128)}
    for kern in ('conv_tc', 'conv_tc_wgrad'):
        req |= {(kern, 'k-tiles per unit mod depth 4', r) for r in range(4)}
        req |= {(kern, 'k-tiles per unit mod depth 3', r) for r in range(3)}
        req |= {(kern, 'units per CTA', '1'), (kern, 'units per CTA', '>= 2, ragged last wave'),
                (kern, 'M', '< 128'), (kern, 'M', 'ragged last tile')}
    req |= {('conv_tc', 'depth', 4), ('conv_tc', 'depth', 3), ('conv_tc', 'N', 'ragged above 128')}
    req |= {('conv_tc', 'splits', v) for v in (2, 'many', 'most')}
    req |= {('conv_tc', 'last split', v) for v in ('empty', 'one k-tile')}
    req |= {('dgrad stride 2', 'odd Hi or Wi, k', k) for k in (1, 3, 4)} | {('dgrad stride 2', 'class without taps', True)}
    req |= {('wgrad', 'path', v) for v in ('tc', 'tc_padded')} | {('wgrad', 'splits', v) for v in (1, 'many')}
    req |= {('wgrad', 'pixels', 'not a multiple of 32')}
    req |= {('fprop epilogue under split-K', 'bias + residual', act) for act in EPILOGUES}
    return req


def test_ring_edge_shapes_cover_every_plan_cell(lib):
    """Every cell of the wgmma stage ring's plan - each kernel instantiation, k-tiles per unit at every residue of the
    ring depth, one and several units per CTA, split-K with 2 / many / the most splits and with an empty or one-k-tile
    last split, strided data gradients with and without taps, ragged M and N tiles, both weight-gradient paths, every
    activation epilogue under split-K - is reached by some shape of EDGE_SHAPES.  A planner change that moves a shape
    off its edge fails here instead of silently dropping the coverage of the GPU test."""
    from tests.test_gpu_conv_ring import EDGE_SHAPES
    from tests.net_cases import EPILOGUES
    got = set()
    for shapes in EDGE_SHAPES.values():
        for shape in shapes:
            got = got.union(*ring_cells(lib, shape, EPILOGUES).values())
    missing = sorted(required_cells() - got, key=str)
    assert not missing, 'plan cells no EDGE_SHAPES entry reaches:\n  ' + '\n  '.join(map(str, missing))
