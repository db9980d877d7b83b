"""Host-side tile geometry of the wgmma convolution kernels (conv_tc.cu), no GPU: for every output-channel count the
wgmma N covers the channel tile, the pipeline has 2-4 stages, and the stages plus the barrier / 1 KB alignment slack fit
the 227 KB of shared memory an H100 block may use."""
import ctypes as C

SMEM_MAX = 227 * 1024
A_TILE = 128 * 32 * 4          # one A operand copy of one stage: 128 rows x 32 fp32


def test_tc_plan_fits_shared_memory():
    import __graft_entry__ as ge
    from cc_b200 import _lib
    lib = C.CDLL(ge.build())
    _lib._bind(lib)
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
