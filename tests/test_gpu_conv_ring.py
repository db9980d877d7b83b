"""The wgmma convolution kernels' stage ring at its edges - empty and one-k-tile splits, every k-tile count modulo the
ring depth, parity classes without taps, ragged channel counts and pixel tiles - against torch fp64 and the CUDA-core
kernels, and a CUDA-graph replay of each kernel variant against its eager run, bit for bit.  Every result is held
element by element to the layer audit's bound (tests/layer_audit.py), not only to rel_err: one k-stage that lost its
tf32 lo terms passes rel_err <= 1e-4 at K of a few hundred.  tests/test_conv_tc_plan.py maps every shape to the plan
cells it reaches and asserts that all are covered.  GPU only.

With $CCB_PARITY_REPORT_DIR set, the worst r of every shape and implementation is written there as conv_ring_<case>.json."""
import json
import os
import pytest
import torch
import torch.nn.functional as F
from tests.util import conv_impl, assert_close, device_lib   # noqa: F401  (device_lib: module fixture, the sm_90a library)
from tests.net_cases import _conv_cross_check
from tests.layer_audit import assert_conv_within_bound

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]

# B, Ci, H, W, Co, k, stride, pad.  The ring is 4 stages deep below 128 output channels, 3 at 128 (tc_geometry).
# Worst r against the layer audit's bound (R = 10) over these shapes on an H100 80GB HBM3 (132 SMs, 700 W power limit):
# 0.90 on the tensor-core kernels (a data gradient at wgmma N = 128), 2.32 on the CUDA-core kernels (a data gradient).
EDGE_SHAPES = {
    # one 64-pixel tile, 9 k-tiles in 4 splits of 3: the last split is empty and must contribute zeros
    'empty_split': [(1, 32, 8, 8, 20, 3, 1, 1)],
    # 1x1 over 4 channels: one k-tile; 68 channels: a ragged wgmma N of 128
    'one_ktile': [(2, 4, 20, 36, 68, 1, 1, 0)],
    # >= 132 pixel tiles (no split-K): each CTA runs all 2, 3, 4, 5, 7 or 9 k-tiles of a 4-deep ring ...
    'depth4_residues': [(2, 64, 96, 96, 32, 1, 1, 0), (2, 96, 96, 96, 32, 1, 1, 0), (2, 128, 96, 96, 32, 1, 1, 0),
                        (2, 160, 96, 96, 32, 1, 1, 0), (2, 224, 96, 96, 32, 1, 1, 0), (2, 32, 96, 96, 32, 3, 1, 1)],
    # ... and 3, 4, 5 k-tiles of a 3-deep ring, with ragged last channel tiles (275 = 2 x 128 + 19, 196, 136)
    'depth3_residues': [(2, 96, 96, 96, 275, 1, 1, 0), (2, 128, 96, 96, 196, 1, 1, 0), (2, 160, 96, 96, 136, 1, 1, 0)],
    # strided data gradients: 1x1 stride 2 has three parity classes without taps (one all-zero k-tile each)
    'parity_classes': [(2, 64, 16, 24, 20, 1, 2, 0), (2, 20, 15, 24, 2, 3, 2, 1)],
    # 780 and 741 pixels: the last tile's rows past M
    'ragged_m': [(3, 17, 13, 20, 40, 3, 1, 1), (3, 36, 13, 19, 196, 3, 1, 1)],
    # odd Hi or Wi, so the parity classes differ in size: 1x1 (three classes without taps) and 4x4 (four of 2 x 2 taps)
    'odd_parity_classes': [(2, 64, 15, 23, 20, 1, 2, 0), (2, 24, 15, 21, 40, 4, 2, 1)],
    # fprop split 2 ways (4 k-tiles); 13 k-tiles in 4 splits of 4, 4, 4, 1; 144 k-tiles in the most splits, 32 (29 of
    # 5, 5, ..., 4, three empty); 18 k-tiles in 9 splits of 2.  Every fprop runs each epilogue with bias + residual.
    'split_k': [(2, 128, 16, 16, 32, 1, 1, 0), (2, 44, 64, 66, 32, 3, 1, 1), (1, 512, 8, 8, 64, 3, 1, 1),
                (2, 64, 16, 16, 64, 3, 1, 1)],
}


@pytest.mark.parametrize('case', sorted(EDGE_SHAPES))
def test_ring_edges(case):
    rows = _conv_cross_check(torch.device('cuda:0'), EDGE_SHAPES[case], 17, case)
    out = os.environ.get('CCB_PARITY_REPORT_DIR')
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'conv_ring_%s.json' % case), 'w') as f:
            json.dump(rows, f, indent=1)


def test_ring_conv_transpose():
    """ConvTranspose2d forward runs the strided data-gradient parity classes; ragged 20 output channels."""
    from cc_b200 import _lib, nn as cnn
    g = torch.Generator().manual_seed(19)
    dev = torch.device('cuda:0')
    x = torch.randn(2, 48, 9, 14, generator=g).to(dev)
    b = torch.randn(20, generator=g).to(dev)
    for (k, op) in ((4, 0), (3, 1), (1, 1)):
        w = (torch.randn(48, 20, k, k, generator=g) * 0.1).to(dev)
        zd = F.conv_transpose2d(x.double(), w.double(), b.double(), 2, 1 if k > 1 else 0, op)
        outs = []
        for impl in (_lib.IMPL_TC, _lib.IMPL_FFMA):
            with conv_impl(impl):
                outs.append(cnn.conv_transpose2d(x, w, b, 2, 1 if k > 1 else 0, op, None))
            assert_close(outs[-1], zd, 1e-4, f'convT k{k} impl {impl}')
            assert_conv_within_bound('convT', x, w, 2, 1 if k > 1 else 0, bias=b, out_pad=op, y=outs[-1],
                                     what=f'convT k{k} impl {impl}')
        assert_close(outs[0], outs[1], 1e-4, f'convT k{k} tensor-core vs CUDA-core kernels')


# Ci == Co == c selects the wgmma N (16, 32, 64, 128) of all three kernels; the last runs the strided data gradient
@pytest.mark.parametrize('c,stride', [(8, 1), (20, 1), (40, 1), (100, 1), (40, 2)])
def test_graph_replay_is_bitwise_eager(c, stride):
    from cc_b200 import _lib, nn as cnn
    g = torch.Generator().manual_seed(23)
    dev = torch.device('cuda:0')
    B, H, W, k, pad = 2, 24, 32, 3, 1
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    x = torch.randn(B, c, H, W, generator=g).to(dev)
    w = (torch.randn(c, c, k, k, generator=g) / (9 * c) ** 0.5).to(dev)
    bias = torch.randn(c, generator=g).to(dev)
    dy = torch.randn(B, c, Ho, Wo, generator=g).to(dev)

    def run(outs):
        y, dx, dw = outs
        with conv_impl(_lib.IMPL_TC):
            d = cnn._desc(B, c, H, W, c, Ho, Wo, k, stride, pad, _lib.ACT_LEAKY, 0.2)
            cnn._run(_lib.CONV_FPROP, d, x, w, bias, None, y)
            d = cnn._desc(B, c, H, W, c, Ho, Wo, k, stride, pad, _lib.ACT_NONE, 0.0)
            cnn._run(_lib.CONV_DGRAD, d, dy, w, None, None, dx)
            cnn._run(_lib.CONV_WGRAD, d, x, dy, dw)

    def buffers():
        return (torch.full((B, c, Ho, Wo), float('nan'), device=dev), torch.full_like(x, float('nan')),
                torch.full_like(w, float('nan')))

    eager = buffers()
    run(eager)
    torch.cuda.synchronize()
    for got, (name, ref) in zip(eager, (('fprop', F.leaky_relu(F.conv2d(x.double(), w.double(), bias.double(), stride, pad), 0.2)),
                                         ('dgrad', torch.nn.grad.conv2d_input(x.shape, w.double(), dy.double(), stride, pad)),
                                         ('wgrad', torch.nn.grad.conv2d_weight(x.double(), w.shape, dy.double(), stride, pad)))):
        assert_close(got, ref, 1e-4, f'eager {name} c{c} s{stride}')
    tag = f'eager c{c} s{stride}'
    assert_conv_within_bound('conv', x, w, stride, pad, bias=bias, act='leaky', slope=0.2, y=eager[0], what=tag)
    assert_conv_within_bound('conv', x, w, stride, pad, g=dy, dx=eager[1], dw=eager[2], what=tag)
    replayed = buffers()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run(replayed)
    graph.replay()
    torch.cuda.synchronize()
    for a, b_, name in zip(eager, replayed, ('fprop', 'dgrad', 'wgrad')):
        assert torch.equal(a, b_), f'graph replay of {name} c{c} s{stride} differs from the eager run'
