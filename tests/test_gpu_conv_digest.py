"""The tensor-core fprop and data-gradient convolutions held to fixed bits: the SHA-256 of each output at seeded shapes
that cover every wgmma N (16/32/64/128), both im2col gather paths (one filter tap per k-stage, and stages straddling
taps), split-K, strided data gradients and a ragged last pixel tile.  The digests in tests/golden/conv_tc_digests.json
were recorded on an H100; a kernel change that keeps the products and their summation order keeps every digest.

Record them again (only when the arithmetic is meant to change):  python -m tests.test_gpu_conv_digest OUT.json"""
import hashlib
import json
import os
import sys
import pytest
import torch
from tests.util import GOLDEN, conv_impl, device_lib   # noqa: F401  (device_lib: module fixture, the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]

DIGESTS = os.path.join(GOLDEN, 'conv_tc_digests.json')

# name: op, (B, Ci, H, W, Co, k, stride, pad).  N is Co for fprop and Ci for dgrad; the gather reads Ci (fprop) or Co
# (dgrad) channels, and a k-stage of 32 stays inside one filter tap when that count is a multiple of 32.
CASES = {
    'fprop_n16_fast':          ('fprop', (2, 32, 24, 40, 16, 3, 1, 1)),
    'fprop_n32_straddle':      ('fprop', (2, 20, 23, 37, 24, 3, 1, 1)),     # 1702 pixels: ragged last tile
    'fprop_n64_fast':          ('fprop', (2, 64, 32, 48, 64, 3, 1, 1)),
    'fprop_n128_fast':         ('fprop', (2, 128, 32, 64, 128, 3, 1, 1)),
    'fprop_n128_ragged_n':     ('fprop', (2, 96, 30, 41, 196, 1, 1, 0)),    # 196 = 128 + 68 channels, 2460 pixels
    'fprop_n32_k7s2_straddle': ('fprop', (2, 3, 64, 96, 32, 7, 2, 3)),
    'fprop_n128_splitk':       ('fprop', (1, 256, 8, 13, 128, 3, 1, 1)),    # one pixel tile, 72 k-tiles: split-K
    'dgrad_n16_straddle':      ('dgrad', (2, 16, 24, 40, 20, 3, 1, 1)),
    'dgrad_n64_fast':          ('dgrad', (2, 64, 32, 48, 64, 3, 1, 1)),
    'dgrad_n128_s2_fast':      ('dgrad', (2, 128, 32, 64, 64, 3, 2, 1)),    # four parity classes
    'dgrad_n32_k4s2_straddle': ('dgrad', (2, 32, 30, 42, 20, 4, 2, 1)),
    'dgrad_n128_splitk':       ('dgrad', (1, 128, 8, 16, 256, 3, 1, 1)),
}


def _digest(name):
    from cc_b200 import _lib, nn as cnn
    op, (B, Ci, H, W, Co, k, s, p) = CASES[name]
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    dev = torch.device('cuda:0')
    w = (torch.randn(Co, Ci, k, k, generator=g) / (k * k * Ci) ** 0.5).to(dev)
    with conv_impl(_lib.IMPL_TC):
        if op == 'fprop':
            x = torch.randn(B, Ci, H, W, generator=g).to(dev)
            bias = torch.randn(Co, generator=g).to(dev)
            y = torch.full((B, Co, Ho, Wo), float('nan'), device=dev)
            d = cnn._desc(B, Ci, H, W, Co, Ho, Wo, k, s, p, _lib.ACT_LEAKY, 0.1)
            cnn._run(_lib.CONV_FPROP, d, x, w, bias, None, y)
        else:
            dy = torch.randn(B, Co, Ho, Wo, generator=g).to(dev)
            y = torch.full((B, Ci, H, W), float('nan'), device=dev)
            d = cnn._desc(B, Ci, H, W, Co, Ho, Wo, k, s, p, _lib.ACT_NONE, 0.0)
            cnn._run(_lib.CONV_DGRAD, d, dy, w, None, None, y)
        kernel = (_lib.lib().ccb_debug_last_conv_kernel() or b'').decode()
    torch.cuda.synchronize()
    assert kernel == 'conv_tc', f'{name} ran on {kernel!r}, not the tensor-core kernel'
    return hashlib.sha256(y.cpu().numpy().tobytes()).hexdigest()


@pytest.mark.parametrize('name', sorted(CASES))
def test_conv_tc_digest(name):
    with open(DIGESTS) as f:
        want = json.load(f)[name]
    assert _digest(name) == want, f'{name}: the tensor-core convolution output changed bits'


if __name__ == '__main__':
    from tests.util import _bound
    with _bound(None):
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        got = {n: _digest(n) for n in sorted(CASES)}
    with open(sys.argv[1], 'w') as f:
        json.dump(got, f, indent=1, sort_keys=True)
        f.write('\n')
    print(json.dumps(got, indent=1, sort_keys=True))
