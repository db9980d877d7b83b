"""The tensor-core weight-gradient convolution held to fixed bits: the SHA-256 of dw at seeded shapes that cover every
wgmma N (16/32/64/128, and 196 = 128 + 68 output channels), 1x1 / 3x3 / 7x7 filters and stride 2, input channels
padded to 4 (Ci 3 and 2), a last row tile that is not full, pixel k-tiles that straddle output rows and images, split-K
from 1 split to the plan's maximum, more work units than SMs, and the padded-rows path of an output width that is not
a multiple of 4.  The digests in tests/golden/conv_tc_wgrad_digests.json were recorded on an H100; a kernel change that
keeps the products and their summation order keeps every digest.

Record them again (only when the arithmetic is meant to change):  python -m tests.test_gpu_conv_wgrad_digest OUT.json"""
import hashlib
import json
import os
import sys
import pytest
import torch
from tests.util import GOLDEN, conv_impl, device_lib   # noqa: F401  (device_lib: module fixture, the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]

DIGESTS = os.path.join(GOLDEN, 'conv_tc_wgrad_digests.json')

# name: (B, Ci, H, W, Co, k, stride, pad).  Rows of the GEMM are (tap, ci) with ci padded to 4 (Mtot = k*k*cpad), columns
# are the Co output channels (wgmma N), k runs over the B*Ho*Wo output pixels in k-tiles of 32.  Splits: tc_plan's
# split-K count for the shape; units = row tiles x channel tiles x splits.
CASES = {
    'n16_co1_k3':             (2, 32, 24, 40, 1, 3, 1, 1),      # Mtot 288 (3 row tiles, last ragged), 15 splits
    'n16_ci3_k7s2':           (2, 3, 64, 96, 16, 7, 2, 3),      # Ci 3 -> cpad 4, Mtot 196, 24 splits
    'n16_ci3_max_splits':     (2, 3, 64, 264, 16, 3, 1, 1),     # 1056 k-tiles: 264 splits, 264 units > 132 SMs
    'n32_co20_ci2_straddle':  (3, 2, 23, 36, 20, 3, 1, 1),      # Ho*Wo 828, P 2484: k-tiles straddle rows and images
    'n32_k1_ragged_p':        (1, 48, 20, 52, 32, 1, 1, 0),     # P 1040: last k-tile half full
    'n32_padded_rows':        (2, 64, 13, 26, 32, 3, 1, 1),     # Wo 26: x and dy copied into rows of 28
    'n64_k3':                 (2, 64, 32, 48, 64, 3, 1, 1),     # Mtot 576, 24 splits
    'n64_k3s2':               (2, 32, 32, 64, 64, 3, 2, 1),     # stride 2
    'n64_one_split':          (1, 16, 8, 16, 64, 3, 1, 1),      # 4 k-tiles: 1 split
    'n128_k3_few_splits':     (2, 128, 15, 28, 128, 3, 1, 1),   # Ho*Wo 420, 9 row tiles, 6 splits
    'n128_co196_k7':          (1, 64, 16, 32, 196, 7, 1, 3),    # 196 = 128 + 68 channels, 25 x 2 tiles x 4 splits
}


def _digest(name):
    from cc_b200 import _lib, nn as cnn
    B, Ci, H, W, Co, k, s, p = CASES[name]
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    dev = torch.device('cuda:0')
    x = torch.randn(B, Ci, H, W, generator=g).to(dev)
    dy = torch.randn(B, Co, Ho, Wo, generator=g).to(dev)
    dw = torch.full((Co, Ci, k, k), float('nan'), device=dev)
    with conv_impl(_lib.IMPL_TC):
        d = cnn._desc(B, Ci, H, W, Co, Ho, Wo, k, s, p, _lib.ACT_NONE, 0.0)
        cnn._run(_lib.CONV_WGRAD, d, x, dy, dw)
        kernel = (_lib.lib().ccb_debug_last_conv_kernel() or b'').decode()
    torch.cuda.synchronize()
    assert kernel == 'conv_tc_wgrad', f'{name} ran on {kernel!r}, not the tensor-core weight gradient'
    return hashlib.sha256(dw.cpu().numpy().tobytes()).hexdigest()


@pytest.mark.parametrize('name', sorted(CASES))
def test_conv_tc_wgrad_digest(name):
    with open(DIGESTS) as f:
        want = json.load(f)[name]
    assert _digest(name) == want, f'{name}: the tensor-core weight gradient changed bits'


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
