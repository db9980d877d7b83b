"""The reference's flowutils/flowlib.py colour coding on the device (ccb_flow_color).

  flow_to_image(flow)   [2,H,W] -> the Middlebury colour image.  A numpy array returns what the reference returns (float64
                        [3,H,W], uint8 levels / 255), computed on the current CUDA device; a tensor returns the uint8 levels
                        [3,H,W] on its device.  Unlike the reference, the argument is not modified (the reference zeroes
                        its unknown pixels in place).
  make_color_wheel()    the 55 x 3 wheel (RY 15, YG 6, GC 4, CB 11, BM 13, MR 6 steps)."""
import numpy as np
import torch
from .. import _lib

UNKNOWN_FLOW_THRESH = 1e7


def flow_to_image(flow):
    from ..evaluate import flow_colors
    if torch.is_tensor(flow):
        assert flow.dim() == 3 and flow.shape[0] == 2, flow.shape
        return flow_colors(flow[None, None])[0]
    flow = np.asarray(flow)
    assert flow.ndim == 3 and flow.shape[0] == 2, flow.shape
    levels = flow_colors(torch.from_numpy(np.ascontiguousarray(flow, np.float32))[None, None].to(_lib.device()))[0]
    return levels.cpu().numpy() / 255.


def make_color_wheel():
    wheel = []
    for n, fixed, ramp, rising in ((15, 0, 1, True), (6, 1, 0, False), (4, 1, 2, True), (11, 2, 1, False),
                                   (13, 2, 0, True), (6, 0, 2, False)):
        for k in range(n):
            c = [0.0, 0.0, 0.0]
            c[fixed] = 255.0
            c[ramp] = 255 * k // n if rising else 255 - 255 * k // n
            wheel.append(c)
    return np.array(wheel)
