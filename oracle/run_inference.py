"""run_inference.py restated on numpy, Pillow and torch's CPU ops: matplotlib's colormaps as utils.py builds them
(LinearSegmentedColormap, ListedColormap and Colormap.__call__ of matplotlib 3.x before 3.9), tensor2array (utils.py:36-53)
and the script's body for one image (run_inference.py:56-80), with DispNetS (models/DispNetS.py:86-133) as a functional
forward over its state_dict.  tests/golden/run_inference_small.npz holds what the reference's own main() wrote for the
same folder; tests/golden/make_run_inference.py runs it with the colormap classes below standing in for matplotlib."""
import numpy as np
import torch
import torch.nn.functional as F
from .make3d_eval import imresize
from .nets import _crop_like


# ---- matplotlib (colors.py, cm.py, _cm.py) ----------------------------------------------------------------------------
class Colormap:
    """Colormap.__call__ on a float array, bytes=False, alpha=None: the fp64 RGBA of each value."""

    def __init__(self, name, N=256):
        self.name, self.N = name, int(N)
        self._i_under, self._i_over, self._i_bad = self.N, self.N + 1, self.N + 2
        self._lut = None

    def _set_extremes(self):
        self._lut[self._i_under] = self._lut[0]
        self._lut[self._i_over] = self._lut[self.N - 1]
        self._lut[self._i_bad] = (0.0, 0.0, 0.0, 0.0)

    def __call__(self, X):
        if self._lut is None:
            self._init()
        mask_bad = np.isnan(X)
        xa = np.array(X, copy=True)
        with np.errstate(invalid='ignore'):
            xa *= self.N
            xa[xa < 0] = -1
            xa[xa == self.N] = self.N - 1
            np.clip(xa, -1, self.N, out=xa)
            xa = xa.astype(int)
        xa[xa > self.N - 1] = self._i_over
        xa[xa < 0] = self._i_under
        xa[mask_bad] = self._i_bad
        return self._lut.copy().take(xa, axis=0, mode='clip')


def create_lookup_table(N, data, gamma=1.0):
    """colors._create_lookup_table for segment data rows (x, y0, y1)."""
    adata = np.array(data)
    x, y0, y1 = adata[:, 0], adata[:, 1], adata[:, 2]
    if N == 1:
        lut = np.array(y0[-1])
    else:
        x = x * (N - 1)
        xind = (N - 1) * np.linspace(0, 1, N) ** gamma
        ind = np.searchsorted(x, xind)[1:-1]
        distance = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
        lut = np.concatenate([[y1[0]], distance * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]])
    return np.clip(lut, 0.0, 1.0)


class LinearSegmentedColormap(Colormap):
    def __init__(self, name, segmentdata, N=256, gamma=1.0):
        super().__init__(name, N)
        self._segmentdata, self._gamma = segmentdata, gamma

    def _init(self):
        self._lut = np.ones((self.N + 3, 4), float)
        for k, c in enumerate(('red', 'green', 'blue')):
            self._lut[:-3, k] = create_lookup_table(self.N, self._segmentdata[c], self._gamma)
        if 'alpha' in self._segmentdata:
            self._lut[:-3, 3] = create_lookup_table(self.N, self._segmentdata['alpha'], 1.0)
        self._set_extremes()

    @staticmethod
    def from_list(name, colors, N=256, gamma=1.0):
        """(value, colour) pairs -> a map through those stops; an RGB colour gets alpha 1."""
        vals, colors = zip(*colors)
        rgba = np.array([tuple(c) + (1.0,) if len(c) == 3 else tuple(c) for c in colors], float)
        cdict = {k: np.column_stack([vals, rgba[:, i], rgba[:, i]]) for i, k in enumerate(('red', 'green', 'blue', 'alpha'))}
        return LinearSegmentedColormap(name, cdict, N, gamma)


class ListedColormap(Colormap):
    def __init__(self, colors, name='from_list', N=None):
        self.colors = np.asarray(colors, float)
        super().__init__(name, len(self.colors) if N is None else N)

    def _init(self):
        self._lut = np.zeros((self.N + 3, 4), float)
        rgba = self.colors if self.colors.shape[1] == 4 else np.column_stack([self.colors, np.ones(len(self.colors))])
        self._lut[:-3] = rgba
        self._set_extremes()


BONE_DATA = {'red': ((0., 0., 0.), (0.746032, 0.652778, 0.652778), (1.0, 1.0, 1.0)),
             'green': ((0., 0., 0.), (0.365079, 0.319444, 0.319444), (0.746032, 0.777778, 0.777778), (1.0, 1.0, 1.0)),
             'blue': ((0., 0., 0.), (0.365079, 0.444444, 0.444444), (1.0, 1.0, 1.0))}


def get_cmap(name, lut=None):
    """cm.get_cmap for 'bone' (a LinearSegmentedColormap, resampled to `lut` entries) and 'magma'.  run_inference.py never
    looks magma up, but utils.py builds it at import: here it is a grey 256-entry ListedColormap, not matplotlib's."""
    if name == 'bone':
        return LinearSegmentedColormap('bone', BONE_DATA, 256 if lut is None else lut)
    if name == 'magma':
        return ListedColormap(np.repeat(np.linspace(0, 1, 256)[:, None], 3, 1), 'magma')
    raise ValueError(name)


# ---- utils.py ---------------------------------------------------------------------------------------------------------
def opencv_rainbow(resolution=1000):
    """utils.py:18-28."""
    data = ((0.000, (1.00, 0.00, 0.00)), (0.400, (1.00, 1.00, 0.00)), (0.600, (0.00, 1.00, 0.00)),
            (0.800, (0.00, 0.00, 1.00)), (1.000, (0.60, 0.00, 1.00)))
    return LinearSegmentedColormap.from_list('opencv_rainbow', data, resolution)


COLORMAPS = {'rainbow': opencv_rainbow(), 'bone': get_cmap('bone', 10000)}


def tensor2array(tensor, max_value=None, colormap='rainbow'):
    """utils.py:36-47 for a [1,H,W] or [H,W] map: float32 [3,H,W]."""
    tensor = tensor.detach().cpu()
    if max_value is None:
        max_value = tensor.max().item()
    norm_array = tensor.squeeze().numpy() / max_value
    return COLORMAPS[colormap](norm_array).astype(np.float32)[:, :, :3].transpose(2, 0, 1)


def colorize(x, colormap, max_value=None):
    """(255 * tensor2array(x, max_value, colormap)).astype(np.uint8) as an HWC image."""
    return np.ascontiguousarray((255 * tensor2array(torch.as_tensor(x), max_value, colormap)).astype(np.uint8)
                                .transpose(1, 2, 0))


def uint8_table(name):
    """The uint8 [N,3] image of every colour of COLORMAPS[name], as (255 * ...).astype(np.uint8) makes it."""
    cm = COLORMAPS[name]
    cm(np.zeros(1, np.float32))
    return (255 * cm._lut[:cm.N, :3].astype(np.float32)).astype(np.uint8)


# ---- run_inference.py ---------------------------------------------------------------------------------------------------
def net_input(img, h=128, w=416, no_resize=False):
    """run_inference.py:58-67: a uint8 HxWx3 image -> [1,3,h,w] fp32, resized as imresize does to a float32 image unless
    no_resize or it is h x w already, then ((x/255 - 0.5)/0.2) by torch."""
    x = np.asarray(img).astype(np.float32)
    if not no_resize and x.shape[:2] != (h, w):
        x = imresize(x, (h, w)).astype(np.float32)
    t = torch.from_numpy(np.transpose(x, (2, 0, 1)).copy()).unsqueeze(0)
    return (t / 255 - 0.5) / 0.2


def images(disp):
    """run_inference.py:71-78 for one [1,H,W] disparity map: (disp image, depth image) uint8 HWC."""
    disp = torch.as_tensor(disp).float()
    return colorize(disp, 'bone'), colorize(1 / disp, 'rainbow', 10)


def dispnets_forward(p, x, alpha=10, beta=0.01):
    """DispNetS in eval mode (models/DispNetS.py:86-133): its disp1, in the dtype of x and p."""
    def conv(name, t, stride=1):
        w = p[name + '.weight']
        return F.relu(F.conv2d(t, w, p[name + '.bias'], stride, (w.shape[-1] - 1) // 2))

    def up(n, t):
        return F.relu(F.conv_transpose2d(t, p[f'upconv{n}.0.weight'], p[f'upconv{n}.0.bias'], stride=2, padding=1,
                                         output_padding=1))

    def pred(n, t):
        return alpha * torch.sigmoid(F.conv2d(t, p[f'predict_disp{n}.0.weight'], p[f'predict_disp{n}.0.bias'], 1, 1)) + beta

    def up2(d, ref):
        return _crop_like(F.interpolate(d, scale_factor=2, mode='bilinear', align_corners=False), ref)

    c = [x]
    for n in range(1, 8):
        c.append(conv(f'conv{n}.2', conv(f'conv{n}.0', c[-1], 2)))
    feat = c[7]
    disp = None
    for n in range(7, 0, -1):
        parts = [_crop_like(up(n, feat), c[n - 1])] + ([c[n - 1]] if n > 1 else [])
        if n <= 3:
            parts.append(up2(disp, c[n - 1]))
        feat = conv(f'iconv{n}.0', torch.cat(parts, 1))
        if n <= 4:
            disp = pred(n, feat)
    return disp
