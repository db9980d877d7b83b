"""Input pipeline on the device (SURVEY.md 8f N1): the reference's training transform
    Compose([RandomHorizontalFlip(), RandomScaleCrop(), ArrayToTensor(), Normalize(.5, .5)])      (train.py:165-172)
applied by ONE kernel (csrc/io_ops.cu: prep_frames_kernel) to uint8 frames that cross PCIe as uint8 - 4x fewer H2D
bytes than the fp32 tensors the reference's DataLoader ships (train.py:448-451) - plus the matching intrinsics
update (custom_transforms.py:47-58,98-118) and K^-1 (datasets/sequence_folders.py:51-61).

The random parameters are drawn on the host with the reference's own generators and call order
(random.random(); np.random.uniform(1, 1.1, 2); np.random.randint(...) twice), so a seeded run makes the same
augmentation decisions as the reference loader.

Documented deviation: the reference resizes with scipy.misc.imresize (PIL BILINEAR on uint8: fixed-point, the
horizontally and vertically resampled images are each rounded back to uint8); here the same half-pixel-centre
bilinear lookup is evaluated in fp32 without re-quantisation, so a pixel differs from the reference by at most
one uint8 step per pass (<= 2/255 before normalisation); with scale 1 the result is identical.

The reference's other transforms run on the device as well, bit-exact with Pillow (the library behind scipy.misc):
  * RandomRotate (custom_transforms.py:75-85, first in the train transform whenever the flow net trains, train.py:178-185):
    DeviceAugment(rotate=True) rotates the uint8 frames (csrc/io_ops.cu: ccb_rotate_frames_u8) before flip / scale-crop;
  * NormalizeLocally (custom_transforms.py:33-44, --data-normalization local): normalization='local' writes v/255
    (ccb_prep_frames_unit) and normalises each sample by its own per-channel mean and unbiased std over all its frames
    (ccb_normalize_local);
  * Scale(h, w) (custom_transforms.py:120-137, the validation-flow transform, train.py:189-190): scale_frames, behind
    DeviceScale, the validations and every evaluation's net input, stretches each uint8 frame to its own [min, max]
    (ccb_bytescale_u8), as scipy.misc.imresize does to the float32 copy the reference's loaders hand it (load_as_float),
    resamples it as Pillow's BILINEAR resize does (ccb_resize_u8, antialiased on a downscale), then normalises.
Documented deviation: scale_frames passes frames that already are h x w through as they are, as the reference's
evaluation scripts do (test_make3d.py:101, test_pose.py:54); its Scale would imresize them too, which stretches a frame
that does not span 0..255."""
import math
import random
import numpy as np
import torch
from . import _lib


def draw_params(B, Hs, Ws, H=None, W=None, rng_random=random, rng_np=np.random, flip=True, scale_crop=True, rotate=False):
    """Per-sample augmentation decisions, reference generators and order.  Returns a dict of numpy arrays."""
    H, W = H or Hs, W or Ws
    out = dict(flip=np.zeros(B, np.float32), x_scaling=np.ones(B), y_scaling=np.ones(B), scaled_h=np.full(B, Hs), scaled_w=np.full(B, Ws),
               offset_x=np.zeros(B, np.int32), offset_y=np.zeros(B, np.int32), rotate=np.zeros(B, bool), angle=np.zeros(B))
    for b in range(B):
        if rotate and not rng_np.random() > 0.5:                          # custom_transforms.py:78
            out['rotate'][b], out['angle'][b] = True, rng_np.uniform(0, 10)   # :82
        if flip and rng_random.random() < 0.5:                       # custom_transforms.py:52
            out['flip'][b] = 1.0
        if scale_crop:
            xs, ys = rng_np.uniform(1, 1.1, 2)                          # :107
            sh, sw = int(Hs * ys), int(Ws * xs)                          # :108
            out['x_scaling'][b], out['y_scaling'][b], out['scaled_h'][b], out['scaled_w'][b] = xs, ys, sh, sw
            out['offset_y'][b] = rng_np.randint(sh - H + 1)             # :117
            out['offset_x'][b] = rng_np.randint(sw - W + 1)             # :118
    return out


def pil_rotate_affine(angle, W, H):
    """The 6 coefficients Pillow's Image.rotate(angle) (no expand, centre (W/2, H/2)) hands its affine transform: output
    pixel centre (x, y) -> input point (a0 x + a1 y + a2, a3 x + a4 y + a5).  Restated from Pillow, including its
    rounding of cos / sin to 15 decimals, so that the device rotation samples the same points."""
    t = -math.radians(float(angle) % 360.0)
    m = [round(math.cos(t), 15), round(math.sin(t), 15), 0.0, round(-math.sin(t), 15), round(math.cos(t), 15), 0.0]
    cx, cy = W / 2, H / 2
    m[2], m[5] = m[0] * -cx + m[1] * -cy + m[2], m[3] * -cx + m[4] * -cy + m[5]
    m[2] += cx
    m[5] += cy
    return m


IDENTITY_AFFINE = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0]


def augment_intrinsics(K, p, Ws):
    """K [B,3,3] float32 numpy -> augmented K (custom_transforms.py:55,110-111,122-123), same fp32 arithmetic."""
    K = np.array(K, dtype=np.float32, copy=True)
    for b in range(K.shape[0]):
        if p['flip'][b]:
            K[b, 0, 2] = Ws - K[b, 0, 2]
        K[b, 0] *= p['x_scaling'][b]
        K[b, 1] *= p['y_scaling'][b]
        K[b, 0, 2] -= p['offset_x'][b]
        K[b, 1, 2] -= p['offset_y'][b]
    return K


NORMALIZATIONS = ('global', 'local')


def rotate_affines(p, B, Hs, Ws):
    """[B,6] fp64: Pillow's rotation matrix for the rotated samples of `p`, the identity for the others."""
    rot, ang = p.get('rotate', np.zeros(B, bool)), p.get('angle', np.zeros(B))
    return np.array([pil_rotate_affine(ang[b], Ws, Hs) if rot[b] else IDENTITY_AFFINE for b in range(B)], np.float64)


def to_device(a, device):
    """A host array or tensor -> `device`.  To a GPU it goes through pinned memory, asynchronously: the host does not wait
    for the device, and the caching host allocator keeps the pinned block until the copy has run."""
    t = torch.as_tensor(a)
    if torch.device(device).type == 'cuda' and not t.is_cuda:
        t = t.pin_memory()
    return t.to(device, non_blocking=True)


def device_tensor(a):
    """A tensor as it is (contiguous); a numpy array copied to the library's device (_lib.device())."""
    if torch.is_tensor(a):
        return a.contiguous()
    return torch.from_numpy(np.ascontiguousarray(a)).to(_lib.device())


def rotate_frames(src, affine):
    """src [B,F,H,W,3] uint8 on the device, affine [B,6] fp64 (host or device) -> rotated copy (ccb_rotate_frames_u8)."""
    B, F, H, W, _ = src.shape
    aff = to_device(torch.as_tensor(affine, dtype=torch.float64), src.device).contiguous()
    assert aff.shape == (B, 6)
    dst = torch.empty_like(src)
    _lib.call('ccb_rotate_frames_u8', src, aff, dst, B, F, H, W, src)
    return dst


def resize_frames(src, h, w):
    """src [..., Hs, Ws, 3] uint8 on the device -> [..., h, w, 3] uint8 resampled as Pillow's BILINEAR resize (ccb_resize_u8)."""
    Hs, Ws = src.shape[-3], src.shape[-2]
    N = src.numel() // (Hs * Ws * 3)
    dst = torch.empty(tuple(src.shape[:-3]) + (h, w, 3), dtype=torch.uint8, device=src.device)
    work, nb = _lib.workspace('ccb_resize_u8_workspace_bytes', N, Hs, Ws, h, w, like=src)
    _lib.call('ccb_resize_u8', src, dst, N, Hs, Ws, h, w, work, nb, src)
    return dst


def bytescale_frames(src):
    """src [..., H, W, 3] uint8 on the device -> the contrast stretch scipy.misc.imresize gives a float32 copy of each image
    before resizing it (scipy 1.1 bytescale: its [min, max] onto [0, 255] in float32), uint8 of the same shape
    (ccb_bytescale_u8)."""
    H, W = src.shape[-3], src.shape[-2]
    N = src.numel() // (H * W * 3)
    dst = torch.empty_like(src)
    work, nb = _lib.workspace('ccb_bytescale_u8_workspace_bytes', N, H, W, like=src)
    _lib.call('ccb_bytescale_u8', src, N, H, W, work, nb, dst, src)
    return dst


def normalize_local(frames):
    """NormalizeLocally (custom_transforms.py:33-44) in place on F tensors [B,3,H,W] (sample b's frames are frames[f][b]);
    returns the statistics [B,3,2] = {mean, unbiased std} per sample and channel (ccb_normalize_local)."""
    B, _, H, W = frames[0].shape
    F = len(frames)
    stats = torch.empty(B, 3, 2, device=frames[0].device)
    work, nb = _lib.workspace('ccb_normalize_local_workspace_bytes', B, H, W, like=frames[0])
    _lib.call('ccb_normalize_local', frames, B, F, H, W, stats, work, nb, frames[0])
    return stats


def _prep(src, par, offs, B, F, Hs, Ws, H, W, normalization):
    """uint8 [B,F,Hs,Ws,3] on the device -> F tensors [B,3,H,W]: flip / scale-crop lookup, ArrayToTensor, then Normalize(.5,
    .5) (global) or NormalizeLocally (local; returns its statistics, else None)."""
    outs = [torch.empty(B, 3, H, W, device=src.device) for _ in range(F)]
    fn = 'ccb_prep_frames' if normalization == 'global' else 'ccb_prep_frames_unit'
    _lib.call(fn, src, outs, par, offs, B, F, Hs, Ws, H, W, src)
    return outs, (normalize_local(outs) if normalization == 'local' else None)


class DeviceAugment:
    """frames_u8 [B,F,Hs,Ws,3] uint8 (pinned host or device) + intrinsics [B,3,3] -> (tgt, refs, K, Kinv) on `device`.

    The reference's train transform (train.py:165-185) with
      rotate        RandomRotate first (the flow net trains: no --fix-flownet): the uint8 frames are rotated into a device
                    scratch buffer, then flipped / scale-cropped.  As in the reference, rotation leaves the intrinsics
                    unchanged (custom_transforms.py:85 returns them as they came), although the rotated image no longer
                    fits them;
      normalization 'global' Normalize(.5, .5) or 'local' NormalizeLocally (--data-normalization); the statistics of the
                    last 'local' call are kept in `self.stats` ([B,3,2] = {mean, std}).
    With the defaults the launches and the output are those of the plain flip / scale-crop transform."""

    def __init__(self, device, H=None, W=None, flip=True, scale_crop=True, rotate=False, normalization='global'):
        assert normalization in NORMALIZATIONS, normalization
        self.device, self.H, self.W, self.flip, self.scale_crop = torch.device(device), H, W, flip, scale_crop
        self.rotate, self.normalization, self.stats = rotate, normalization, None

    def __call__(self, frames_u8, intrinsics, params=None, tgt_index=None):
        assert frames_u8.dtype == torch.uint8 and frames_u8.dim() == 5 and frames_u8.size(4) == 3
        B, F, Hs, Ws, _ = frames_u8.shape
        H, W = self.H or Hs, self.W or Ws
        p = params if params is not None else draw_params(B, Hs, Ws, H, W, flip=self.flip, scale_crop=self.scale_crop,
                                                          rotate=self.rotate)
        src = frames_u8.to(self.device, non_blocking=True).contiguous()
        if self.rotate:
            src = rotate_frames(src, rotate_affines(p, B, Hs, Ws))
        par = torch.from_numpy(np.stack([p['flip'], (p['scaled_w'] / Ws).astype(np.float32), (p['scaled_h'] / Hs).astype(np.float32),
                                         np.zeros(B, np.float32)], 1).astype(np.float32))
        par = to_device(par, self.device)
        offs = to_device(np.stack([p['offset_x'], p['offset_y']], 1).astype(np.int32), self.device)
        outs, self.stats = _prep(src, par, offs, B, F, Hs, Ws, H, W, self.normalization)
        K = augment_intrinsics(intrinsics.cpu().numpy() if torch.is_tensor(intrinsics) else intrinsics, p, Ws)
        Kinv = np.linalg.inv(K).astype(np.float32)                     # sequence_folders.py:61
        t = F // 2 if tgt_index is None else tgt_index                # sequence_folders.py:16-21: the target is the middle frame
        refs = [o for i, o in enumerate(outs) if i != t]
        return outs[t], refs, to_device(K, self.device), to_device(Kinv, self.device)


def scale_intrinsics(K, Hs, Ws, h, w):
    """K [B,3,3] -> Scale's intrinsics (custom_transforms.py:133-134): rows 0 / 1 times w/Ws, h/Hs in float32."""
    K = np.array(K, dtype=np.float32, copy=True)
    K[:, 0] *= np.float32(w / Ws)
    K[:, 1] *= np.float32(h / Hs)
    return K


def flow_intrinsics(K, Hs, Ws, h=256, w=832, device=None):
    """ValidationFlow's intrinsics after Scale (scale_intrinsics) and their float32 inverse (validation_flow.py:137),
    computed on the host from the raw K [B,3,3] -> (K, Kinv) fp32 on `device` (the library's device by default)."""
    K = scale_intrinsics(K.cpu().numpy() if torch.is_tensor(K) else K, Hs, Ws, h, w)
    Kinv = np.linalg.inv(K).astype(np.float32)
    dev = device or _lib.device()
    return torch.from_numpy(K).to(dev), torch.from_numpy(Kinv).to(dev)


def scale_frames(frames_u8, h, w, normalization='global'):
    """Compose([Scale(h, w), ArrayToTensor(), normalize]) on the frames: uint8 [B,F,Hs,Ws,3] (a numpy array goes to the
    library's device) -> F tensors [B,3,h,w] and the 'local' statistics (None for 'global'), as _prep returns them.
    Where (Hs, Ws) != (h, w) each frame is stretched (bytescale_frames) and resized (resize_frames) as imresize does to
    a float32 frame; frames already h x w go through as they are.  The identity lookup parameters are filled on the
    device, so the call makes no host synchronisation and can be captured in a CUDA graph."""
    assert normalization in NORMALIZATIONS, normalization
    src = device_tensor(frames_u8)
    assert src.dtype == torch.uint8 and src.dim() == 5 and src.size(4) == 3, (src.dtype, src.shape)
    B, F, Hs, Ws = (int(v) for v in src.shape[:4])
    if (Hs, Ws) != (h, w):
        src = resize_frames(bytescale_frames(src), h, w)
    par = torch.zeros(B, 4, device=src.device)                 # no flip, scale 1
    par[:, 1:3] = 1.0
    offs = torch.zeros(B, 2, dtype=torch.int32, device=src.device)
    return _prep(src, par, offs, B, F, h, w, h, w, normalization)


class DeviceScale:
    """The validation-flow transform Compose([Scale(h, w), ArrayToTensor(), normalize]) (train.py:189-190):
    frames_u8 [B,F,Hs,Ws,3] uint8 + intrinsics [B,3,3] -> (tgt, refs, K, Kinv) on `device`.  The frames go through
    scale_frames ('global' or 'local', as DeviceAugment; the statistics of the last 'local' call are kept in
    `self.stats`), K and K^-1 through flow_intrinsics.  The target is frame 0: validation_flow.py:130-133 orders the frames
    [tgt] + refs."""

    def __init__(self, device, h=256, w=832, normalization='global'):
        assert normalization in NORMALIZATIONS, normalization
        self.device, self.h, self.w, self.normalization, self.stats = torch.device(device), h, w, normalization, None

    def __call__(self, frames_u8, intrinsics, tgt_index=0):
        Hs, Ws = frames_u8.shape[2:4]
        outs, self.stats = scale_frames(frames_u8.to(self.device, non_blocking=True), self.h, self.w, self.normalization)
        K, Kinv = flow_intrinsics(intrinsics, Hs, Ws, self.h, self.w, self.device)
        refs = [o for i, o in enumerate(outs) if i != tgt_index]
        return outs[tgt_index], refs, K, Kinv
