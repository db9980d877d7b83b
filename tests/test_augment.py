"""The reference's remaining data transforms (RandomRotate, NormalizeLocally, Scale) without a GPU: the io_ops.cu kernels
compiled for the CPU simulator (tests/sim) against the fixture frozen from the reference and against Pillow itself on
random images, the numpy restatements of Pillow against Pillow, and the host-side parameter draw.  The same fixture cases
and the full-size ones run on the H100 in tests/test_gpu_augment.py."""
import random
import numpy as np
import pytest
import torch

from cc_b200 import input_pipeline as CI
from tests import augment_cases as AC, augment_oracle as AO
from tests.util import sim_lib      # noqa: F401  (module fixture: the simulator library)

CPU = torch.device('cpu')
ROTATE_CASES = [((23, 37), a) for a in (0.2, 1.5, 4.4, 8.05, 9.9)] + [((12, 9), 6.1), ((1, 5), 3.0)]
RESIZE_CASES = [((30, 50), (20, 34)), ((19, 23), (31, 40)), ((16, 40), (16, 27)), ((20, 20), (13, 20)), ((9, 11), (9, 11)),
                ((40, 7), (6, 3)), ((5, 6), (17, 29))]


@pytest.mark.parametrize('case', AC.AUGMENT_CASES, ids=lambda f: f.__name__)
def test_augment_case(case, sim_lib):
    case(CPU)


def _pillow():
    return pytest.importorskip('PIL.Image')


@pytest.mark.parametrize('shape,angle', ROTATE_CASES, ids=['%dx%d-%g' % (s + (a,)) for s, a in ROTATE_CASES])
def test_rotate_kernel_vs_pillow(shape, angle, sim_lib):
    Image = _pillow()
    H, W = shape
    im = np.random.RandomState(int(angle * 100) + H).randint(0, 256, size=(2, 1, H, W, 3)).astype(np.uint8)
    aff = [CI.pil_rotate_affine(angle, W, H), CI.IDENTITY_AFFINE]
    got = CI.rotate_frames(torch.from_numpy(im), aff).numpy()
    assert np.array_equal(got[0, 0], np.array(Image.fromarray(im[0, 0]).rotate(angle, resample=Image.BILINEAR)))
    assert np.array_equal(got[1], im[1]), 'the identity must reproduce the frame'


@pytest.mark.parametrize('src,dst', RESIZE_CASES, ids=['%dx%d-%dx%d' % (s + d) for s, d in RESIZE_CASES])
def test_resize_kernel_vs_pillow(src, dst, sim_lib):
    Image = _pillow()
    (Hs, Ws), (h, w) = src, dst
    im = np.random.RandomState(Hs * Ws + h).randint(0, 256, size=(2, Hs, Ws, 3)).astype(np.uint8)
    got = CI.resize_frames(torch.from_numpy(im), h, w).numpy()
    for n in range(2):
        assert np.array_equal(got[n], np.array(Image.fromarray(im[n]).resize((w, h), Image.BILINEAR))), n


def test_oracle_vs_pillow():
    """tests/augment_oracle.py, used where Pillow is not at hand, against Pillow at KITTI and training sizes."""
    Image = _pillow()
    rs = np.random.RandomState(12)
    for (Hs, Ws), (h, w) in (((375, 1242), (256, 832)), ((370, 1226), (256, 832)), ((128, 416), (136, 446)),
                             ((256, 832), (281, 915))):
        im = rs.randint(0, 256, size=(Hs, Ws, 3)).astype(np.uint8)
        assert np.array_equal(AO.resize_u8(im, h, w), np.array(Image.fromarray(im).resize((w, h), Image.BILINEAR))), (Hs, Ws, h, w)
    im = rs.randint(0, 256, size=(37, 53, 3)).astype(np.uint8)
    for angle in (7.3, 0.01, 5.0):
        want = np.array(Image.fromarray(im).rotate(angle, resample=Image.BILINEAR))
        assert np.array_equal(AO.rotate_u8(im, CI.pil_rotate_affine(angle, 53, 37)), want), angle


def test_normalize_local_kernel_vs_oracle(sim_lib):
    """Two samples, three frames each: statistics over all frames of a sample, per channel; the second sample's first
    channel is constant, so its std is 0 and the frames become nan, as the reference's do."""
    rs = np.random.RandomState(5)
    x = rs.rand(3, 2, 3, 7, 11).astype(np.float32)
    x[:, 1, 0] = 0.25
    frames = [torch.from_numpy(x[f].copy()) for f in range(3)]
    stats = CI.normalize_local(frames).numpy()
    got = np.stack([f.numpy() for f in frames], 1)
    for b in range(2):
        wo, wm, ws = AO.normalize_locally(x[:, b])
        assert np.all(np.abs(stats[b, :, 0] - wm) <= np.spacing(np.abs(wm))), (stats[b], wm)
        assert np.all(np.abs(stats[b, :, 1] - ws) <= np.spacing(np.abs(ws))), (stats[b], ws)
        assert np.array_equal(got[b], wo, equal_nan=True)
    assert stats[1, 0, 1] == 0 and np.isnan(got[1, :, 0]).all()


def test_draw_params_rotate_order():
    """rotate=True draws np.random.random() (and np.random.uniform(0, 10) when it is <= .5) for a sample before its flip
    draw; rotate=False leaves the draw sequence as it was."""
    random.seed(1)
    np.random.seed(2)
    p0 = CI.draw_params(3, 40, 60)
    random.seed(1)
    np.random.seed(2)
    p1 = CI.draw_params(3, 40, 60, rotate=True)
    random.seed(1)
    np.random.seed(2)
    p2 = CI.draw_params(3, 40, 60)
    assert all(np.array_equal(p0[k], p2[k]) for k in p0) and not p0['rotate'].any()
    np.random.seed(2)
    for b in range(3):
        r = np.random.random()
        assert p1['rotate'][b] == (r <= 0.5)
        if r <= 0.5:
            assert p1['angle'][b] == np.random.uniform(0, 10)
        xs, ys = np.random.uniform(1, 1.1, 2)
        assert p1['x_scaling'][b] == xs and p1['y_scaling'][b] == ys
        np.random.randint(int(40 * ys) - 40 + 1)
        np.random.randint(int(60 * xs) - 60 + 1)
    assert np.array_equal(p1['flip'], p0['flip'])


def test_pil_rotate_affine():
    """The identity at angle 0; a rotation about the frame centre otherwise (the centre maps to itself)."""
    assert np.array_equal(CI.pil_rotate_affine(0.0, 40, 30), CI.IDENTITY_AFFINE)
    a = CI.pil_rotate_affine(7.0, 40, 30)
    assert abs(a[0] * 20 + a[1] * 15 + a[2] - 20) < 1e-12 and abs(a[3] * 20 + a[4] * 15 + a[5] - 15) < 1e-12
    assert a[0] == a[4] == round(np.cos(np.radians(7.0)), 15)


def test_device_classes_validate_normalization():
    with pytest.raises(AssertionError):
        CI.DeviceAugment('cpu', normalization='batch')
    with pytest.raises(AssertionError):
        CI.DeviceScale('cpu', normalization='none')
