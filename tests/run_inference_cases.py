"""Cases of run_inference on the device (cc_b200.evaluate.colorize over ccb_colorize, the 'inference' normalisation of
input_pipeline.scale_frames over ccb_prep_frames_inference, cc_b200.run_inference.infer and main()), run on the CPU
simulator build (tests/test_run_inference.py) and on the H100 (tests/test_gpu_run_inference.py).

The references are tests/golden/run_inference_small.npz (the reference's own run_inference.main() on the folder written
here, tests/golden/make_run_inference.py) and the oracle restatement (oracle/run_inference.py).  The builders of the
folder live here so that the fixture maker and the tests write the same files."""
import os
import numpy as np
import torch
from cc_b200 import evaluate as CE, models as CM, run_inference as RI, synth
from cc_b200.input_pipeline import scale_frames
from oracle import run_inference as ORI
from tests.util import golden

FIXTURE = 'run_inference_small'
SIZE = (64, 128)                 # --img-height, --img-width of the runs: small enough for the simulator
CKPT_SEED = 23
# the folder: name -> (height, width, seed); two sizes, one of them the target size, PNG and JPEG
PHOTOS = {'a.png': (64, 128, 1), 'b.png': (80, 150, 2), 'c.jpg': (80, 150, 3), 'sub/b.png': (64, 128, 4)}
LIST = ['c.jpg', 'sub/b.png', 'a.png', 'b.png']        # sub/b.png and b.png write the same files: the later one wins
RUNS = {
    'glob': ['--output-disp', '--output-depth', '--pretrained', 'ckpt.pth.tar', '--img-height', '64', '--img-width',
             '128', '--dataset-dir', 'photos', '--output-dir', 'out'],
    'list': ['--output-disp', '--output-depth', '--pretrained', 'ckpt.pth.tar', '--img-height', '64', '--img-width',
             '128', '--dataset-dir', 'photos', '--dataset-list', 'list.txt', '--output-dir', 'out', '--img-exts', 'jpg'],
    'noresize_depth': ['--output-depth', '--pretrained', 'ckpt.pth.tar', '--no-resize', '--img-exts', 'jpg', 'png',
                       '--dataset-dir', 'photos', '--output-dir', 'out'],
    'none': ['--pretrained', 'ckpt.pth.tar', '--dataset-dir', 'photos', '--output-dir', 'out'],
}


def g():
    return golden(FIXTURE)


def photo(h, w, seed):
    """A smooth photo-like uint8 image that does not span 0..255, so that imresize's contrast stretch matters."""
    rs = np.random.RandomState(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    base = np.stack([np.sin(x / (7 + c) + seed) * np.cos(y / (5 + 2 * c)) for c in range(3)], 2)
    img = 110 + 70 * base + rs.randn(h, w, 3) * 12
    return np.clip(img, 20 + seed, 230).astype(np.uint8)


def checkpoint():
    """The seeded DispNetS checkpoint of the runs: {'state_dict': ...}, the same weights as the reference's module gets."""
    return {'state_dict': synth.seeded_fill(CM.DispNetS(), CKPT_SEED).state_dict()}


def write_work_dir(root):
    """root/photos (PHOTOS), root/list.txt (LIST) and root/ckpt.pth.tar."""
    from PIL import Image
    for name, (h, w, seed) in PHOTOS.items():
        p = os.path.join(root, 'photos', name)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        Image.fromarray(photo(h, w, seed)).save(p)
    with open(os.path.join(root, 'list.txt'), 'w') as f:
        f.write('\n'.join(LIST) + '\n')
    torch.save(checkpoint(), os.path.join(root, 'ckpt.pth.tar'))


def to(device, a):
    return torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a).to(device)


# ---- colormaps ------------------------------------------------------------------------------------------------------
def case_tables(device):
    """The product's uint8 tables equal the fixture's stand-in tables and the oracle's."""
    d = g()
    for name in ('bone', 'rainbow'):
        got = CE.colormap_table(name)
        assert got.dtype == np.uint8 and np.array_equal(got, d['table_' + name]), name
        assert np.array_equal(got, ORI.uint8_table(name)), name


def edge_maps():
    """[4,6,7] maps: x == max, x above the fixed max, 0, negatives, +inf (from 1/0), NaN, bin edges; an all-zero image;
    images whose maxima differ by orders of magnitude."""
    rs = np.random.RandomState(9)
    m = rs.uniform(0.01, 12, (4, 6, 7)).astype(np.float32)
    m[0, 0, :6] = [10.0, 10.5, 0.0, -0.0, -3.0, np.inf]
    m[0, 1, :3] = [np.nan, 1e-30, 9.9999]
    m[0, 2, :4] = np.float32([0.1, 0.2, 0.3, 0.7]) * 10       # rainbow bin edges at max_value 10
    m[1] = 0.0
    m[2] *= 1e-3
    m[3, 0, 0] = m[3].max() * 4
    return m


def check_colorize(device, maps):
    """colorize against the oracle's tensor2array image by image, for both maps, per-image and fixed scales, inverted or
    not, at batch B and one image at a time."""
    x = to(device, maps)
    for colormap, max_value, invert in (('bone', None, False), ('rainbow', 10, True), ('rainbow', None, False),
                                        ('bone', 10, True), ('bone', 2.5, False)):
        got = CE.colorize(x, colormap, max_value, invert).cpu().numpy()
        assert got.shape == maps.shape + (3,) and got.dtype == np.uint8
        for b in range(maps.shape[0]):
            t = torch.from_numpy(maps[b:b + 1])
            want = ORI.colorize(1 / t if invert else t, colormap, max_value)
            bad = (got[b] != want).any(-1)
            assert not bad.any(), '%s max %s invert %s image %d: %d pixels differ, first at %s' % (
                colormap, max_value, invert, b, bad.sum(), np.argwhere(bad)[0])
            one = CE.colorize(x[b:b + 1], colormap, max_value, invert).cpu().numpy()[0]
            assert np.array_equal(one, got[b])


def case_colorize_edges(device):
    check_colorize(device, edge_maps())
    nan_img = edge_maps()[:1].copy()
    got = CE.colorize(to(device, nan_img), 'bone').cpu().numpy()
    assert not got.any(), 'a NaN anywhere makes the per-image maximum NaN: the whole image is black'


def case_colorize_fixture(device):
    """The fixture's disparity maps, as the script colours them (bone scaled by its maximum, rainbow of 1/disp at 10),
    against the fixture's imsave arrays."""
    d = g()
    for run in ('glob', 'list'):
        n = len([k for k in d if k.startswith(run + '_disp_')])
        disp = np.concatenate([d['%s_disp_%d' % (run, k)][:, 0] for k in range(n)])
        got_d = CE.colorize(to(device, disp), 'bone').cpu().numpy()
        got_z = CE.colorize(to(device, disp), 'rainbow', 10, invert=True).cpu().numpy()
        for k in range(n):
            assert np.array_equal(got_d[k], d['%s_saved_%d' % (run, 2 * k)].transpose(1, 2, 0)), (run, k)
            assert np.array_equal(got_z[k], d['%s_saved_%d' % (run, 2 * k + 1)].transpose(1, 2, 0)), (run, k)
        check_colorize(device, disp)


def case_colorize_arg_errors(device):
    """Null pointers, bad sizes, a bad table size and a short workspace return CCB_ERR_ARG and launch nothing."""
    from cc_b200 import _lib
    lib = _lib.lib()
    B, H, W = 2, 5, 6
    maps = torch.rand(B, H, W, device=device)
    lut = torch.zeros(10, 3, dtype=torch.uint8, device=device)
    out = torch.zeros(B, H, W, 3, dtype=torch.uint8, device=device)
    nb = lib.ccb_colorize_workspace_bytes(B, H, W, 1)
    assert nb == 8 * B and lib.ccb_colorize_workspace_bytes(B, H, W, 0) == 0
    work = torch.zeros(B, dtype=torch.int64, device=device)
    good = dict(maps=maps.data_ptr(), B=B, H=H, W=W, lut=lut.data_ptr(), N=10, invert=0, per=1, mx=_c_float(0.0),
                work=work.data_ptr(), nb=nb, out=out.data_ptr(), stream=_lib.stream(maps))
    before = lib.ccb_launch_count()
    for change in [dict(maps=None), dict(lut=None), dict(out=None), dict(B=0), dict(H=0), dict(W=-1), dict(N=0),
                   dict(work=None), dict(nb=nb - 1)]:
        assert lib.ccb_colorize(*dict(good, **change).values()) == -1, change
        assert lib.ccb_last_error_string().startswith(b'colorize')
    assert lib.ccb_launch_count() == before and not out.any()
    assert lib.ccb_colorize_workspace_bytes(0, H, W, 1) == -1


def _c_float(v):
    import ctypes
    return ctypes.c_float(v)


# ---- normalisation and the pipeline ---------------------------------------------------------------------------------
def case_inference_normalisation(device):
    """All 256 levels at the frame's own size: ((x/255 - 0.5)/0.2) of torch's CPU ops in fp32, bit for bit; the other
    normalisations are unchanged."""
    levels = np.arange(256, dtype=np.uint8)
    frame = np.stack([levels, levels[::-1], np.roll(levels, 7)], 1).reshape(16, 16, 3)
    x = scale_frames(to(device, frame[None, None]), 16, 16, 'inference')[0][0].cpu()
    t = torch.from_numpy(frame.astype(np.float32).transpose(2, 0, 1).copy())[None]
    want = (t / 255 - 0.5) / 0.2
    assert torch.equal(x.view(torch.int32), want.view(torch.int32))
    g5 = scale_frames(to(device, frame[None, None]), 16, 16, 'global')[0][0].cpu()
    assert torch.equal(g5, (t / 255 - 0.5) / 0.5)


def case_net_input(device):
    """The net input of both photo sizes (stretched and resized, or passed through) equals the oracle's net_input."""
    for name, (h, w, seed) in PHOTOS.items():
        img = photo(h, w, seed)
        for no_resize in (False, True):
            hh, ww = (h, w) if no_resize else SIZE
            got = scale_frames(to(device, img[None, None]), hh, ww, 'inference')[0][0].cpu()
            want = ORI.net_input(img, SIZE[0], SIZE[1], no_resize)
            assert torch.equal(got, want), (name, no_resize)


ALL_CASES = [case_tables, case_colorize_edges, case_colorize_fixture, case_colorize_arg_errors,
             case_inference_normalisation, case_net_input]


# ---- the command ----------------------------------------------------------------------------------------------------
def disp_tolerance(disp):
    """The conv engine's fp32 tolerance on a disparity map, relative to its largest value (tests/eval_cases.py's 1e-4 bar
    for a forward, doubled)."""
    return 2e-4 * float(np.abs(disp).max())


def check_image(got, want, disp, colormap, max_value, invert, tol, what):
    """got == want, except pixels whose two colours are adjacent bins of the table where the disparity lies within tol of
    the edge between them (measured on the disparity axis) -> the number of such pixels."""
    bad = (got != want).any(-1)
    if not bad.any():
        return 0
    N = CE.COLORMAPS[colormap][1]
    d = disp.astype(np.float64)
    v = 1 / d if invert else d
    mx = float(max_value) if max_value is not None else float(v.max())
    e = np.clip(np.round(v / mx * N), 1, N - 1)
    ve = e * mx / N
    de = 1 / ve if invert else ve
    table = CE.colormap_table(colormap)
    e = e.astype(np.int64)
    lo, hi = table[e - 1], table[e]
    adjacent = (np.all(got == lo, -1) | np.all(got == hi, -1)) & (np.all(want == lo, -1) | np.all(want == hi, -1))
    ok = adjacent & (np.abs(de - d) <= tol)
    assert ok[bad].all(), '%s: %d of %d differing pixels are not one bin apart at a bin edge' % (
        what, (~ok[bad]).sum(), bad.sum())
    return int(bad.sum())


def run_main(tmp, run, device, workers=2, capsys=None):
    """main() on a fresh copy of the work folder with RUNS[run] -> (result, stdout, output folder)."""
    write_work_dir(str(tmp))
    cwd = os.getcwd()
    os.chdir(str(tmp))
    try:
        res = RI.main(RUNS[run], device=device, workers=workers)
    finally:
        os.chdir(cwd)
    out = capsys.readouterr().out if capsys is not None else None
    return res, out, os.path.join(str(tmp), 'out')


def case_main(device, tmp, capsys, run):
    """main() on the fixture's folder: the printed lines and the files.  The images are those infer() makes of the same
    photos; each equals the reference's imsave array (transposed to HWC) or is one bin apart where the disparity lies
    within the conv engine's tolerance of the bin edge.  PNG files decode to infer()'s image; JPEG files are Pillow's
    encoding of it, byte for byte, and so of the reference's array wherever the two arrays are equal.
    Returns the number of pixels one bin apart."""
    import io
    from PIL import Image
    d = g()
    res, out, odir = run_main(tmp, run, device, capsys=capsys)
    assert out == str(d[run + '_stdout']), (out, str(d[run + '_stdout']))
    names = [str(n) for n in d[run + '_saved_names']]
    if run == 'none':
        assert res is None and not names and not os.path.exists(odir)
        return 0
    final = {n: k for k, n in enumerate(names)}
    assert sorted(os.listdir(odir)) == sorted(final), (os.listdir(odir), sorted(final))
    assert sorted(os.path.relpath(p, 'out') for p in res['written']) == sorted(final)      # main() ran in tmp
    argv = RUNS[run]
    kinds = [k for k in ('disp', 'depth') if '--output-' + k in argv]
    size = (int(argv[argv.index('--img-height') + 1]), int(argv[argv.index('--img-width') + 1])) if '--img-height' in argv \
        else (128, 416)
    frames = [RI.decode(os.path.join(str(tmp), f)) for f in res['files']]
    net = RI.load_disp_net(checkpoint(), 'DispNetS', device)
    prod = RI.infer(net, frames, *size, no_resize='--no-resize' in argv, output_disp='disp' in kinds,
                    output_depth='depth' in kinds)
    # a --dataset-dir folder is listed in os.listdir order, which differs between file systems: the fixture holds the
    # order of the machine that made it, so each image is matched by its output name - the last photo that writes it
    source = {}
    for i, f in enumerate(res['files']):
        for kind, p in zip(('disp', 'depth'), RI.output_names(f, 'out')):
            if kind in kinds:
                source[os.path.basename(p)] = (i, kind)
    assert sorted(source) == sorted(final), (sorted(source), sorted(final))
    differing = 0
    for n, k in final.items():
        i, kind = source[n]
        assert kind == kinds[k % len(kinds)], (n, kind)
        disp = d['%s_disp_%d' % (run, k // len(kinds))][0, 0]
        want = np.ascontiguousarray(d['%s_saved_%d' % (run, k)].transpose(1, 2, 0))
        got = prod[i][kind].cpu().numpy()
        cm, mv, inv = ('bone', None, False) if kind == 'disp' else ('rainbow', 10, True)
        differing += check_image(got, want, disp, cm, mv, inv, 2 * disp_tolerance(disp), '%s %s' % (run, n))
        path = os.path.join(odir, n)
        if n.endswith('.jpg'):
            buf = io.BytesIO()
            Image.fromarray(got).save(buf, format='JPEG')
            with open(path, 'rb') as f:
                data = f.read()
            assert data == buf.getvalue(), n
            if np.array_equal(got, want):
                buf = io.BytesIO()
                Image.fromarray(want).save(buf, format='JPEG')
                assert data == buf.getvalue(), n
        else:
            assert np.array_equal(np.asarray(Image.open(path)), got), n
    return differing


def case_refusal(device, tmp, capsys, mode):
    """An RGBA or greyscale photo is refused, and the message names it."""
    import pytest
    from PIL import Image
    write_work_dir(str(tmp))
    p = os.path.join(str(tmp), 'photos', 'odd.png')
    img = photo(64, 128, 8)
    Image.fromarray(np.concatenate([img, img[:, :, :1]], 2) if mode == 'RGBA' else img[:, :, 0]).save(p)
    cwd = os.getcwd()
    os.chdir(str(tmp))
    try:
        with pytest.raises(ValueError, match='odd.png'):
            RI.main(RUNS['glob'], device=device, workers=1)
    finally:
        os.chdir(cwd)


def kitti_case(device, name, sizes=((375, 1242), (376, 1241)), target=(128, 416), n=1, seed=60):
    """KITTI-size frames through infer() with a seeded net: the disparity within the conv tolerance of the oracle's fp64
    forward (DispNetS: oracle.run_inference.dispnets_forward; DispResNet6: oracle.nets.disp_forward), and every pixel of
    both images equal to the oracle's tensor2array of the fp64 disparity or one bin apart at a bin edge."""
    from oracle import nets as ON
    net = synth.seeded_fill(getattr(CM, name)(), seed).to(device)
    p = {k: v.detach().cpu().double() for k, v in net.state_dict().items()}
    frames = [photo(h, w, seed + k) for k, (h, w) in enumerate(sizes) for _ in range(n)]
    res = RI.infer(net, frames, *target)
    for k, img in enumerate(frames):
        x = ORI.net_input(img, *target).double()
        with torch.no_grad():
            ref = ORI.dispnets_forward(p, x) if name == 'DispNetS' else ON.disp_forward(p, x, training=False)
        ref = ref[0].float()
        got = res[k]['disp_map'].cpu()
        tol = disp_tolerance(ref.numpy())
        assert (got - ref[0]).abs().max().item() <= tol, (name, k, (got - ref[0]).abs().max().item(), tol)
        want_d, want_z = ORI.images(ref)
        dref = ref[0].numpy()
        check_image(res[k]['disp'].cpu().numpy(), want_d, dref, 'bone', None, False, tol, '%s %d disp' % (name, k))
        check_image(res[k]['depth'].cpu().numpy(), want_z, dref, 'rainbow', 10, True, tol, '%s %d depth' % (name, k))
