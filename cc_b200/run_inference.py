"""The reference's run_inference.py on this stack: `python -m cc_b200.run_inference --pretrained CKPT --output-disp
--output-depth --dataset-dir DIR --output-dir OUT` writes, for each photo, its disparity as {stem}_disp{ext} (the bone
colormap scaled by the image's own maximum) and its depth 1/disparity as {stem}_depth{ext} (the rainbow colormap,
max_value 10), the images utils.tensor2array gives.

  files       --dataset-list (each line joined to --dataset-dir) or, for each --img-exts in turn, the files of
              --dataset-dir matching *.{ext} in os.listdir order, as path.py's files() lists them.
  decode      host worker processes decode the photos (np.asarray(Image.open(p)), what scipy.misc.imread returned), a
              chunk ahead of the device.
  device      infer(): the frames of a chunk grouped by size; a group that is not --img-height x --img-width (and
              without --no-resize) is contrast-stretched and resized as scipy.misc.imresize does to a float32 image
              (input_pipeline.scale_frames), then normalised as (x/255 - 0.5)/0.2; the net runs in eval mode on the
              whole group; evaluate.colorize makes each kind of image in one call.
  encode      the workers write the images with Pillow (Image.fromarray(hwc).save(p)).  Where two photos give the same
              output name, the later one's image is the file, as in the reference, which writes them in order.

Extension: --dispnet picks the architecture of the checkpoint: DispNetS (the default, the reference's only choice),
DispNetS6, DispResNet6 (Competitive Collaboration's own disparity checkpoints) or DispResNetS6.

Documented deviations:
  image layout  the reference hands scipy.misc.imsave the [3,H,W] array tensor2array returns.  scipy 1.1's imsave calls
                toimage(arr, channel_axis=2), which takes axis 2, the width, as the channels and raises ValueError unless
                the width is 3 or 4; the script as committed therefore writes no image of a real photo.  Here the
                H x W x 3 colour image the script means to write is saved.
  refusal       a file that does not decode to H x W x 3 uint8 (greyscale, RGBA, 16-bit) is refused with an error that
                names it; the reference crashes on it, inside the net for RGBA.
  batching      the frames of one size run through the net together; the reference runs one image at a time."""
import argparse
import contextlib
import fnmatch
import multiprocessing
import os
import sys
import numpy as np

DISPNETS = ('DispNetS', 'DispNetS6', 'DispResNet6', 'DispResNetS6')
CHUNK = 64                      # photos decoded ahead of the device: 64 KITTI frames are 89 MB of uint8
WORKERS = 4


def build_parser():
    p = argparse.ArgumentParser(description='Inference script for DispNet learned with Structure from Motion Learner '
                                            'inference on KITTI and CityScapes Dataset',
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    a = p.add_argument
    a('--output-disp', action='store_true', help='save disparity img')
    a('--output-depth', action='store_true', help='save depth img')
    a('--pretrained', required=True, type=str, help='pretrained DispNet path')
    a('--img-height', default=128, type=int, help='Image height')
    a('--img-width', default=416, type=int, help='Image width')
    a('--no-resize', action='store_true', help='no resizing is done')
    a('--dataset-list', default=None, type=str, help='Dataset list file')
    a('--dataset-dir', default='.', type=str, help='Dataset directory')
    a('--output-dir', default='output', type=str, help='Output directory')
    a('--img-exts', default=['png', 'jpg', 'bmp'], nargs='*', type=str, help='images extensions to glob')
    a('--dispnet', default='DispNetS', choices=DISPNETS, help='architecture of the pretrained disparity net')
    return p


def load_disp_net(weights, name='DispNetS', device=None):
    """The disparity net `name` in eval mode on `device`: weights a checkpoint path or the loaded dict holding 'state_dict',
    loaded strictly."""
    import torch
    from . import models
    assert name in DISPNETS, name
    if not isinstance(weights, dict):
        weights = torch.load(weights, map_location='cpu')
    net = getattr(models, name)()
    net.load_state_dict(weights['state_dict'])
    return net.to(device or torch.device('cuda')).eval()


def test_files(dataset_dir, dataset_list=None, img_exts=('png', 'jpg', 'bmp')):
    """run_inference.py:48-52: the list's lines joined to dataset_dir, or for each extension in turn the files of
    dataset_dir matching '*.ext' in os.listdir order."""
    if dataset_list is not None:
        with open(dataset_list, 'r') as f:
            return [os.path.join(dataset_dir, line) for line in f.read().splitlines()]
    names = os.listdir(dataset_dir)
    return [os.path.join(dataset_dir, n) for ext in img_exts for n in names
            if fnmatch.fnmatch(n, '*.{}'.format(ext)) and os.path.isfile(os.path.join(dataset_dir, n))]


def output_names(file, output_dir):
    """(disp file, depth file) of a photo: {namebase}_disp{ext} and {namebase}_depth{ext} under output_dir."""
    stem, ext = os.path.splitext(os.path.basename(file))
    return os.path.join(output_dir, '{}_disp{}'.format(stem, ext)), os.path.join(output_dir, '{}_depth{}'.format(stem, ext))


# ---- host workers ------------------------------------------------------------------------------------------------------
def decode(path):
    """One photo in a worker: np.asarray(Image.open(path)), refused unless it is H x W x 3 uint8."""
    from PIL import Image
    with Image.open(path) as im:
        img = np.asarray(im)
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
        raise ValueError('%s: run_inference needs an 8-bit RGB image, this one decodes to %s %s'
                         % (path, img.dtype, img.shape))
    return img


def encode(path, img):
    """imsave of an H x W x 3 uint8 image (Pillow, its default settings for the extension)."""
    from PIL import Image
    Image.fromarray(img).save(path)


@contextlib.contextmanager
def worker_pool(workers):
    """`workers` spawned host processes for the block: closed when it ends, terminated when it raises, and joined before
    the block is left either way."""
    pool = multiprocessing.get_context('spawn').Pool(workers)
    try:
        yield pool
        pool.close()
    except BaseException:
        pool.terminate()
        raise
    finally:
        pool.join()


def chunks_ahead(pool, fn, chunks):
    """pool.map(fn, chunk) of each chunk in turn, the next chunk handed to the workers before this one is yielded: the
    host work of chunk k + 1 overlaps the device work of chunk k."""
    pending = pool.map_async(fn, chunks[0]) if chunks else None
    for k in range(len(chunks)):
        res = pending.get()
        pending = pool.map_async(fn, chunks[k + 1]) if k + 1 < len(chunks) else None
        yield res


def host_arrays(tensors):
    """Device tensors of any shapes -> numpy arrays of the same shapes, in one device-to-host copy."""
    import torch
    flat = torch.cat([t.reshape(-1) for t in tensors]).cpu().numpy()
    ends = np.cumsum([t.numel() for t in tensors])
    return [a.reshape(t.shape) for a, t in zip(np.split(flat, ends[:-1]), tensors)]


# ---- device ------------------------------------------------------------------------------------------------------------
def infer(disp_net, frames, img_height=128, img_width=416, no_resize=False, output_disp=True, output_depth=True):
    """run_inference.py:56-78 for a list of uint8 H x W x 3 frames (numpy or device tensors, any sizes) -> one dict per
    frame of device tensors: 'disp_map' the net's disparity [h,w] fp32, and as asked 'disp' (bone, scaled by the map's
    own maximum) and 'depth' (rainbow of 1/disparity, max_value 10), uint8 [h,w,3].  Frames of one size form one group:
    one stretch and resize where the size is not img_height x img_width (unless no_resize), one net call in eval mode, one
    colorize call per output kind.  No host synchronisation."""
    import torch
    from . import _lib
    from .evaluate import colorize
    from .input_pipeline import scale_frames, to_device
    device = _lib.device()
    shapes = list(dict.fromkeys(tuple(f.shape) for f in frames))
    out = [None] * len(frames)
    disp_net.eval()
    with torch.no_grad():
        for shape in shapes:
            idx = [i for i, f in enumerate(frames) if tuple(f.shape) == shape]
            assert len(shape) == 3 and shape[2] == 3, shape
            group = [frames[i] for i in idx]
            src = torch.stack(group) if torch.is_tensor(group[0]) else torch.from_numpy(np.stack(group))
            src = to_device(src[:, None], device).contiguous()
            h, w = shape[:2] if no_resize else (img_height, img_width)
            x = scale_frames(src, h, w, 'inference')[0][0]
            disp = disp_net(x)[:, 0]
            res = {'disp_map': disp}
            if output_disp:
                res['disp'] = colorize(disp, 'bone')
            if output_depth:
                res['depth'] = colorize(disp, 'rainbow', max_value=10, invert=True)
            for j, i in enumerate(idx):
                out[i] = {k: v[j] for k, v in res.items()}
    return out


# ---- command line ------------------------------------------------------------------------------------------------------
def main(argv=None, device=None, workers=WORKERS):
    """run_inference.py main(): returns the list of photos and the files written (None when no output is asked for).
    Every worker process is joined before it returns or raises."""
    args = build_parser().parse_args(sys.argv[1:] if argv is None else argv)
    if not (args.output_disp or args.output_depth):
        print('You must at least output one value !')
        return None
    from . import _lib
    disp_net = load_disp_net(args.pretrained, args.dispnet, device or _lib.device())
    os.makedirs(args.output_dir, exist_ok=True)
    files = test_files(args.dataset_dir, args.dataset_list, args.img_exts)
    print('{} files to test'.format(len(files)))
    names = [output_names(f, args.output_dir) for f in files]
    last = {}                                     # output file -> the last photo that writes it
    for i, (dname, zname) in enumerate(names):
        if args.output_disp:
            last[dname] = i
        if args.output_depth:
            last[zname] = i
    chunks = [range(i, min(i + CHUNK, len(files))) for i in range(0, len(files), CHUNK)]
    written, writes = [], []
    with worker_pool(workers) as pool:
        for c, frames in zip(chunks, chunks_ahead(pool, decode, [[files[i] for i in c] for c in chunks])):
            res = infer(disp_net, frames, args.img_height, args.img_width, args.no_resize, args.output_disp,
                        args.output_depth)
            host = {kind: host_arrays([r[kind] for r in res]) for kind in ('disp', 'depth') if kind in res[0]}
            jobs = []
            for j, i in enumerate(c):
                for kind, name in zip(('disp', 'depth'), names[i]):
                    if kind in host and last.get(name) == i:
                        jobs.append((name, host[kind][j]))
                        written.append(name)
            writes.append(pool.starmap_async(encode, jobs))
        for wr in writes:
            wr.get()
    return dict(files=files, written=written)


if __name__ == '__main__':
    main()
