"""The reference's test_disp.py on this stack: `python -m cc_b200.test_disp --dispnet DispResNet6 --pretrained-dispnet CKPT
[--pretrained-posenet CKPT] --dataset-dir KITTI_raw --dataset-list kitti_eval/test_files_eigen.txt` evaluates a disparity
net's depth on the Eigen split (--gt-type KITTI, velodyne ground truth) or on Stillbox (--gt-type stillbox, .npy depth) and
prints the script's lines and result rows: abs_rel sq_rel rms log_rms a1 a2 a3 averaged over the test files, scaled by
the pose net's displacements (with --pretrained-posenet) and by the median ratio.

  files       --dataset-list's lines, or for each --img-exts in turn the files of --dataset-dir matching *.{ext}, relative
              to it.  evaluate.kitti_depth_framework / stillbox_depth_framework give each sample's frames, ground-truth
              source and displacements; the reference frames' count comes from the pose checkpoint
              (conv1.0.weight.size(1) / 3, evaluate.load_pose_net), none without one.
  load        host worker processes decode the frames (run_inference.decode: a file that is not H x W x 3 uint8 is refused,
              and the error names it) and read the velodyne sweeps, calibrations or .npy depths, a chunk ahead of the
              device.
  device      evaluate_chunk(): the samples of a chunk grouped by frame size and ground-truth size; per group the KITTI
              ground truth in one velodyne_depth call, the frames through input_pipeline.scale_frames (imresize's
              contrast stretch and resize to a float32 image unless they are --img-height x --img-width or --no-resize,
              then (x/255 - 0.5)/0.5), and evaluate.depth_eval_batch: the disparity net, spatial_normalize with the flag,
              the pose net on the same frames, the spline zoom and both scalings' errors.  The errors stay on the device
              until the rows are printed (evaluate.depth_summary).  A sample without a positive displacement gets scale 0
              in row 0; its 'not good !' line is decided on the host from the displacements alone.
  output      --output-dir: predictions.npy, float64 [len(test_files), h, w] of 1/disparity (rows of missing files stay
              zero, at the end), and viz/{j:04d}img.png (the normalised input mapped back as tensor2array does),
              depth.png (the disparity through matplotlib's 'hot', scaled by its maximum) and gt.png (the ground truth
              filled by interp_gt_disp in the workers, zeros as 1000, then (1/x).clamp(0, 10) through 'hot').
A missing target file is skipped but still counts in the mean, as a column of zeros.  The output does not depend on the
worker count; every worker is joined when main() returns or raises.

Extension: --posenet also takes PoseNetB6 and PoseNet6 (Competitive Collaboration's own pose checkpoints).  The reference
builds the pose net with output_exp=False, which only PoseExpNet accepts: any other raises TypeError.

Documented deviations:
  --output-dir  crashes in the reference at its first sample: utils.COLORMAPS has no 'hot' (KeyError), and it would then
                hand Pillow [3,H,W] arrays.  Here the intended H x W x 3 images and predictions.npy are written
                (predictions.npy only once a sample exists: the reference has no array to save before one).
  --min-depth   has no type in the reference, so a value given makes a string and crashes; here it is a float.
  file list     the reference lists --dataset-dir's files as file.relpathto(dataset_dir), the path from the file to the
                folder ('..'); here they are relative to the folder, as meant.  Neither framework parses a bare file name,
                so without --dataset-list the run stops with an error that names the file.
  refusals      --gt-type npy and png are refused by the parser (the reference has no framework for them and raises
                NameError); --no-resize with --output-dir on frames of different sizes is refused (the reference raises
                ValueError filling its predictions array); a reference frame of another size than its target is refused.
  batching      a size group runs through the nets in one batch; the reference runs one sample at a time.
The README's --pretrained-posent is not a flag of either program: it is --pretrained-posenet."""
import argparse
import os
import sys
import numpy as np
from . import run_inference as RI

CHUNK = 32                      # samples loaded ahead of the device: 32 KITTI samples of 5 frames are 210 MB of uint8
WORKERS = 4
ERROR_NAMES = ['abs_rel', 'sq_rel', 'rms', 'log_rms', 'a1', 'a2', 'a3']
NO_POSENET = ('no PoseNet specified, scale_factor will be determined by median ratio, which is kiiinda cheating'
              '            (but consistent with original paper)')


def build_parser():
    from .evaluate import POSE_NETS
    p = argparse.ArgumentParser(description='Script for DispNet testing with corresponding groundTruth',
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    a = p.add_argument
    a('--dispnet', dest='dispnet', type=str, default='DispResNet6', choices=RI.DISPNETS, help='dispnet architecture')
    a('--posenet', dest='posenet', type=str, default='PoseExpNet', choices=POSE_NETS, help='posenet architecture')
    a('--pretrained-dispnet', required=True, type=str, help='pretrained DispNet path')
    a('--pretrained-posenet', default=None, type=str, help='pretrained PoseNet path (for scale factor)')
    a('--img-height', default=256, type=int, help='Image height')
    a('--img-width', default=832, type=int, help='Image width')
    a('--no-resize', action='store_true', help='no resizing is done')
    a('--spatial-normalize', action='store_true', help='spatial normalization')
    a('--min-depth', default=1e-3, type=float)
    a('--max-depth', default=80, type=float)
    a('--dataset-dir', default='.', type=str, help='Dataset directory')
    a('--dataset-list', default=None, type=str, help='Dataset list file')
    a('--output-dir', default=None, type=str, help='Output directory for saving predictions in a big 3D numpy file')
    a('--gt-type', default='KITTI', type=str, help='GroundTruth data type', choices=['npy', 'png', 'KITTI', 'stillbox'])
    a('--img-exts', default=['png', 'jpg', 'bmp'], nargs='*', type=str, help='images extensions to glob')
    return p


def listed_files(dataset_dir, dataset_list=None, img_exts=('png', 'jpg', 'bmp')):
    """The test files: the list's lines as they are, or for each extension in turn the files of dataset_dir matching
    '*.ext' in os.listdir order, relative to dataset_dir."""
    if dataset_list is not None:
        with open(dataset_list, 'r') as f:
            return list(f.read().splitlines())
    return [os.path.relpath(f, dataset_dir) for f in RI.test_files(dataset_dir, None, img_exts)]


# ---- host workers ------------------------------------------------------------------------------------------------------
def load_sample(sample):
    """One sample in a worker: 'frames' uint8 [1 + R, H, W, 3] (the target, then its references, all of one size) and its
    ground-truth source: KITTI's velodyne 'points' and projection 'P', or Stillbox's depth 'gt'."""
    from . import evaluate as CE
    frames = [RI.decode(sample['path'])] + [RI.decode(r) for r in sample['refs']]
    for f, r in zip(frames[1:], sample['refs']):
        if f.shape != frames[0].shape:
            raise ValueError('%s: a reference frame of %s is %dx%d, the target %dx%d' % (
                r, sample['path'], f.shape[1], f.shape[0], frames[0].shape[1], frames[0].shape[0]))
    out = dict(frames=np.stack(frames))
    if 'velo' in sample:
        out['points'] = CE.load_velodyne_points(sample['velo'])
        out['P'] = CE.kitti_velo_to_image(sample['calib_dir'], sample['cam'])
    else:
        out['gt'] = np.load(sample['depth'])
    return out


def interp_gt_disp(depth):
    """test_disp.py's interp_gt_disp of a copy of `depth`: scipy's linear griddata through the pixels that are neither 0
    nor NaN/inf, 0 outside their convex hull."""
    from scipy.interpolate import griddata
    d = np.asarray(depth, np.float64)
    yy, xx = np.mgrid[0:d.shape[0], 0:d.shape[1]]
    ok = np.isfinite(d) & (d != 0)
    return griddata((xx[ok], yy[ok]), d[ok], (xx, yy), method='linear', fill_value=0)


# ---- device ------------------------------------------------------------------------------------------------------------
def evaluate_chunk(disp_net, pose_net, loaded, displacements, crop='eigen', img_height=256, img_width=832, no_resize=False,
                   spatial_normalize=False, min_depth=1e-3, max_depth=80.0, want_viz=False):
    """test_disp.py:75-141 for the loaded samples of a chunk (load_sample's dicts, numpy) with their displacements -> one
    dict per sample of device tensors: 'errors' fp64 [2,7] (row 0 zeros without a pose net) and, with want_viz, 'disp'
    the disparity [h,w] (after spatial_normalize), 'gt' the ground truth fp64 [H,W], 'img' and 'depth' uint8 [h,w,3].
    Samples of one frame size and ground-truth size form one group: one velodyne_depth call (KITTI), one scale_frames
    call, one depth_eval_batch.  No host synchronisation."""
    import torch
    from . import _lib
    from .evaluate import colorize, depth_eval_batch, velodyne_depth
    from .input_pipeline import scale_frames, to_device
    device = _lib.device()
    keys = [(s['frames'].shape, s['gt'].shape if 'gt' in s else s['frames'].shape[1:3]) for s in loaded]
    out = [None] * len(loaded)
    with torch.no_grad():
        for key in dict.fromkeys(keys):
            idx = [i for i, k in enumerate(keys) if k == key]
            (_, Hs, Ws, _), (Hg, Wg) = key
            group = [loaded[i] for i in idx]
            if 'gt' in group[0]:
                gt = to_device(np.stack([s['gt'] for s in group]).astype(np.float64), device)
            else:
                offsets = np.cumsum([0] + [len(s['points']) for s in group]).astype(np.int64)
                gt = velodyne_depth(to_device(np.concatenate([s['points'] for s in group]), device),
                                    to_device(offsets, device), to_device(np.stack([s['P'] for s in group]), device), Hg, Wg)
            h, w = (Hs, Ws) if no_resize else (img_height, img_width)
            outs = scale_frames(to_device(np.stack([s['frames'] for s in group]), device), h, w)[0]
            tgt, refs = outs[0], outs[1:]
            with_pose = pose_net is not None
            disp_t = to_device(np.array([displacements[i] for i in idx], np.float64).reshape(len(idx), -1), device)
            errors, disp = depth_eval_batch(disp_net, tgt, gt, min_depth, max_depth, crop, pose_net if with_pose else None,
                                            refs if with_pose else None, disp_t if with_pose else None, spatial_normalize,
                                            want_disp=True)
            res = {'errors': errors}
            if want_viz:
                res.update(disp=disp[:, 0], gt=gt, depth=colorize(disp, 'hot'),
                           img=(255 * (0.5 + tgt * 0.5)).to(torch.uint8).permute(0, 2, 3, 1))
            for j, i in enumerate(idx):
                out[i] = {k: v[j] for k, v in res.items()}
    return out


def gt_image(filled):
    """gt.png of interp_gt_disp's fp64 maps [B,H,W] (a device tensor): float32, zeros as 1000, (1/x).clamp(0, 10), then
    'hot' scaled by each image's maximum -> uint8 [B,H,W,3]."""
    from .evaluate import colorize
    g = filled.float()
    g[g == 0] = 1000
    return colorize((1 / g).clamp(0, 10), 'hot')


# ---- command line ------------------------------------------------------------------------------------------------------
def _frame_size(path):
    from PIL import Image
    with Image.open(path) as im:
        return im.size


def main(argv=None, device=None, workers=WORKERS):
    """test_disp.py main() -> dict(test_files, samples, errors): errors float32 [len(test_files), 2, 7] as the script's
    `errors` array holds them (per sample, zeros after the last sample).  Every worker is joined before it returns or
    raises."""
    parser = build_parser()
    args = parser.parse_args(sys.argv[1:] if argv is None else argv)
    if args.gt_type not in ('KITTI', 'stillbox'):
        parser.error('--gt-type %s: there is no test framework for this ground truth (KITTI and stillbox have one)'
                     % args.gt_type)
    import torch
    from . import _lib
    from . import evaluate as CE
    device = device or _lib.device()
    disp_net = RI.load_disp_net(args.pretrained_dispnet, args.dispnet, device)
    pose_net, seq_length = None, 0
    if args.pretrained_posenet is None:
        print(NO_POSENET)
    else:
        pose_net, seq_length = CE.load_pose_net(args.pretrained_posenet, args.posenet, device)
    test_files = listed_files(args.dataset_dir, args.dataset_list, args.img_exts)
    framework, crop = ((CE.kitti_depth_framework, 'eigen') if args.gt_type == 'KITTI'
                       else (CE.stillbox_depth_framework, 'stillbox'))
    samples = framework(args.dataset_dir, test_files, seq_length)
    print('{} files to test'.format(len(test_files)))
    out_dir = args.output_dir
    if out_dir is not None:
        if args.no_resize:
            sizes = {}
            for s in samples:
                sizes.setdefault(_frame_size(s['path']), s['path'])
            if len(sizes) > 1:
                parser.error('--no-resize with --output-dir needs frames of one size: %s' % ', '.join(
                    '%s is %dx%d' % (p, w, h) for (w, h), p in sizes.items()))
        os.makedirs(os.path.join(out_dir, 'viz'), exist_ok=True)
    errors, preds, writes = [], [], []
    chunks = [samples[i:i + CHUNK] for i in range(0, len(samples), CHUNK)]
    with RI.worker_pool(workers) as pool:
        for k, (chunk, loaded) in enumerate(zip(chunks, RI.chunks_ahead(pool, load_sample, chunks))):
            for s in chunk:
                if seq_length > 0 and not any(d > 0 for d in s['displacements']):
                    print('not good ! ', s['path'], np.array(s['displacements']))
            res = evaluate_chunk(disp_net, pose_net, loaded, [s['displacements'] for s in chunk], crop, args.img_height,
                                 args.img_width, args.no_resize, args.spatial_normalize, args.min_depth, args.max_depth,
                                 want_viz=out_dir is not None)
            errors += [r['errors'] for r in res]
            if out_dir is None:
                continue
            preds += [1 / r['disp'] for r in res]
            filled = pool.map(interp_gt_disp, RI.host_arrays([r['gt'] for r in res]))
            gts = [gt_image(torch.from_numpy(f)[None].to(device))[0] for f in filled]
            imgs = RI.host_arrays([r[kind] for r in res for kind in ('img', 'depth')] + gts)
            jobs = []
            for j in range(len(res)):
                name = os.path.join(out_dir, 'viz', str(k * CHUNK + j).zfill(4))
                jobs += [(name + 'img.png', imgs[2 * j]), (name + 'depth.png', imgs[2 * j + 1]),
                         (name + 'gt.png', imgs[2 * len(res) + j])]
            writes.append(pool.starmap_async(RI.encode, jobs))
        for wr in writes:
            wr.get()
    per_sample = np.zeros((len(test_files), 2, 7), np.float32)
    if errors:
        per_sample[:len(errors)] = torch.stack(errors).cpu().numpy()
    mean_errors = CE.depth_summary(per_sample)
    if args.pretrained_posenet:
        print('Results with scale factor determined by PoseNet : ')
        print('{:>10}, {:>10}, {:>10}, {:>10}, {:>10}, {:>10}, {:>10}'.format(*ERROR_NAMES))
        print('{:10.4f}, {:10.4f}, {:10.4f}, {:10.4f}, {:10.4f}, {:10.4f}, {:10.4f}'.format(*mean_errors[0]))
    print('Results with scale factor determined by GT/prediction ratio (like the original paper) : ')
    print('{:>10}, {:>10}, {:>10}, {:>10}, {:>10}, {:>10}, {:>10}'.format(*ERROR_NAMES))
    print('{:10.4f}, {:10.4f}, {:10.4f}, {:10.4f}, {:10.4f}, {:10.4f}, {:10.4f}'.format(*mean_errors[1]))
    if out_dir is not None and preds:
        predictions = np.zeros((len(test_files),) + tuple(preds[0].shape))
        predictions[:len(preds)] = torch.stack(preds).cpu().numpy()
        np.save(os.path.join(out_dir, 'predictions.npy'), predictions)
    return dict(test_files=test_files, samples=samples, errors=per_sample)


if __name__ == '__main__':
    main()
