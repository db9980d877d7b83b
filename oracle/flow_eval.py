"""test_flow.py / test_back2future.py's KITTI-2015 evaluation restated on numpy and torch's CPU ops: ValidationFlow's
files and samples (datasets/validation_flow.py:94-141, transform None), test_flow.py's sample body (:127-140) around given
net outputs, test_back2future.py's compute_all_epes(gt, fwd, fwd, 1 - obj) and AverageMeter's averages.  Sample by
sample at batch 1, as the scripts loop; tests/golden/flow_eval_small.npz holds what the reference's own code returns for
the same inputs."""
import os
import numpy as np
import torch
from PIL import Image
from oracle import metrics as OM


def sample_paths(root, index, phase='training', occ='flow_occ', sequence_length=5):
    """ValidationFlow.__getitem__'s paths -> (target, refs, flow_gt, calib, obj_map)."""
    name = str(index).zfill(6)
    seq_ids = [x + 10 for x in range(-int(sequence_length / 2), int(sequence_length / 2) + 1) if x != 0]
    img = lambda k: os.path.join(root, 'data_scene_flow_multiview', phase, 'image_2', name + '_' + str(k).zfill(2) + '.png')  # noqa: E731
    return (img(10), [img(k) for k in seq_ids], os.path.join(root, 'data_scene_flow', phase, occ, name + '_10.png'),
            os.path.join(root, 'data_scene_flow_calib', phase, 'calib_cam_to_cam', name + '.txt'),
            os.path.join(root, 'data_scene_flow', phase, 'obj_map', name + '_10.png'))


def read_png16(path):
    """A 16-bit RGB PNG as uint16 [H,W,3], decoded with Pillow's PNG reader through numpy (big-endian rows)."""
    import zlib
    data = open(path, 'rb').read()
    pos, idat, hdr = 8, b'', None
    while pos < len(data):
        n = int.from_bytes(data[pos:pos + 4], 'big')
        kind, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        if kind == b'IHDR':
            hdr = (int.from_bytes(body[:4], 'big'), int.from_bytes(body[4:8], 'big'), body[8], body[9])
        elif kind == b'IDAT':
            idat += body
        pos += 12 + n
    W, H, depth, color = hdr
    assert depth == 16 and color == 2, hdr
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(H, 1 + W * 6)
    bpp, out, prev = 6, np.zeros((H, W * 6), np.int64), np.zeros(W * 6, np.int64)
    for y in range(H):
        f, line = raw[y, 0], raw[y, 1:].astype(np.int64)
        cur = np.zeros(W * 6, np.int64)
        for x in range(W * 6):
            a = cur[x - bpp] if x >= bpp else 0
            b, c = prev[x], (prev[x - bpp] if x >= bpp else 0)
            p = [0, a, b, (a + b) // 2, None][f] if f != 4 else \
                (a if abs(b - c) <= abs(a - c) and abs(b - c) <= abs(a + b - 2 * c) else
                 b if abs(a - c) <= abs(a + b - 2 * c) else c)
            cur[x] = (line[x] + p) & 0xff
        out[y], prev = cur, cur
    return (out.reshape(H, W, 3, 2)[..., 0] * 256 + out.reshape(H, W, 3, 2)[..., 1]).astype(np.uint16)


def load_sample(root, index, phase='training', occ='flow_occ'):
    """ValidationFlow(transform=None)[index] -> (tgt float32 [H,W,3], refs, K float32 [3,3], Kinv, gt float32 [3,Hg,Wg],
    obj (float32, or float64 ones where obj_map is missing))."""
    tgt_p, ref_ps, gt_p, calib_p, obj_p = sample_paths(root, index, phase, occ)
    tgt = np.asarray(Image.open(tgt_p)).astype(np.float32)
    refs = [np.asarray(Image.open(p)).astype(np.float32) for p in ref_ps]
    obj = np.asarray(Image.open(obj_p)).astype(np.float32) if os.path.isfile(obj_p) else np.ones(tgt.shape[:2])
    I = read_png16(gt_p)
    gt = np.dstack(((I[:, :, 0].astype('float64') - 2 ** 15) / 64.0, (I[:, :, 1].astype('float64') - 2 ** 15) / 64.0,
                    I[:, :, 2]))
    gt = torch.FloatTensor(gt.transpose(2, 0, 1)).numpy()
    data = {}
    for line in open(calib_p).readlines():
        key, value = line.split(':', 1)
        try:
            data[key] = np.array([float(x) for x in value.split()])
        except ValueError:
            pass
    K = np.reshape(data['P_rect_02'], (3, 4))[:, :3].astype('float32')
    return tgt, refs, K, np.linalg.inv(K), gt, obj


def sample_errors(emask, flow_cam, flow_fwd, flow_gt, obj_map, THRESH=0.01, epe_thresh=0.5):
    """test_flow.py:127-140 on one sample's net outputs (batch 1): emask [1,C,h,w], flow_cam / flow_fwd [1,2,h,w], flow_gt
    [1,3,Hg,Wg], obj_map [1,Hg,Wg] -> (the 8 numbers, combined [1,1,h,w])."""
    with torch.no_grad():
        rigid = 1 - (1 - emask[:, 1]) * (1 - emask[:, 2]).unsqueeze(1) > 0.5
        soft = (flow_cam - flow_fwd).abs()
        census = (soft[:, 0] < THRESH).type_as(flow_fwd) * (soft[:, 1] < THRESH).type_as(flow_fwd)
        combined = 1 - (1 - rigid.type_as(emask)) * (1 - census.type_as(emask))
        obj = obj_map.unsqueeze(1).type_as(flow_fwd)
        errs = OM.compute_all_epes(flow_gt, flow_cam, flow_fwd, combined, epe_thresh) + \
            OM.compute_all_epes(flow_gt, flow_cam, flow_fwd, 1 - obj, epe_thresh)
    return errs, combined


def back2future_errors(flow_fwd, flow_gt, obj_map, epe_thresh=0.5):
    """test_back2future.py's compute_all_epes(gt, fwd, fwd, 1 - obj) of one sample -> 4 numbers."""
    with torch.no_grad():
        return OM.compute_all_epes(flow_gt, flow_fwd, flow_fwd, 1 - obj_map.unsqueeze(1).type_as(flow_fwd), epe_thresh)


def summary(per_sample):
    """AverageMeter(i=n).update(row) for every row in order -> avg (python floats)."""
    sums, count = [0] * len(per_sample[0]), 0
    for row in per_sample:
        count += 1
        for k, v in enumerate(row):
            sums[k] += v * 1
    return [s / count for s in sums]
