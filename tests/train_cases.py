"""The training driver's data tree (rebuilt from tests/golden/train_data_small.npz, which holds its bytes) and helpers the
CPU and GPU driver tests share."""
import os
import numpy as np
from tests.util import golden

SEQ_SCENES = {'scene_a': 7, 'scene_b': 6, 'scene_c': 3}        # scene_c is shorter than a 5-frame sequence
STACKED = {'scene_s': 4}
H, W = 64, 128


def tree_files(seed=5):
    """{relative path: bytes} of the tree: seq/ (sequential format: jpgs, cam.txt, .npy depths, train.txt, val.txt) and
    stacked/ (5 frames side by side per jpg, a *_cam.txt per frame, train.txt of `scene frame` lines)."""
    import io
    from PIL import Image
    rng = np.random.RandomState(seed)
    files = {}

    def jpg(a):
        b = io.BytesIO()
        Image.fromarray(a).save(b, format='JPEG', quality=90)
        return b.getvalue()

    def img(h, w):
        y, x = np.mgrid[0:h, 0:w]
        base = np.stack([x * 255 // w, y * 255 // h, (x + y) % 256], -1)
        return np.clip(base + rng.randint(-6, 7, (h, w, 3)), 0, 255).astype(np.uint8)

    def depth():
        y, x = np.mgrid[0:H, 0:W]
        d = (5 + (x + 2 * y) % 70 + rng.randint(0, 3, (H, W))).astype(np.float32)
        d[rng.rand(H, W) < 0.3] = 0                              # no ground truth at these pixels
        return d

    def npy(a):
        b = io.BytesIO()
        np.save(b, a)
        return b.getvalue()

    def cam(f):
        return ('%.6f,0.000000,%.6f\n0.000000,%.6f,%.6f\n0.000000,0.000000,1.000000\n' % (f, W / 2 + 0.5, f, H / 2 - 0.25)).encode()

    for k, (scene, n) in enumerate(SEQ_SCENES.items()):
        files['seq/%s/cam.txt' % scene] = cam(100.0 + 10 * k)
        for i in range(n):
            files['seq/%s/%07d.jpg' % (scene, i)] = jpg(img(H, W))
            files['seq/%s/%07d.npy' % (scene, i)] = npy(depth())
    files['seq/train.txt'] = b'scene_b\nscene_a\nscene_c\n'
    files['seq/val.txt'] = b'scene_c\nscene_a\n'
    lines = []
    for scene, n in STACKED.items():
        for i in range(n):
            files['stacked/%s/%07d.jpg' % (scene, i)] = jpg(img(H, 5 * W))
            files['stacked/%s/%07d_cam.txt' % (scene, i)] = cam(90.0 + i)
            lines.append('%s %07d\n' % (scene, i))
    files['stacked/train.txt'] = ''.join(lines[::-1]).encode()
    return files


def write_tree(root, files=None):
    """Write the tree under `root` from the fixture's bytes (or `files`)."""
    if files is None:
        g = golden('train_data_small')
        files = {str(n): g['tree_%d' % i].tobytes() for i, n in enumerate(g['tree_names'])}
    for rel, b in files.items():
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, 'wb') as f:
            f.write(b)
    return root


def rel(root, p):
    return os.path.relpath(p, root)


def write_synth_dump(root, scenes=2, frames=14, H=64, W=128, seed=0, quality=95):
    """A sequential dump of seeded cc_b200.synth frames: root/scene_<k>/<i>.jpg (JPEG), cam.txt (synth.intrinsics), a
    positive .npy depth beside every jpg, train.txt and val.txt listing every scene."""
    import torch
    from PIL import Image
    from cc_b200 import synth
    os.makedirs(root, exist_ok=True)
    names = []
    K = synth.intrinsics(1, H, W)[0][0].numpy()
    for k in range(scenes):
        name = 'scene_%d' % k
        d = os.path.join(root, name)
        os.makedirs(d, exist_ok=True)
        names.append(name)
        g = torch.Generator().manual_seed(seed * 1000 + k)
        # one wide image; the camera pans 3 pixels per frame over it
        wide = synth._smooth_field(g, 1, 3, H, W + 3 * frames).clamp(-0.95, 0.95)
        wide = ((wide[0].permute(1, 2, 0) + 1) * 127.5).round().clamp(0, 255).to(torch.uint8).numpy()
        for i in range(frames):
            Image.fromarray(np.ascontiguousarray(wide[:, 3 * i:3 * i + W])).save(
                os.path.join(d, '%07d.jpg' % i), quality=quality)
            np.save(os.path.join(d, '%07d.npy' % i), (1 + 60 * np.random.RandomState(seed + i).rand(H, W)).astype(np.float32))
        np.savetxt(os.path.join(d, 'cam.txt'), K, delimiter=',')
    for f in ('train.txt', 'val.txt'):
        with open(os.path.join(root, f), 'w') as fh:
            fh.write(''.join(n + '\n' for n in names))
    return root
