"""Reference arm: the UNMODIFIED reference modules (anuragranj/cc @ 2b4e362) driven through the body of the
reference's own train() loop (train.py:454-509,566-568), on the CPU (the `--impl reference` arm of bench.py and
its `cpu_baseline`) or on a CUDA device (`reference_gpu`, the "reference PyTorch on one GPU" comparator of
BASELINE.md section 4).  NOTHING of cc_b200 or the oracle restatement is on this path.

`oracle/_ref/` holds a verbatim copy of the reference's hot-path files (inverse_warp.py, ssim.py,
loss_functions.py, models/*.py); `__graft_entry__.build()` makes that copy from the reference checkout: the one named by
the CC_REFERENCE environment variable, else a directory `reference` next to this repository, when it exists.  The directory is git-ignored (never committed); without it
the reference arm reports itself unavailable.

Two stubs, both required for the reference to import at all (SURVEY.md F11):
  * `spatial_correlation_sampler`: the third-party CUDA extension is not installed and its source is not in the
    reference tree -> the pure-torch restatement below (81 shifted channel means); results carry the label
    "stub correlation".
  * on a CPU run only: `Tensor.cuda()` / `Module.cuda()` become no-ops (back2future.py:58-59,302,311 call them
    unconditionally).
"""
import os
import sys
import types
import warnings
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, '_ref')
FILES = ['inverse_warp.py', 'ssim.py', 'loss_functions.py', 'models']

# README.md:59-65 command line + train.py:120-130 defaults
HP = dict(w1=1.0, w2=0.1, w3=0.1, w4=0.5, w5=0.3, wssim=0.997, qch=0.5, lambda_oob=0.0, THRESH=0.01, wbce=0.5,
          wrig=1.0, lr=1e-4, momentum=0.9, beta=0.999)
_ORIG_CUDA = None
NETS_OF = {'cfg1': ('disp', 'pose'), 'cfg2': ('flow',), 'cfg3': ('disp', 'pose', 'mask', 'flow')}


def available():
    return all(os.path.exists(os.path.join(REF_DIR, f)) for f in FILES)


def reference_checkout():
    """Where the reference lives: $CC_REFERENCE, else a checkout named `reference` next to this repository."""
    return os.environ.get('CC_REFERENCE') or os.path.join(os.path.dirname(os.path.dirname(HERE)), 'reference')


def install(src=None):
    """Copy the reference's hot-path files from `src` (default: reference_checkout()) into oracle/_ref.  Where there is
    no checkout (a GPU host that only received this repository) nothing is copied and the reference arm reports itself
    unavailable."""
    import shutil
    src = src or reference_checkout()
    if not os.path.isdir(src):
        return False
    os.makedirs(REF_DIR, exist_ok=True)
    for f in FILES:
        s, d = os.path.join(src, f), os.path.join(REF_DIR, f)
        if os.path.isdir(s):
            os.makedirs(d, exist_ok=True)
            for g in os.listdir(s):
                if g.endswith('.py'):
                    shutil.copyfile(os.path.join(s, g), os.path.join(d, g))
        else:
            shutil.copyfile(s, d)
    return True


def _corr_stub(input1, input2, kernel_size=1, patch_size=9, stride=1, padding=0, dilation=1, dilation_patch=1):
    """out[b, i, j, y, x] = sum_c in1[b,c,y,x] * in2[b,c,y+i-r,x+j-r]  (zero outside), r = patch_size // 2;
    first patch index = vertical displacement (the published behaviour of spatial-correlation-sampler)."""
    B, C, H, W = input1.shape
    r = patch_size // 2
    p2 = F.pad(input2, (r, r, r, r))
    out = [(input1 * p2[:, :, i:i + H, j:j + W]).sum(1) for i in range(patch_size) for j in range(patch_size)]
    return torch.stack(out, 1).view(B, patch_size, patch_size, H, W)


class Ref:
    """The imported reference modules + the nets/optimizer of one configuration on `device`."""

    def __init__(self, cfg, device, seed=0):
        assert available(), 'oracle/_ref is missing: run `python __graft_entry__.py` with a reference checkout beside this repository (or CC_REFERENCE=<checkout>)'
        warnings.filterwarnings('ignore')
        self.cfg, self.device = cfg, torch.device(device)
        stub = types.ModuleType('spatial_correlation_sampler')
        stub.spatial_correlation_sample = _corr_stub
        sys.modules['spatial_correlation_sampler'] = stub
        global _ORIG_CUDA
        if _ORIG_CUDA is None:
            _ORIG_CUDA = (torch.Tensor.cuda, torch.nn.Module.cuda)
        if self.device.type == 'cpu':
            torch.Tensor.cuda = lambda self_, *a, **k: self_
            torch.nn.Module.cuda = lambda self_, *a, **k: self_
        else:
            torch.Tensor.cuda, torch.nn.Module.cuda = _ORIG_CUDA
        if REF_DIR not in sys.path:
            sys.path.insert(0, REF_DIR)
        import inverse_warp as RW
        import loss_functions as RL
        import models as RM
        assert os.path.dirname(os.path.abspath(RW.__file__)) == REF_DIR, 'a foreign inverse_warp module shadows the reference'
        self.RW, self.RL, self.RM = RW, RL, RM
        torch.manual_seed(seed)
        with torch.cuda.device(self.device) if self.device.type == 'cuda' else _null():
            mk = {'disp': lambda: RM.DispResNet6(), 'pose': lambda: RM.PoseNetB6(nb_ref_imgs=4),
                  'mask': lambda: RM.MaskNet6(nb_ref_imgs=4, output_exp=True), 'flow': lambda: RM.Back2Future(nlevels=6)}
            self.nets = {}
            for n in NETS_OF[cfg]:
                net = mk[n]()
                net.init_weights()                                        # train.py:257-284 (no pretrained weights)
                self.nets[n] = net.to(self.device).train()
        params = [p for n in NETS_OF[cfg] for p in self.nets[n].parameters()]
        self.opt = torch.optim.Adam(params, HP['lr'], betas=(HP['momentum'], HP['beta']), weight_decay=0)   # train.py:307-310

    def loss(self, tgt_img, ref_imgs, intrinsics, intrinsics_inv):
        RW, RL, hp, cfg = self.RW, self.RL, HP, self.cfg
        w1, w2, w3, w4, w5 = hp['w1'], hp['w2'], hp['w3'], hp['w4'], hp['w5']
        if cfg == 'cfg2':
            flow_fwd, flow_bwd, _ = self.nets['flow'](tgt_img, ref_imgs[1:3])
            loss_4 = RL.photometric_flow_loss(tgt_img, ref_imgs[1:3], [flow_bwd, flow_fwd], [None] * 6,
                                              lambda_oob=hp['lambda_oob'], qch=hp['qch'], wssim=hp['wssim'])
            loss_3 = RL.edge_aware_smoothness_loss(tgt_img, flow_fwd) + RL.edge_aware_smoothness_loss(tgt_img, flow_bwd)
            return w4 * loss_4 + w3 * loss_3
        disparities = self.nets['disp'](tgt_img)                                           # train.py:454
        depth = [1 / disp for disp in disparities]                                         # :458
        pose = self.nets['pose'](tgt_img, ref_imgs)                                        # :459
        if cfg == 'cfg1':
            loss_1 = RL.photometric_reconstruction_loss(tgt_img, ref_imgs, intrinsics, intrinsics_inv, depth, [None] * 6, pose,
                                                        lambda_oob=hp['lambda_oob'], qch=hp['qch'], wssim=hp['wssim'])
            return w1 * loss_1 + w3 * RL.edge_aware_smoothness_loss(tgt_img, depth)
        explainability_mask = self.nets['mask'](tgt_img, ref_imgs)                         # :460
        flow_fwd, flow_bwd, _ = self.nets['flow'](tgt_img, ref_imgs[1:3])                  # :463
        flows_cam_fwd = [RW.pose2flow(d.squeeze(1), pose[:, 2], intrinsics, intrinsics_inv) for d in depth]   # :470
        flows_cam_bwd = [RW.pose2flow(d.squeeze(1), pose[:, 1], intrinsics, intrinsics_inv) for d in depth]   # :471
        exp_masks_target = RL.consensus_exp_masks(flows_cam_fwd, flows_cam_bwd, flow_fwd, flow_bwd, tgt_img, ref_imgs[2],
                                                  ref_imgs[1], wssim=hp['wssim'], wrig=hp['wrig'], ws=w3)     # :473
        rigidity_mask_fwd = [(a - b).abs() for a, b in zip(flows_cam_fwd, flow_fwd)]       # :475
        rigidity_mask_bwd = [(a - b).abs() for a, b in zip(flows_cam_bwd, flow_bwd)]       # :476
        flow_exp_mask = [1 - m[:, 1:3] for m in explainability_mask]                       # :488
        loss_1 = RL.photometric_reconstruction_loss(tgt_img, ref_imgs, intrinsics, intrinsics_inv, depth, explainability_mask,
                                                    pose, lambda_oob=hp['lambda_oob'], qch=hp['qch'], wssim=hp['wssim'])  # :490
        loss_2 = RL.explainability_loss(explainability_mask)                               # :493
        loss_3 = RL.edge_aware_smoothness_loss(tgt_img, depth) + RL.edge_aware_smoothness_loss(tgt_img, flow_fwd)          # :500
        loss_3 = loss_3 + RL.edge_aware_smoothness_loss(tgt_img, flow_bwd) + RL.edge_aware_smoothness_loss(tgt_img, explainability_mask)
        loss_4 = RL.photometric_flow_loss(tgt_img, ref_imgs[1:3], [flow_bwd, flow_fwd], flow_exp_mask,
                                          lambda_oob=hp['lambda_oob'], qch=hp['qch'], wssim=hp['wssim'])      # :503
        loss_5 = RL.consensus_depth_flow_mask(explainability_mask, rigidity_mask_bwd, rigidity_mask_fwd, exp_masks_target,
                                              exp_masks_target, THRESH=hp['THRESH'], wbce=hp['wbce'])         # :506
        return w1 * loss_1 + w2 * loss_2 + w3 * loss_3 + w4 * loss_4 + w5 * loss_5         # :509

    def step(self, tgt_img, ref_imgs, intrinsics, intrinsics_inv):
        loss = self.loss(tgt_img, ref_imgs, intrinsics, intrinsics_inv)
        self.opt.zero_grad()                                                               # train.py:566-568
        loss.backward()
        self.opt.step()
        return loss.detach()


class _null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False
