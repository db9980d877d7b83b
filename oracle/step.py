"""Oracle: one CC training step (reference train.py:445-568) on CPU.  TEST INFRASTRUCTURE.

Used as the parity checker for the step-level tests and as the CPU baseline
(`bench.py` cpu_baseline / --impl reference, kind "port")."""
import torch
from . import nets
from .geometry import pose2flow
from . import losses as L

# README.md:59-65 command line + train.py:120-130 defaults
HP = dict(w1=1.0, w2=0.1, w3=0.1, w4=0.5, w5=0.3, wssim=0.997, qch=0.5, lambda_oob=0.0,
          THRESH=0.01, wbce=0.5, wrig=1.0, lr=1e-4, beta1=0.9, beta2=0.999, smoothness='edgeaware')


def _smooth(hp, tgt, preds):
    if hp['smoothness'] == 'edgeaware':
        return L.edge_aware_smoothness_loss(tgt, preds)
    return L.smooth_loss(preds)


def loss_cfg1(P, tgt, refs, K, Kinv, hp=HP):
    """DispResNet6+PoseNetB6 depth/pose step (SURVEY 8d cfg1): explainability_mask=[None]*6."""
    disp = nets.disp_forward(P['disp'], tgt, training=True)
    depth = [1 / d for d in disp]
    pose = nets.pose_forward(P['pose'], tgt, refs)
    l1 = L.photometric_reconstruction_loss(tgt, refs, K, Kinv, depth, [None] * len(depth), pose,
                                           lambda_oob=hp['lambda_oob'], qch=hp['qch'], wssim=hp['wssim'])
    l3 = _smooth(hp, tgt, depth)
    loss = hp['w1'] * l1 + hp['w3'] * l3
    return loss, dict(loss_1=l1, loss_3=l3, disp=disp, pose=pose)


def loss_cfg2(P, tgt, refs, K, Kinv, hp=HP, flownet='Back2Future'):
    """Flow net (Back2Future by default) + flow photometric(+SSIM) + smoothness (cfg2)."""
    ff, fb = nets.flow_pair(P['flow'], tgt, refs, flownet)
    l4 = L.photometric_flow_loss(tgt, refs[1:3], [fb, ff], [None] * len(ff),
                                 lambda_oob=hp['lambda_oob'], qch=hp['qch'], wssim=hp['wssim'])
    l3 = _smooth(hp, tgt, ff) + _smooth(hp, tgt, fb)
    loss = hp['w4'] * l4 + hp['w3'] * l3
    return loss, dict(loss_4=l4, loss_3=l3, flow_fwd=ff, flow_bwd=fb)


def loss_cfg3(P, tgt, refs, K, Kinv, hp=HP, flownet='Back2Future'):
    """Full joint step body.  Reference train.py:454-509."""
    disp = nets.disp_forward(P['disp'], tgt, training=True)
    depth = [1 / d for d in disp]
    pose = nets.pose_forward(P['pose'], tgt, refs)
    emask = nets.mask_forward(P['mask'], tgt, refs, training=True)
    ff, fb = nets.flow_pair(P['flow'], tgt, refs, flownet)
    cam_f = [pose2flow(d.squeeze(1), pose[:, 2], K, Kinv) for d in depth]
    cam_b = [pose2flow(d.squeeze(1), pose[:, 1], K, Kinv) for d in depth]
    tgt_masks = L.consensus_exp_masks(cam_f, cam_b, ff, fb, tgt, refs[2], refs[1],
                                      wssim=hp['wssim'], wrig=hp['wrig'], ws=hp['w3'])
    rig_f = [(a - b).abs() for a, b in zip(cam_f, ff)]
    rig_b = [(a - b).abs() for a, b in zip(cam_b, fb)]
    flow_emask = [1 - m[:, 1:3] for m in emask]
    l1 = L.photometric_reconstruction_loss(tgt, refs, K, Kinv, depth, emask, pose,
                                           lambda_oob=hp['lambda_oob'], qch=hp['qch'], wssim=hp['wssim'])
    l2 = L.explainability_loss(emask) if hp['w2'] > 0 else 0
    l3 = _smooth(hp, tgt, depth) + _smooth(hp, tgt, ff) + _smooth(hp, tgt, fb) + _smooth(hp, tgt, emask)
    l4 = L.photometric_flow_loss(tgt, refs[1:3], [fb, ff], flow_emask,
                                 lambda_oob=hp['lambda_oob'], qch=hp['qch'], wssim=hp['wssim'])
    l5 = L.consensus_depth_flow_mask(emask, rig_b, rig_f, tgt_masks, tgt_masks,
                                     THRESH=hp['THRESH'], wbce=hp['wbce'])
    loss = hp['w1'] * l1 + hp['w2'] * l2 + hp['w3'] * l3 + hp['w4'] * l4 + hp['w5'] * l5
    return loss, dict(loss_1=l1, loss_2=l2, loss_3=l3, loss_4=l4, loss_5=l5,
                      disp=disp, pose=pose, emask=emask, flow_fwd=ff, flow_bwd=fb)


LOSS_FNS = {'cfg1': loss_cfg1, 'cfg2': loss_cfg2, 'cfg3': loss_cfg3}
NETS_OF = {'cfg1': ('disp', 'pose'), 'cfg2': ('flow',), 'cfg3': ('disp', 'pose', 'mask', 'flow')}


def make_params(cfg, requires_grad=True):
    mk = {'disp': nets.disp_params, 'pose': nets.pose_params, 'mask': nets.mask_params,
          'flow': nets.flow_params}
    return {n: nets.clone_params(mk[n](), requires_grad=requires_grad) for n in NETS_OF[cfg]}


class Adam:
    """torch.optim.Adam semantics (reference train.py:307-310: betas=(momentum, beta), wd 0)."""

    def __init__(self, params, lr, beta1=0.9, beta2=0.999, eps=1e-8):
        self.params = [p for p in params if p.requires_grad]
        self.lr, self.b1, self.b2, self.eps = lr, beta1, beta2, eps
        self.m = [torch.zeros_like(p) for p in self.params]
        self.v = [torch.zeros_like(p) for p in self.params]
        self.t = 0

    def zero_grad(self):
        for p in self.params:
            p.grad = None

    @torch.no_grad()
    def step(self):
        self.t += 1
        bc1 = 1 - self.b1 ** self.t
        bc2 = 1 - self.b2 ** self.t
        for p, m, v in zip(self.params, self.m, self.v):
            if p.grad is None:
                continue
            g = p.grad
            m.mul_(self.b1).add_(g, alpha=1 - self.b1)
            v.mul_(self.b2).addcmul_(g, g, value=1 - self.b2)
            denom = (v.sqrt() / (bc2 ** 0.5)).add_(self.eps)
            p.addcdiv_(m, denom, value=-self.lr / bc1)


def train_step(cfg, P, opt, tgt, refs, K, Kinv, hp=HP, flownet='Back2Future'):
    """zero_grad -> forward -> backward -> Adam (reference train.py:566-568).  flownet: the net P['flow'] holds
    (cfg2 / cfg3)."""
    opt.zero_grad()
    fn = LOSS_FNS[cfg]
    loss, aux = fn(P, tgt, refs, K, Kinv, hp) if cfg == 'cfg1' else fn(P, tgt, refs, K, Kinv, hp, flownet)
    loss.backward()
    opt.step()
    return loss.detach(), aux


def all_params(P):
    out = []
    for n in P:
        out += [t for k, t in P[n].items() if t.requires_grad]
    return out
