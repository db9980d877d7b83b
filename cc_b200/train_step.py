"""One Competitive-Collaboration training step on the libccb200 kernels - the body of the reference's
``train()`` loop (train.py:445-568) for the BASELINE.json configurations:

  cfg1  DispResNet6 + PoseNetB6 depth/pose step (explainability_mask = [None]*6)
  cfg2  Back2Future flow + flow photometric/SSIM + smoothness
  cfg3  full joint step (Disp + Pose + Mask + Flow, all five losses)

The flow net is Back2Future unless `flownet='FlowNetC6'` is chosen, as the reference's --flownet (train.py:90,252-255).

Hyper-parameters default to the README command line (README.md:59-65; train.py:120-130)."""
import torch
from . import models, loss_functions as LF, dist as cdist
from .inverse_warp import pose2flow
from .optim import FlatAdam

HP = dict(w1=1.0, w2=0.1, w3=0.1, w4=0.5, w5=0.3, wssim=0.997, qch=0.5, lambda_oob=0.0,
          THRESH=0.01, wbce=0.5, wrig=1.0, lr=1e-4, beta1=0.9, beta2=0.999, smoothness='edgeaware')
NETS_OF = {'cfg1': ('disp', 'pose'), 'cfg2': ('flow',), 'cfg3': ('disp', 'pose', 'mask', 'flow')}
FLOWNETS = ('Back2Future', 'FlowNetC6')          # the choices of --flownet, train.py:90


def build_nets(cfg, device, state_dicts=None, seed=0, flownet='Back2Future'):
    """Instantiate the nets of a configuration (reference constructor arguments, train.py:245-255)."""
    if flownet not in FLOWNETS:
        raise ValueError('flownet must be one of %s, got %r' % (FLOWNETS, flownet))
    torch.manual_seed(seed)
    nets = {}
    for name in NETS_OF[cfg]:
        if name == 'disp':
            net = models.DispResNet6()
        elif name == 'pose':
            net = models.PoseNetB6(nb_ref_imgs=4)
        elif name == 'mask':
            net = models.MaskNet6(nb_ref_imgs=4, output_exp=True)
        elif flownet == 'FlowNetC6':
            net = models.FlowNetC6(nlevels=6)
        else:
            # the five occlusion decoders are dead work in training: train.py:463 discards `occ` and they get no
            # gradient (SURVEY.md F9); their parameters stay in the module (checkpoint contract) and in the optimiser
            net = models.Back2Future(nlevels=6, compute_occ=False)
        net.init_weights()
        if state_dicts is not None and name in state_dicts:
            net.load_state_dict({k: v.clone() for k, v in state_dicts[name].items()}, strict=True)
        nets[name] = net.to(device).train()
    return nets


def _smooth(hp, tgt, preds):
    if hp['smoothness'] == 'edgeaware':
        return LF.edge_aware_smoothness_loss(tgt, preds)
    return LF.smooth_loss(preds)


def flow_pair(flow_net, tgt, refs):
    """(flow_fwd, flow_bwd) of the training step, train.py:462-466: Back2Future sees both neighbours in one call,
    another flow net is called once per direction (the target tower is recomputed in each call, as in the reference)."""
    if isinstance(flow_net, models.Back2Future):
        ff, fb, _ = flow_net(tgt, refs[1:3])
        return ff, fb
    return flow_net(tgt, refs[2]), flow_net(tgt, refs[1])


def loss_cfg1(nets, tgt, refs, K, Kinv, hp=HP):
    disp = nets['disp'](tgt)
    depth = [1 / d for d in disp]
    pose = nets['pose'](tgt, refs)
    l1 = LF.photometric_reconstruction_loss(tgt, refs, K, Kinv, depth, [None] * len(depth), pose,
                                            lambda_oob=hp['lambda_oob'], qch=hp['qch'], wssim=hp['wssim'])
    l3 = _smooth(hp, tgt, depth)
    return hp['w1'] * l1 + hp['w3'] * l3, dict(loss_1=l1, loss_3=l3, disp=disp, pose=pose)


def loss_cfg2(nets, tgt, refs, K, Kinv, hp=HP):
    ff, fb = flow_pair(nets['flow'], tgt, refs)
    l4 = LF.photometric_flow_loss(tgt, refs[1:3], [fb, ff], [None] * len(ff),
                                  lambda_oob=hp['lambda_oob'], qch=hp['qch'], wssim=hp['wssim'])
    l3 = _smooth(hp, tgt, ff) + _smooth(hp, tgt, fb)
    return hp['w4'] * l4 + hp['w3'] * l3, dict(loss_4=l4, loss_3=l3, flow_fwd=ff, flow_bwd=fb)


def loss_cfg3(nets, tgt, refs, K, Kinv, hp=HP):
    """Reference train.py:454-509."""
    disp = nets['disp'](tgt)
    depth = [1 / d for d in disp]
    pose = nets['pose'](tgt, refs)
    emask = nets['mask'](tgt, refs)
    ff, fb = flow_pair(nets['flow'], tgt, refs)
    cam_f = [pose2flow(d.squeeze(1), pose[:, 2], K, Kinv) for d in depth]
    cam_b = [pose2flow(d.squeeze(1), pose[:, 1], K, Kinv) for d in depth]
    tgt_masks = LF.consensus_exp_masks(cam_f, cam_b, ff, fb, tgt, refs[2], refs[1],
                                       wssim=hp['wssim'], wrig=hp['wrig'], ws=hp['w3'])
    rig_f = [(a - b).abs() for a, b in zip(cam_f, ff)]
    rig_b = [(a - b).abs() for a, b in zip(cam_b, fb)]
    flow_emask = [1 - m[:, 1:3] for m in emask]
    l1 = LF.photometric_reconstruction_loss(tgt, refs, K, Kinv, depth, emask, pose,
                                            lambda_oob=hp['lambda_oob'], qch=hp['qch'], wssim=hp['wssim'])
    l2 = LF.explainability_loss(emask) if hp['w2'] > 0 else 0
    l3 = _smooth(hp, tgt, depth) + _smooth(hp, tgt, ff) + _smooth(hp, tgt, fb) + _smooth(hp, tgt, emask)
    l4 = LF.photometric_flow_loss(tgt, refs[1:3], [fb, ff], flow_emask,
                                  lambda_oob=hp['lambda_oob'], qch=hp['qch'], wssim=hp['wssim'])
    l5 = LF.consensus_depth_flow_mask(emask, rig_b, rig_f, tgt_masks, tgt_masks, THRESH=hp['THRESH'], wbce=hp['wbce'])
    loss = hp['w1'] * l1 + hp['w2'] * l2 + hp['w3'] * l3 + hp['w4'] * l4 + hp['w5'] * l5
    return loss, dict(loss_1=l1, loss_2=l2, loss_3=l3, loss_4=l4, loss_5=l5, disp=disp, pose=pose, emask=emask,
                      flow_fwd=ff, flow_bwd=fb)


LOSS_FNS = {'cfg1': loss_cfg1, 'cfg2': loss_cfg2, 'cfg3': loss_cfg3}


class Trainer:
    """Nets + one flat Adam + (optionally) one NCCL gradient all-reduce; `step()` is
    optimizer.zero_grad(); loss.backward(); optimizer.step() of train.py:566-568.

    `fixed` names nets of the configuration that are not trained, as the reference's --fix-dispnet / --fix-posenet /
    --fix-masknet / --fix-flownet (train.py:332-346): their parameters get requires_grad = False, so no gradient reaches
    them, and their Adam group keeps its step count.  They stay in train mode (a fixed DispResNet6 still updates its
    BatchNorm running statistics, train.py:438-441).  The README's command is Trainer('cfg3', dev, fixed=('mask', 'flow'))."""

    def __init__(self, cfg, device, hp=HP, state_dicts=None, seed=0, flownet='Back2Future', fixed=()):
        self.cfg, self.hp, self.device, self.flownet = cfg, dict(hp), device, flownet
        self.nets = build_nets(cfg, device, state_dicts, seed, flownet)
        # one Adam group per net, in the reference's chain(disp, pose, mask, flow) order (train.py:307)
        groups = [list(self.nets[n].parameters()) for n in NETS_OF[cfg]]
        self.opt = FlatAdam([p for g in groups for p in g], lr=hp['lr'], betas=(hp['beta1'], hp['beta2']), groups=groups)
        cdist.broadcast_params(self.opt)
        self.buckets = cdist.GradBuckets(self.opt)          # overlapped gradient exchange (no-op at world size 1)
        self.graph = None
        self.fixed = ()
        # prepared conv weights are refreshed once per optimiser step (one launch), not once per conv call
        from . import nn as cnn, _lib
        self.wcache = None if (_lib.is_simulator() or torch.device(device).type != 'cuda') else cnn.WeightCache(torch.device(device))
        self.set_fixed(fixed)

    def set_fixed(self, fixed):
        """Change the set of fixed nets (between epochs or phases of training).  Drops any captured graph and the learned
        gradient buckets (re-learned on the next step)."""
        names = NETS_OF[self.cfg]
        want = (fixed,) if isinstance(fixed, str) else tuple(fixed)
        bad = [n for n in want if n not in names]
        if bad:
            raise ValueError('fixed nets %s are not nets of %s %s' % (bad, self.cfg, names))
        fixed = tuple(n for n in names if n in want)
        if len(fixed) == len(names):
            raise ValueError('every net of %s is fixed: there is nothing to train' % self.cfg)
        for n, group in zip(names, self.opt.groups):
            for p in group:
                p.requires_grad_(n not in fixed)
        self.opt.freeze([i for i, n in enumerate(names) if n in fixed])
        if fixed != self.fixed:
            self.graph = None
            if self.buckets.enabled and self.buckets.buckets is not None:
                # the next step re-learns the buckets and re-packs the flat buffers; the weight cache keys its copies by
                # parameter address, so it records its layouts again after that
                self.buckets.buckets = None
                if self.wcache is not None:
                    from . import nn as cnn
                    self.wcache = cnn.WeightCache(self.wcache.device)
        self.fixed = fixed

    def refresh_weights(self):
        """Call after changing parameters behind the trainer's back (load_state_dict, manual edits)."""
        if self.wcache is not None:
            self.wcache.refresh()

    def step(self, tgt, refs, K, Kinv):
        from . import nn as cnn, pyramid
        pyramid.clear()                                     # the per-step memo of frame pyramids never outlives a step
        self.opt.zero_grad()
        self.buckets.begin()
        # the weight cache keys its copies by parameter address: it starts recording only after the bucket scheduler has
        # re-packed the flat buffers (its learning step moves every parameter)
        use_cache = self.wcache is not None and (not self.buckets.enabled or self.buckets.buckets is not None)
        cnn.WCACHE = self.wcache.h if use_cache else None
        try:
            loss, aux = LOSS_FNS[self.cfg](self.nets, tgt, refs, K, Kinv, self.hp)
            loss.backward()
        finally:
            cnn.WCACHE = None
        self.buckets.finish()                               # waits for the bucket all-reduces issued during backward
        self.opt.step()
        if use_cache:
            if not self.wcache.committed:
                self.wcache.commit()                        # this step recorded the layouts: allocate + prepare
            else:
                self.wcache.refresh()
        pyramid.clear()
        return loss.detach(), aux

    def _snapshot(self):
        bufs = [b for n in self.nets.values() for b in n.buffers()]
        return self.opt.snapshot(), [b.clone() for b in bufs]

    def _restore(self, snap):
        self.opt.restore(snap[0])
        with torch.no_grad():
            for b, s in zip([b for n in self.nets.values() for b in n.buffers()], snap[1]):
                b.copy_(s)
        self.refresh_weights()

    # ---- whole-step CUDA graph (static shapes): removes per-launch host latency --------------------
    def capture(self, tgt, refs, K, Kinv, warmup=2):
        """Capture zero_grad + forward + backward + all-reduce + Adam into one CUDA graph replaying on
        the static input buffers `tgt/refs/K/Kinv` (the caller copies each batch into them)."""
        from . import pyramid, nn as cnn
        self.static_in = (tgt, refs, K, Kinv)
        assert bool(torch.isfinite(tgt).all()), 'capture(): the static input buffers must hold a real batch'
        # The warm-up runs real steps (allocator warm-up; bucket learning on the first one): they must not train.
        # Parameters, Adam moments / step counter and BatchNorm buffers are restored afterwards.
        snap = self._snapshot()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            need = 2 if (self.buckets.enabled and self.buckets.buckets is None) else 0
            if self.wcache is not None and not self.wcache.committed:
                need = max(need, 1)                     # the weight cache records its layouts in an eager step
            for _ in range(max(warmup, need)):
                pyramid.clear()
                self.step(tgt, refs, K, Kinv)
        torch.cuda.current_stream().wait_stream(s)
        self._restore(snap)
        pyramid.clear()
        cnn.GRAPH_LIVE = True                                # conv workspaces referenced by the graph are never freed
        self._captured = dict(lr=self.opt.lr, grad_scale=self.opt.grad_scale, fixed=self.fixed)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.static_loss, _ = self.step(tgt, refs, K, Kinv)
        self._restore(snap)                                  # capture itself does not execute, but keep the contract explicit
        pyramid.clear()
        return self.graph

    def replay(self):
        # lr and grad_scale are kernel arguments baked into the graph: refuse to replay a stale one
        assert self.opt.lr == self._captured['lr'] and self.opt.grad_scale == self._captured['grad_scale'], \
            'learning rate / world size changed after capture(): re-capture the step'
        # the fixed set decides which gradients and Adam ranges the graph computes (set_fixed() drops the graph)
        assert self.graph is not None and self.fixed == self._captured['fixed'], \
            'the fixed nets changed after capture(): re-capture the step'
        self.graph.replay()
        return self.static_loss


class HostFeeder:
    """Pinned-host batches -> the trainer's static input buffers, one batch ahead.

    The reference's DataLoader (train.py: pin_memory=True, `.to(device)` in the loop) hands the step a fresh host batch
    every iteration.  Here batch i+1 crosses PCIe on a copy stream while step i computes; `feed(i)` waits for batch i,
    copies it device-to-device into the static buffers the CUDA graph reads, and starts the transfer of batch i+1.
    Every batch still crosses PCIe exactly once; only the wait is hidden."""

    def __init__(self, static_inputs, batch_of):
        self.static = list(static_inputs)                  # device tensors the (captured) step reads
        self.batch_of = batch_of                           # i -> list of pinned host tensors, same order / shapes
        self.stage = [[torch.empty_like(t) for t in self.static] for _ in range(2)]
        self.stream = torch.cuda.Stream()
        self.ready = [torch.cuda.Event(), torch.cuda.Event()]
        self.next = None

    def _start(self, i):
        self.stream.wait_stream(torch.cuda.current_stream())      # the slot's previous reader (a D2D copy) is done
        with torch.cuda.stream(self.stream):
            for d, h in zip(self.stage[i & 1], self.batch_of(i)):
                d.copy_(h, non_blocking=True)
            self.ready[i & 1].record(self.stream)
        self.next = i

    def feed(self, i, prefetch=True):
        if self.next != i:
            self._start(i)
        torch.cuda.current_stream().wait_event(self.ready[i & 1])
        for s, d in zip(self.static, self.stage[i & 1]):
            s.copy_(d, non_blocking=True)
        if prefetch:
            self._start(i + 1)
