"""Step-level parity: cc_b200.train_step.Trainer (nets + fused losses + flat Adam) vs the oracle's
train_step (reference train.py:445-568 restated) on identical seeded inputs / weights."""
import math
import torch
from tests.util import assert_close, rel_err, conv_impl
from cc_b200 import synth, nn as cnn, pyramid, _lib, models as CM
from cc_b200.optim import FlatAdam
from cc_b200.train_step import Trainer, HP, NETS_OF
from oracle import step as OS, nets as ON
from tests import flownetc6_cases as FC6

U32 = 2.0 ** -24           # fp32 unit roundoff
TINY32 = 1e-44             # a few fp32 subnormal steps: the absolute error of a product that underflows


def f32(x):
    """A Python float rounded to fp32: FlatAdam hands lr, betas and eps to its kernel as fp32 arguments."""
    return float(torch.tensor(x, dtype=torch.float32))


def adam_reference(p, m, v, g, t, lr, betas, eps, grad_scale=1.0):
    """One torch.optim.Adam step (weight decay 0, step count t after the step) in fp64 from the fp32 state before it
    (oracle/step.Adam's update), and per-element bounds on what an fp32 evaluation of that step may differ by.
    Returns ((p, m, v), (bound_p, bound_m, bound_v)), all fp64.  Pass lr / betas / eps as the kernel receives them (f32).

    The bounds are error analysis of one fp32 step, u = 2^-24, |.| elementwise, g' = grad_scale * g:
      m:  4u (b1 |m| + (1 - b1) |g'|)              - relative to the summands, not to m: m cancels when g changes sign
      v:  6u v                                     - every term is non-negative
      p:  2u |p| + 8u |upd| + |upd| dd / denom + (lr / bc1) bound_m / denom
          fl(p - upd) rounds once (2u |p|: about an ulp of p); the update itself takes ~6 roundings, including the fp32
          bias corrections kept in the optimiser state (8u |upd|); the error allowed in m and in v (dd: the change of
          denom when v moves by bound_v) passes into the update through m / denom.
    TINY32 is added to every bound, for squares and products of gradients that underflow fp32."""
    p, m, v, g = (x.double() for x in (p, m, v, g))
    b1, b2 = betas
    g = g * grad_scale
    m1 = b1 * m + (1 - b1) * g
    v1 = b2 * v + (1 - b2) * g * g
    bc1, bc2s = 1 - b1 ** t, math.sqrt(1 - b2 ** t)
    denom = v1.sqrt() / bc2s + eps
    upd = (lr / bc1) * m1 / denom
    p1 = p - upd
    bm = 4 * U32 * (b1 * m.abs() + (1 - b1) * g.abs()) + TINY32
    bv = 6 * U32 * v1 + TINY32
    dd = ((v1 + bv).sqrt() - v1.sqrt()) / bc2s
    bp = 2 * U32 * p1.abs() + 8 * U32 * upd.abs() + upd.abs() * dd / denom + (lr / bc1) * bm / denom + TINY32
    return (p1, m1, v1), (bp, bm, bv)


def assert_adam_step(before, after, g, t, lr, betas, eps, grad_scale, what):
    """`after` = (flat_p, exp_avg, exp_avg_sq, state) of a FlatAdam right after its t-th step from `before` (the same
    fp32 buffers, state excluded) with gradient g: every element within adam_reference's bound, state[:3] = the step
    count and the bias corrections 1 - b1^t, sqrt(1 - b2^t) of step t."""
    lr, betas, eps = f32(lr), (f32(betas[0]), f32(betas[1])), f32(eps)
    n, chunk = g.numel(), 1 << 23               # fp64 temporaries of a full-size model, a slice at a time
    for c0 in range(0, n, chunk):
        sl = slice(c0, min(n, c0 + chunk))
        ref, bound = adam_reference(before[0][sl], before[1][sl], before[2][sl], g[sl], t, lr, betas, eps, grad_scale)
        for got, r, b, nm in zip(after[:3], ref, bound, ('flat_p', 'exp_avg', 'exp_avg_sq')):
            got = got[sl]
            err = (got.double() - r).abs()
            bad = err > b
            if bool(bad.any()):
                i = int((err / b).argmax())
                raise AssertionError(f'{what}: {nm}: {int(bad.sum())} of {err.numel()} elements from {c0} outside the fp32 '
                                     f'bound; worst [{c0 + i}] {got[i].item():.9g} vs fp64 {r[i].item():.9g} (bound {b[i].item():.3g})')
    st = after[3].double().cpu()
    want = torch.tensor([float(t), 1 - betas[0] ** t, math.sqrt(1 - betas[1] ** t)], dtype=torch.float64)
    assert st[0].item() == t and bool(((st[1:3] - want[1:]).abs() <= 2 * U32 * want[1:]).all()), \
        f'{what}: optimiser state {st[:3].tolist()}, want {want.tolist()}'


def case_adam_fp64(device, steps=5):
    """FlatAdam (ccb_adam_step_ranges, one group) over three parameters for 5 steps against the fp64 reference, element by
    element, on synthetic gradients: exact zeros (every step, or every other step), values near eps (1e-9 .. 1e-7), large values
    (1e4), ordinary ones, with random signs that change from step to step, and one step with grad_scale = 0.5.
    Parameters span 1 .. 1e-4 with exact zeros, so the updates are not hidden under the parameters' ulp.  Each step
    starts from the optimiser's own previous buffers; the bounds are adam_reference's."""
    gen = torch.Generator().manual_seed(5)
    shapes = [(16, 3, 3, 3), (257,), (1000,)]
    params = []
    for s in shapes:
        p0 = torch.randn(s, generator=gen) * 10.0 ** (-4 * torch.rand(s, generator=gen))
        p0.view(-1)[::7] = 0.0
        params.append(torch.nn.Parameter(p0.to(device)))
    opt = FlatAdam(params, lr=1e-3)
    n = opt.numel
    cls = torch.arange(n) % 5
    mag = torch.where(cls == 1, 10.0 ** (-9 + 2 * torch.rand(n, generator=gen)),        # near eps
                      torch.where(cls == 2, 1e4 * (0.5 + torch.rand(n, generator=gen)),  # large
                                  torch.randn(n, generator=gen).abs() * 1e-2))           # ordinary
    mag[cls == 0] = 0.0                                                                   # zero at every step
    for t in range(1, steps + 1):
        sign = torch.where(torch.rand(n, generator=gen) < 0.5, -1.0, 1.0)
        g = mag * sign
        if t % 2 == 1:
            g[cls == 4] = 0.0                                                             # zero every other step
        gs = 0.5 if t == 3 else 1.0
        before = (opt.flat_p.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone())
        opt.flat_g.copy_(g.to(device))
        opt.grad_scale = gs
        opt.step()
        after = (opt.flat_p.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone(), opt.state.clone())
        assert_adam_step(before, after, g.to(device), t, opt.lr, opt.betas, opt.eps, gs, f'FlatAdam step {t}')
        assert torch.equal(after[0][cls.to(device) == 0], before[0][cls.to(device) == 0]), 'a parameter without gradient moved'
    opt.grad_scale = 1.0


def case_flat_adam(device):
    """Two conv layers trained 3 steps: FlatAdam (direct flat-buffer weight grads) vs torch.optim.Adam."""
    torch.manual_seed(0)
    c1, c2 = cnn.Conv2d(3, 8, 3, padding=1, act='relu').to(device), cnn.Conv2d(8, 2, 3, padding=1).to(device)
    r1, r2 = torch.nn.Conv2d(3, 8, 3, padding=1).to(device), torch.nn.Conv2d(8, 2, 3, padding=1).to(device)
    for a, b in ((c1, r1), (c2, r2)):
        b.load_state_dict(a.state_dict())
    x = torch.randn(2, 3, 9, 11, generator=torch.Generator().manual_seed(1)).to(device)
    opt = FlatAdam(list(c1.parameters()) + list(c2.parameters()), lr=1e-2)
    ropt = torch.optim.Adam(list(r1.parameters()) + list(r2.parameters()), lr=1e-2)
    for _ in range(3):
        opt.zero_grad()
        l = (c2(c1(x)) ** 2).mean()
        l.backward()
        opt.step()
        ropt.zero_grad()
        lr_ = (r2(torch.relu(r1(x))) ** 2).mean()
        lr_.backward()
        ropt.step()
        assert_close(l, lr_, 1e-5, 'loss')
    for a, b in ((c1, r1), (c2, r2)):
        assert_close(a.weight, b.weight, 1e-4, 'weight after 3 Adam steps')
        assert_close(a.bias, b.bias, 1e-4, 'bias after 3 Adam steps')
    assert abs(opt.state[0].item() - 3.0) < 1e-6


def oracle_state_dicts(P):
    """The oracle's parameter dicts as state dicts for Trainer / build_nets: detached copies."""
    return {n: {k: v.detach().clone() for k, v in d.items()} for n, d in P.items()}


def case_step_cfg1(device, B=2, H=128, W=416, steps=2, gtol=4e-3):
    """cfg1 (BASELINE.json configs[1] at reduced batch/size): loss and gradients of step 1, loss of step 2.
    gtol: 4e-3 with the exact-fp32 FFMA convolutions (measured 1.3e-3: fp32 noise through ~50 layers incl.
    batch-stat BNs over <= 8 values); the tensor-core (3xTF32) path is held to 5e-2 on the same gradients."""
    tgt, refs = synth.frames(B, H, W, seed=50)
    K, Kinv = synth.intrinsics(B, H, W)
    P = OS.make_params('cfg1')
    tr = Trainer('cfg1', device, state_dicts=oracle_state_dicts(P))
    oopt = OS.Adam(OS.all_params(P), HP['lr'], HP['beta1'], HP['beta2'])
    dt, dr, dK, dKi = tgt.to(device), [r.to(device) for r in refs], K.to(device), Kinv.to(device)
    for s in range(steps):
        lo, _ = OS.train_step('cfg1', P, oopt, tgt, refs, K, Kinv)
        lc, _ = tr.step(dt, dr, dK, dKi)
        assert_close(lc, lo, 2e-4, f'cfg1 loss step {s}')
        if s == 0:
            for net in ('disp', 'pose'):
                for name, p in tr.nets[net].named_parameters():
                    g = P[net][name].grad
                    if g is None:
                        continue
                    if name in ('conv1.0.weight', 'conv1.2.weight', 'conv4.0.conv1.weight', 'iconv2.0.conv2.weight',
                                'predict_disp1.0.weight', 'upconv3.0.weight', 'pose_pred.weight', 'conv7.0.downsample.1.weight'):
                        # fp32 noise accumulated through ~50 layers incl. batch-stat BNs over <= 8 values: measured 1.3e-3
                        assert_close(p._ccb_grad, g, gtol, f'{net}.{name} grad')
    return tr


def case_step_cfg3(device, B=2, H=64, W=128):
    """Full joint step (BASELINE.json configs[3] at reduced size): all five loss terms + total vs the oracle."""
    from cc_b200.train_step import loss_cfg3, build_nets
    tgt, refs = synth.frames(B, H, W, seed=60)
    K, Kinv = synth.intrinsics(B, H, W)
    P = OS.make_params('cfg3')
    lo, auxo = OS.loss_cfg3(P, tgt, refs, K, Kinv)
    lo.backward()
    nets = build_nets('cfg3', device, state_dicts=oracle_state_dicts(P))
    dt, dr, dK, dKi = tgt.to(device), [r.to(device) for r in refs], K.to(device), Kinv.to(device)
    lc, auxc = loss_cfg3(nets, dt, dr, dK, dKi)
    lc.backward()
    for k in ('loss_1', 'loss_2', 'loss_3', 'loss_4', 'loss_5'):
        assert_close(auxc[k], auxo[k], 1e-3, 'cfg3 ' + k)
    assert_close(lc, lo, 1e-3, 'cfg3 total loss')
    for i in range(6):
        assert_close(auxc['flow_fwd'][i], auxo['flow_fwd'][i], 1e-3, f'cfg3 flow_fwd{i}')
        assert_close(auxc['emask'][i], auxo['emask'][i], 1e-3, f'cfg3 emask{i}')
    # every parameter of every net received a gradient of the right magnitude (Back2Future's occ decoders excepted)
    for net in ('disp', 'pose', 'mask', 'flow'):
        go = torch.sqrt(sum((t.grad ** 2).sum() for t in P[net].values() if t.requires_grad and t.grad is not None))
        gc = torch.sqrt(sum((p.grad ** 2).sum() for p in nets[net].parameters() if p.grad is not None))
        assert_close(gc, go, 5e-2, f'cfg3 grad norm {net}')


def _record(tr, loss=None):
    """Device copies of everything one training step changes: loss, flat gradient / parameter / Adam buffers, optimiser
    state, every BatchNorm buffer (running statistics and batch counters)."""
    o = tr.opt
    rec = dict(flat_g=o.flat_g.clone(), flat_p=o.flat_p.clone(), exp_avg=o.exp_avg.clone(), exp_avg_sq=o.exp_avg_sq.clone(),
               state=o.state.clone())
    rec.update(('%s.%s' % (n, k), b.clone()) for n, net in tr.nets.items() for k, b in net.named_buffers())
    if loss is not None:
        rec['loss'] = loss.detach().clone()
    return rec


def _assert_same(got, want, what, skip=()):
    for k in want:
        if k in skip:
            continue
        a, b = got[k], want[k]
        if not torch.equal(a, b):
            d = (a.double() - b.double()).abs()
            raise AssertionError(f'{what}: {k} differs in {int((a != b).sum())} of {a.numel()} elements (max {d.max().item():.3e})')


def group_range(opt, gi):
    """(lo, hi) of group gi in the flat buffers (contiguous in the constructor layout)."""
    offs = sorted(opt.offset[p] for p in opt.groups[gi])
    lo, hi = offs[0][0], offs[-1][0] + offs[-1][1]
    assert hi - lo == sum(k for _, k in offs), 'group %d is not contiguous' % gi
    return lo, hi


def assert_groups_step(tr, before, after, want_t, what):
    """Per net of the trainer: an active group's range within assert_adam_step's bound for its own t (want_t[name]); a
    frozen group's parameters, moments and counter bit-unchanged and its gradient range exactly zero."""
    o = tr.opt
    for gi, name in enumerate(NETS_OF[tr.cfg]):
        lo, hi = group_range(o, gi)
        sl = slice(lo, hi)
        st = slice(4 * gi, 4 * gi + 4)
        if name in tr.fixed:
            for k in ('flat_p', 'exp_avg', 'exp_avg_sq'):
                assert torch.equal(after[k][sl], before[k][sl]), f'{what}: fixed {name}: {k} changed'
            assert torch.equal(after['state'][st], before['state'][st]), f'{what}: fixed {name}: step counter changed'
            assert not bool(after['flat_g'][sl].any()), f'{what}: fixed {name} received a gradient'
        else:
            assert_adam_step((before['flat_p'][sl], before['exp_avg'][sl], before['exp_avg_sq'][sl]),
                             (after['flat_p'][sl], after['exp_avg'][sl], after['exp_avg_sq'][sl], after['state'][st]),
                             after['flat_g'][sl], want_t[name], o.lr, o.betas, o.eps, o.grad_scale, f'{what}: {name}')


def case_step_graph_vs_eager(device, cfg, B=2, H=64, W=128, loss_tol=None, seed=70, flownet='Back2Future', fixed=()):
    """The step the benchmark times - Trainer.capture() + replay(): a CUDA graph whose convolutions read a committed
    weight cache and whose Adam keeps its step counts on the device - against Trainer.step() run eagerly, over three
    steps on three different seeded batches, both trainers Trainer(cfg, flownet=flownet, fixed=fixed) built from the same
    oracle weights (FlowNetC6: flownetc6_cases.step_flow_params).

      * replay i equals eager step i BIT FOR BIT: loss, flat gradient / parameters / Adam moments, optimiser state,
        BatchNorm buffers.  (Eager step 0 prepares weights per call while recording the cache; every later step and
        every replay reads what wprep_all_kernel prepared.  Different batches: the replay reads the static inputs.)
      * capture() runs real warm-up steps; afterwards parameters, moments, state and BatchNorm buffers equal the
        snapshot taken before it, bit for bit (the flat gradient still holds warm-up gradients; the graph zeroes it).
        capture() restores the snapshot after the warm-up and again after capturing, which executes nothing, so this
        fails only when neither restore runs.
      * each replay, per Adam group (assert_groups_step): a trained net's parameters / moments / step counter against
        the fp64 Adam reference (adam_reference) applied to that replay's own gradient, from the state recorded before
        it; a fixed net bit-unchanged with an exactly zero gradient.
      * the weight cache is committed, hit, and never missed; the flow net is the one asked for.
      * loss_tol: eager losses against oracle.step.train_step run on the CPU for the same three steps, the fixed nets'
        oracle parameters excluded from its Adam.
      * replay() refuses a graph whose learning rate is stale, and with `fixed`, one captured under another fixed set.
    The trainers run one after the other (full size: one set of activations at a time)."""
    batches = []
    for i in range(3):
        tgt, refs = synth.frames(B, H, W, seed=seed + i)
        batches.append([tgt] + refs + list(synth.intrinsics(B, H, W)))
    P = OS.make_params(cfg)
    if flownet == 'FlowNetC6':
        P['flow'] = ON.clone_params(FC6.step_flow_params(), requires_grad=True)
    sd = oracle_state_dicts(P)
    tag = f'{cfg} {B}x{H}x{W}' + ('' if flownet == 'Back2Future' else ' ' + flownet) + (f' fixed={fixed}' if fixed else '')
    saved = cnn.GRAPH_LIVE
    tr = None
    try:
        with conv_impl(_lib.IMPL_AUTO):
            tr = Trainer(cfg, device, state_dicts=sd, flownet=flownet, fixed=fixed)
            eager = []
            for b in batches:
                d = [t.to(device) for t in b]
                loss, _ = tr.step(d[0], d[1:5], d[5], d[6])
                eager.append(_record(tr, loss))
            del tr, loss, d
            tr = None
            torch.cuda.empty_cache()

            tr = Trainer(cfg, device, state_dicts=sd, flownet=flownet, fixed=fixed)
            if 'flow' in tr.nets:
                assert isinstance(tr.nets['flow'], getattr(CM, flownet)), type(tr.nets['flow'])
            static = [t.to(device) for t in batches[0]]
            snap = _record(tr)
            tr.capture(static[0], static[1:5], static[5], static[6])
            _assert_same(_record(tr), snap, f'{tag}: state after capture()', skip=('flat_g',))
            assert tr.wcache is not None and tr.wcache.committed
            prev = snap
            for i, b in enumerate(batches):
                for s, h in zip(static, b):
                    s.copy_(h)
                cur = _record(tr, tr.replay())
                _assert_same(cur, eager[i], f'{tag}: replay {i} vs eager step {i}')
                assert_groups_step(tr, prev, cur, {n: i + 1 for n in NETS_OF[cfg]}, f'{tag}: Adam of replay {i}')
                prev = cur
            stats = tr.wcache.stats()
            assert stats['hits'] > 0 and stats['misses'] == 0, stats
            o = tr.opt
            lr = o.lr
            o.lr = lr * 0.5
            try:
                tr.replay()
                raise RuntimeError('replay() ran a graph captured with another learning rate')
            except AssertionError:
                pass
            finally:
                o.lr = lr
            if fixed:
                tr.set_fixed(fixed[:-1])
                try:
                    tr.replay()
                    raise RuntimeError('replay() ran a graph captured under another fixed set')
                except AssertionError:
                    pass
    finally:
        if tr is not None:
            tr.graph = None
        tr = None
        torch.cuda.synchronize()
        cnn.GRAPH_LIVE = saved
        pyramid.clear()
    if loss_tol is not None:
        for n in fixed:
            for t in P[n].values():
                t.requires_grad_(False)
        oopt = OS.Adam(OS.all_params(P), HP['lr'], HP['beta1'], HP['beta2'])
        errs = []
        for i, b in enumerate(batches):
            lo, _ = OS.train_step(cfg, P, oopt, b[0], b[1:5], b[5], b[6], flownet=flownet)
            errs.append(rel_err(eager[i]['loss'], lo))
        assert max(errs) <= loss_tol, f'{tag}: relative loss errors of steps 0-2 vs the oracle ' \
                                      f'{["%.2e" % e for e in errs]}, bar {loss_tol:.0e}'
        print(f'{tag}: loss vs oracle {["%.2e" % e for e in errs]}')


STEP_CASES_SIM = [case_flat_adam, case_adam_fp64]
