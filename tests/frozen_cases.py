"""Training with fixed networks (the reference's --fix-* flags): Adam over ranges with one step counter per network, and
the photometric loss without the outputs autograd would throw away.  Shared by the CPU-simulator suite
(tests/test_frozen.py) and the GPU suite (tests/test_gpu_frozen.py)."""
import itertools
import torch
from tests.util import assert_close
from tests.step_cases import assert_adam_step, assert_groups_step, group_range, oracle_state_dicts, _record
from tests import kernel_cases as KC
from cc_b200 import _lib, synth, pyramid, nn as cnn, loss_functions as CL
from cc_b200.optim import FlatAdam, ADAM_BLOCK
from cc_b200.train_step import Trainer, NETS_OF


# ---- Adam over ranges ------------------------------------------------------------------------------------------------
def _adam_setup(device):
    """Three groups of parameters spanning 1 .. 1e-4 with exact zeros, and case_adam_fp64's gradient classes: exact
    zeros, values near eps, large values, ordinary ones."""
    gen = torch.Generator().manual_seed(5)
    shapes = [(16, 3, 3, 3), (257,), (1000,), (300,)]
    params = []
    for s in shapes:
        p0 = torch.randn(s, generator=gen) * 10.0 ** (-4 * torch.rand(s, generator=gen))
        p0.view(-1)[::7] = 0.0
        params.append(torch.nn.Parameter(p0.to(device)))
    groups = [[params[0], params[3]], [params[1]], [params[2]]]
    opt = FlatAdam(params, lr=1e-3, groups=groups)
    n = opt.numel
    cls = torch.arange(n) % 5
    mag = torch.where(cls == 1, 10.0 ** (-9 + 2 * torch.rand(n, generator=gen)),
                      torch.where(cls == 2, 1e4 * (0.5 + torch.rand(n, generator=gen)),
                                  torch.randn(n, generator=gen).abs() * 1e-2))
    mag[cls == 0] = 0.0
    return opt, mag, gen


def _group_mask(opt, gi, device):
    m = torch.zeros(opt.numel, dtype=torch.bool)
    for p in opt.groups[gi]:
        off, k = opt.offset[p]
        m[off:off + k] = True
    return m.to(device)


def _step_ranges(opt, table):
    """ccb_adam_step_ranges over an explicit [(offset, count, group)] table (the optimiser's own buffers and state)."""
    rows, nb = [], 0
    for off, k, gi in table:
        rows += [off, k, gi, nb]
        nb += (k + ADAM_BLOCK - 1) // ADAM_BLOCK
    t = torch.tensor(rows, dtype=torch.int64).to(opt.flat_p.device)
    _lib.call('ccb_adam_step_ranges', opt.flat_p, opt.flat_g, opt.exp_avg, opt.exp_avg_sq, t, len(table), nb, opt._active,
              len(opt.groups), opt.state, opt.lr, opt.betas[0], opt.betas[1], opt.eps, opt.grad_scale, opt.flat_p)


def case_adam_ranges_fp64(device, steps=4):
    """Three groups at step counts 3, 0 and 7, the second frozen: every active element within adam_reference's fp64
    bound for its own group's t; the frozen group's parameters, moments and counter bit-unchanged; and the same step
    with the active ranges cut into more pieces (at offsets that are not multiples of the block) gives the same bits."""
    opt, mag, gen = _adam_setup(device)
    n = opt.numel
    with torch.no_grad():
        opt.state.view(-1, 4)[:, 0] = torch.tensor([3.0, 0.0, 7.0])
        opt.exp_avg.copy_((torch.randn(n, generator=gen) * 1e-3).to(device))
        opt.exp_avg_sq.copy_((torch.rand(n, generator=gen) * 1e-5).to(device))
    opt.freeze([1])
    assert opt.ranges() == [(0, 432, 0), (689, 1000, 2), (1689, 300, 0)], opt.ranges()
    frozen = _group_mask(opt, 1, device)
    for s in range(1, steps + 1):
        sign = torch.where(torch.rand(n, generator=gen) < 0.5, -1.0, 1.0)
        g = (mag * sign).to(device)
        opt.flat_g.copy_(g)
        before = (opt.flat_p.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone(), opt.state.clone())
        # the same step through a table of smaller pieces, from the same buffers
        pieces = []
        for off, k, gi in opt.ranges():
            cuts = sorted({0, k} | {c for c in (1, 255, 300, 511, 700) if c < k})
            pieces += [(off + a, b - a, gi) for a, b in zip(cuts[:-1], cuts[1:])]
        opt.step()
        after = (opt.flat_p.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone(), opt.state.clone())
        with torch.no_grad():
            opt.flat_p.copy_(before[0]); opt.exp_avg.copy_(before[1]); opt.exp_avg_sq.copy_(before[2]); opt.state.copy_(before[3])
        _step_ranges(opt, pieces)
        for a, b, nm in zip(after, (opt.flat_p, opt.exp_avg, opt.exp_avg_sq, opt.state), ('p', 'm', 'v', 'state')):
            assert torch.equal(a, b), f'step {s}: {nm} depends on how the active elements are cut into ranges'
        for nm, a, b in zip(('p', 'm', 'v'), after[:3], before[:3]):
            assert torch.equal(a[frozen], b[frozen]), f'step {s}: frozen {nm} changed'
        assert torch.equal(after[3][4:8], before[3][4:8]), f'step {s}: frozen group counter changed'
        for gi, t0 in ((0, 3), (2, 7)):
            m = _group_mask(opt, gi, device)
            assert_adam_step(tuple(x[m] for x in before[:3]), tuple(x[m] for x in after[:3]) + (after[3][4 * gi:4 * gi + 4],),
                             g[m], t0 + s, opt.lr, opt.betas, opt.eps, 1.0, f'group {gi} step {t0 + s}')
    assert opt.group_steps() == [3 + steps, 0, 7 + steps]


# ---- FlatAdam against torch.optim.Adam over training phases -----------------------------------------------------------
def _nets(device):
    torch.manual_seed(0)
    A = torch.nn.Sequential(cnn.Conv2d(3, 6, 3, padding=1, act='relu'), cnn.Conv2d(6, 4, 3, padding=1, act='relu')).to(device)
    B = torch.nn.Sequential(cnn.Conv2d(4, 5, 3, padding=1, act='relu'), cnn.Conv2d(5, 2, 3, padding=1)).to(device)
    return A, B


def _torch_twins(A, B, device):
    def twin(net):
        t = torch.nn.Sequential(*[torch.nn.Conv2d(c.in_channels, c.out_channels, c.kernel_size, padding=c.padding)
                                  for c in net]).to(device)
        for a, b in zip(net, t):
            b.load_state_dict(a.state_dict())
        return t
    return twin(A), twin(B)


def _torch_fwd(tA, tB, x):
    return tB[1](torch.relu(tB[0](torch.relu(tA[1](torch.relu(tA[0](x)))))))


PHASES = [((), 3), ((1,), 2), ((0,), 2)]       # train A+B, fix B, then fix A and train B


def case_flat_adam_phases(device):
    """Train A+B for 3 steps, fix B for 2, then fix A and train B for 2: FlatAdam with one group per net (freeze() +
    requires_grad) against torch.optim.Adam (requires_grad toggled, zero_grad(set_to_none=True)).  Parameters match;
    state_dict() has torch's state indices and exactly torch's per-parameter step counts after every step; torch's state
    dict loads back with per-group counters and the loaded optimiser continues to match; a relayout in the middle
    changes no bit."""
    A, B = _nets(device)
    tA, tB = _torch_twins(A, B, device)
    A2, B2 = _nets(device)                       # the same nets again, re-packed in reverse order after step 4
    nets = [(A, B), (A2, B2)]
    opts = [FlatAdam(list(a.parameters()) + list(b.parameters()), lr=1e-2, groups=[list(a.parameters()), list(b.parameters())])
            for a, b in nets]
    tparams = list(tA.parameters()) + list(tB.parameters())
    topt = torch.optim.Adam(tparams, lr=1e-2)
    gen = torch.Generator().manual_seed(1)
    loaded = None
    step = 0
    for fixed, nsteps in PHASES:
        for o, (a, b) in zip(opts, nets):
            for gi, net in enumerate((a, b)):
                net.requires_grad_(gi not in fixed)
            o.freeze(fixed)
        for gi, net in enumerate((tA, tB)):
            net.requires_grad_(gi not in fixed)
        for _ in range(nsteps):
            x = torch.randn(2, 3, 7, 9, generator=gen).to(device)
            for o, (a, b) in zip(opts, nets):
                o.zero_grad()
                (b(a(x)) ** 2).mean().backward()
                o.step()
            topt.zero_grad(set_to_none=True)
            (_torch_fwd(tA, tB, x) ** 2).mean().backward()
            topt.step()
            if loaded is not None:
                la, lb, lo = loaded
                lo.zero_grad()
                (lb(la(x)) ** 2).mean().backward()
                lo.step()
            step += 1
            if step == 4:
                opts[1].relayout(list(reversed(opts[1].params)))
            for p, q in zip(list(A.parameters()) + list(B.parameters()), list(A2.parameters()) + list(B2.parameters())):
                assert torch.equal(p, q), f'step {step}: a relayout changed the result'
            for p, q in zip(list(A.parameters()) + list(B.parameters()), tparams):
                assert_close(p, q, 2e-4, f'step {step}: parameter vs torch.optim.Adam')
            sd, tsd = opts[0].state_dict(), topt.state_dict()
            assert sorted(sd['state']) == sorted(tsd['state']), (step, sorted(sd['state']), sorted(tsd['state']))
            for i in tsd['state']:
                assert float(sd['state'][i]['step']) == float(tsd['state'][i]['step']), (step, i)
                assert_close(sd['state'][i]['exp_avg'], tsd['state'][i]['exp_avg'], 2e-4, f'step {step}: exp_avg[{i}]')
            if loaded is not None:
                for p, q in zip(list(loaded[0].parameters()) + list(loaded[1].parameters()), tparams):
                    assert_close(p, q, 2e-4, f'step {step}: loaded optimiser vs torch.optim.Adam')
            if step == 3 + 2:                    # torch's checkpoint after the second phase: A at step 5, B at 3
                la, lb = _nets(device)
                with torch.no_grad():
                    for p, q in zip(list(la.parameters()) + list(lb.parameters()), tparams):
                        p.copy_(q)
                lo = FlatAdam(list(la.parameters()) + list(lb.parameters()), lr=5e-3,
                              groups=[list(la.parameters()), list(lb.parameters())])
                lo.load_state_dict(tsd)
                assert lo.group_steps() == [5, 3] and lo.lr == 1e-2, lo.group_steps()
                loaded = (la, lb, lo)
                for gi, net in enumerate((la, lb)):
                    net.requires_grad_(gi != 0)
                lo.freeze([0])
    assert opts[0].group_steps() == [5, 5]


def case_load_missing_group_state(device):
    """A torch checkpoint in which one net never trained (no state entries) loads as counter 0 for that group, and the
    first step of that group uses t = 1."""
    A, B = _nets(device)
    tA, tB = _torch_twins(A, B, device)
    tB.requires_grad_(False)
    topt = torch.optim.Adam(list(tA.parameters()) + list(tB.parameters()), lr=1e-2)
    gen = torch.Generator().manual_seed(2)
    for _ in range(2):
        topt.zero_grad(set_to_none=True)
        (_torch_fwd(tA, tB, torch.randn(2, 3, 7, 9, generator=gen).to(device)) ** 2).mean().backward()
        topt.step()
    opt = FlatAdam(list(A.parameters()) + list(B.parameters()), lr=1e-2, groups=[list(A.parameters()), list(B.parameters())])
    opt.load_state_dict(topt.state_dict())
    assert opt.group_steps() == [2, 0], opt.group_steps()
    sd = opt.state_dict()
    assert sorted(sd['state']) == sorted(topt.state_dict()['state'])
    opt.zero_grad()
    (B(A(torch.randn(2, 3, 7, 9, generator=gen).to(device))) ** 2).mean().backward()
    before = (opt.flat_p.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone())
    g = opt.flat_g.clone()
    opt.step()
    for gi, t in ((0, 3), (1, 1)):
        m = _group_mask(opt, gi, device)
        assert_adam_step(tuple(x[m] for x in before), (opt.flat_p[m], opt.exp_avg[m], opt.exp_avg_sq[m],
                                                       opt.state[4 * gi:4 * gi + 4]), g[m], t, opt.lr, opt.betas, opt.eps,
                         1.0, f'group {gi} after loading')


# ---- photometric loss: value-only and mask-gradient-free paths -------------------------------------------------------
def _photo(s, mode, wssim, NL, grad, mask_grad):
    """(loss, grads of the non-mask inputs, grads of the masks or None) of one photometric call."""
    em = [m.detach().clone().requires_grad_(mask_grad) for m in s['emask'][:NL]]
    if mode == 'rigid':
        inputs = KC.leafs(s['depth'][:NL]) + [s['pose'].detach().clone().requires_grad_(True)]
        masks = em
        call = lambda: CL.photometric_reconstruction_loss(s['tgt'], s['refs'], s['K'], s['Kinv'], inputs[:NL], masks,
                                                          inputs[NL], wssim=wssim)
    else:
        inputs = KC.leafs(s['flow_fwd'][:NL]) + KC.leafs(s['flow_bwd'][:NL])
        masks = [(1 - m[:, 1:3]) for m in em]
        call = lambda: CL.photometric_flow_loss(s['tgt'], s['refs'][1:3], [inputs[NL:], inputs[:NL]], masks, wssim=wssim)
    if not grad:
        with torch.no_grad():
            return call().detach().clone(), None, None
    l = call()
    want = inputs + (em if mask_grad else [])
    gr = torch.autograd.grad(l, want)
    return l.detach().clone(), gr[:len(inputs)], (gr[len(inputs):] if mask_grad else None)


def case_photo_value_only(device, B=2, H=40, W=72, NL=3, seed=31):
    """Value-only forward (grad mode off, and no input needing a gradient) gives the full forward's loss bit for bit, in
    rigid and flow modes with wssim 0.997 and 0; with a mask that needs no gradient the loss and the depth / pose / flow
    gradients equal the full backward's bit for bit."""
    s = KC.dev_sample(B, H, W, seed, NL, device)
    for mode, wssim in itertools.product(('rigid', 'flow'), (0.997, 0.0)):
        pyramid.clear()
        lf, gf, gm = _photo(s, mode, wssim, NL, True, True)
        assert gm is not None and all(bool(torch.isfinite(t).all()) for t in gm)
        lv, _, _ = _photo(s, mode, wssim, NL, False, False)
        assert torch.equal(lv, lf), f'{mode} wssim={wssim}: value-only loss {lv.item()!r} vs full {lf.item()!r}'
        # grad mode on but nothing requires a gradient: also value-only
        em = [m.detach() for m in s['emask'][:NL]]
        if mode == 'rigid':
            l2 = CL.photometric_reconstruction_loss(s['tgt'], s['refs'], s['K'], s['Kinv'], [d.detach() for d in s['depth'][:NL]],
                                                    em, s['pose'].detach(), wssim=wssim)
        else:
            l2 = CL.photometric_flow_loss(s['tgt'], s['refs'][1:3], [[f.detach() for f in s['flow_bwd'][:NL]],
                                                                     [f.detach() for f in s['flow_fwd'][:NL]]],
                                          [1 - m[:, 1:3] for m in em], wssim=wssim)
        assert not l2.requires_grad and torch.equal(l2.detach(), lf), f'{mode} wssim={wssim}: no-grad inputs'
        ln, gn, gmn = _photo(s, mode, wssim, NL, True, False)
        assert gmn is None
        assert torch.equal(ln, lf), f'{mode} wssim={wssim}: loss without the mask gradient'
        for i, (a, b) in enumerate(zip(gn, gf)):
            assert torch.equal(a, b), f'{mode} wssim={wssim}: gradient {i} differs without the mask gradient'
    pyramid.clear()


# ---- the Trainer with fixed nets (GPU) --------------------------------------------------------------------------------
def _oracle_params(P, names):
    """The oracle's parameters of `names` in chain order (BatchNorm buffers excluded)."""
    return [t for n in names for k, t in P[n].items() if t.is_floating_point() and 'running_' not in k]


def case_canonical_vs_oracle(device, B=2, H=64, W=128, steps=3):
    """Trainer('cfg3', fixed=('mask', 'flow')) - the README's command - against oracle.step.loss_cfg3 on the CPU with
    torch.optim.Adam over all four nets' oracle parameters, mask and flow requires_grad=False: losses of steps 0-2
    within 1e-3; per step, mask / flow bit-unchanged with zero gradient ranges and disp / pose within the fp64 Adam bound
    of the step's own gradient.  The eager step issues fewer launches than the cfg3 step."""
    from oracle import step as OS
    P = OS.make_params('cfg3')
    sd = oracle_state_dicts(P)
    for n in ('mask', 'flow'):
        for t in P[n].values():
            t.requires_grad_(False)
    topt = torch.optim.Adam(_oracle_params(P, ('disp', 'pose', 'mask', 'flow')), lr=OS.HP['lr'],
                            betas=(OS.HP['beta1'], OS.HP['beta2']))
    tr = Trainer('cfg3', device, state_dicts=sd, fixed=('mask', 'flow'))
    launches = []
    for s in range(steps):
        tgt, refs = synth.frames(B, H, W, seed=90 + s)
        K, Kinv = synth.intrinsics(B, H, W)
        before = _record(tr)
        c0 = _lib.lib().ccb_launch_count()
        lc, _ = tr.step(tgt.to(device), [r.to(device) for r in refs], K.to(device), Kinv.to(device))
        torch.cuda.synchronize()
        launches.append(_lib.lib().ccb_launch_count() - c0)
        after = _record(tr, lc)
        assert_groups_step(tr, before, after, dict(disp=s + 1, pose=s + 1), f'canonical step {s}')
        topt.zero_grad(set_to_none=True)
        lo, _ = OS.loss_cfg3(P, tgt, refs, K, Kinv)
        lo.backward()
        topt.step()
        assert_close(lc, lo, 1e-3, f'canonical loss step {s}')
    assert tr.opt.group_steps() == [steps, steps, 0, 0]
    del tr
    full = Trainer('cfg3', device, state_dicts=sd)
    tgt, refs = synth.frames(B, H, W, seed=90)
    K, Kinv = synth.intrinsics(B, H, W)
    c0 = _lib.lib().ccb_launch_count()
    full.step(tgt.to(device), [r.to(device) for r in refs], K.to(device), Kinv.to(device))
    torch.cuda.synchronize()
    n_full = _lib.lib().ccb_launch_count() - c0
    assert launches[-1] < n_full, (launches, n_full)
    print(f'canonical step: {launches[-1]} launches, cfg3 step: {n_full}')


def case_phase_switch(device, B=2, H=64, W=128):
    """2 steps with nothing fixed, 3 with ('mask', 'flow'), 1 with ('disp', 'pose'): counters disp/pose 5, mask/flow 3,
    every step's active ranges within the Adam bound of their own t and the fixed ones bit-unchanged.  A fresh Trainer
    loads a torch-made state dict with disp/pose at step 5 and no mask/flow state; its first step with the mask trained
    uses t = 1 for the mask.  Trainer.opt.state_dict() loads into torch.optim.Adam over chain(nets)."""
    tr = Trainer('cfg3', device, seed=0)
    t = dict(disp=0, pose=0, mask=0, flow=0)
    s = 0
    for fixed, n in (((), 2), (('mask', 'flow'), 3), (('disp', 'pose'), 1)):
        tr.set_fixed(fixed)
        for _ in range(n):
            tgt, refs = synth.frames(B, H, W, seed=200 + s)
            K, Kinv = synth.intrinsics(B, H, W)
            before = _record(tr)
            tr.step(tgt.to(device), [r.to(device) for r in refs], K.to(device), Kinv.to(device))
            for k in t:
                t[k] += k not in fixed
            assert_groups_step(tr, before, _record(tr), t, f'phase step {s} fixed={fixed}')
            s += 1
    assert tr.opt.group_steps() == [5, 5, 3, 3], tr.opt.group_steps()
    sd = tr.opt.state_dict()
    params = [p for n in NETS_OF['cfg3'] for p in tr.nets[n].parameters()]
    tref = torch.optim.Adam([torch.nn.Parameter(p.detach().clone()) for p in params], lr=1e-4)
    tref.load_state_dict(sd)                                        # our checkpoint loads into torch
    # a torch-made checkpoint with disp/pose at step 5 and no mask/flow state
    n_dp = sum(1 for n in ('disp', 'pose') for _ in tr.nets[n].parameters())
    tsd = tref.state_dict()
    tsd['state'] = {i: v for i, v in tsd['state'].items() if i < n_dp}
    tref2 = torch.optim.Adam([torch.nn.Parameter(p.detach().clone()) for p in params], lr=1e-4)
    tref2.load_state_dict(tsd)
    torch_sd = tref2.state_dict()
    del tr
    fresh = Trainer('cfg3', device, seed=0, fixed=('flow',))
    fresh.opt.load_state_dict(torch_sd)
    assert fresh.opt.group_steps() == [5, 5, 0, 0], fresh.opt.group_steps()
    tgt, refs = synth.frames(B, H, W, seed=300)
    K, Kinv = synth.intrinsics(B, H, W)
    before = _record(fresh)
    fresh.step(tgt.to(device), [r.to(device) for r in refs], K.to(device), Kinv.to(device))
    assert_groups_step(fresh, before, _record(fresh), dict(disp=6, pose=6, mask=1), 'first step after loading')
    assert fresh.opt.group_steps() == [6, 6, 1, 0]


def case_fixed_dispnet_batchnorm(device, B=2, H=128, W=416, steps=2):
    """cfg1 with the DispResNet6 fixed: it stays in train mode, so its BatchNorm running statistics follow the oracle's
    (reference train.py:438-441), while its parameters do not move."""
    from oracle import step as OS
    P = OS.make_params('cfg1')
    sd = oracle_state_dicts(P)
    for t in P['disp'].values():
        t.requires_grad_(False)
    topt = torch.optim.Adam(_oracle_params(P, ('disp', 'pose')), lr=OS.HP['lr'], betas=(OS.HP['beta1'], OS.HP['beta2']))
    tr = Trainer('cfg1', device, state_dicts=sd, fixed=('disp',))
    p0 = tr.opt.flat_p.clone()
    lo, hi = group_range(tr.opt, 0)
    for s in range(steps):
        tgt, refs = synth.frames(B, H, W, seed=50 + s)
        K, Kinv = synth.intrinsics(B, H, W)
        tr.step(tgt.to(device), [r.to(device) for r in refs], K.to(device), Kinv.to(device))
        topt.zero_grad(set_to_none=True)
        lo_, _ = OS.loss_cfg1(P, tgt, refs, K, Kinv)
        lo_.backward()
        topt.step()
    assert torch.equal(tr.opt.flat_p[lo:hi], p0[lo:hi]), 'the fixed DispResNet6 moved'
    n = 0
    for k, b in tr.nets['disp'].named_buffers():
        if 'running_' in k:
            assert_close(b, P['disp'][k], 1e-3, f'fixed disp BatchNorm {k}')
            n += 1
    assert n > 0
