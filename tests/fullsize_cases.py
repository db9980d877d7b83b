"""Step-level parity of the PRODUCTION path (Trainer.step on IMPL_AUTO = the wgmma tensor-core kernels) at the
BASELINE.json configurations: b4, 256x832, 6 pyramid levels, cfg1 / cfg2 / cfg3.

For every configuration the CUDA step is compared with the CPU oracle (oracle/step.py = reference
train.py:454-509 restated) on identical seeded inputs and weights:

  * total loss and every loss term, every network output (disparities, pose, masks, flows): bar 1e-4
  * the gradient of EVERY parameter of every net: bar 1e-3 (deep-net gradients, VERDICT r1 item 1)

Errors are max-abs relative to the tensor's max-abs (tests/util.rel_err).  Beside every number the report
carries the *noise floor*: the same oracle code run in fp32 on the GPU (ATen kernels, TF32 off) against
the same oracle on the CPU - two correct fp32 evaluations of the reference that differ only in summation
order.  A tensor may exceed its bar only if it stays within FLOOR_FACTOR x its own measured floor.

DispResNet6 is the exception: its gradient is chaotic - 13 BatchNorms, the deepest over
56 values, and ReLU masks on 2x7 .. 8x26 maps amplify a 1e-7 forward difference ~1e4 times, so the two torch
evaluations already disagree by 7e-4 (median) .. 1e-1 (worst tensor).  The amplification is linear in the
per-op error: the production wgmma tensor-core kernels sit at 4.4 x the floor (median; cfg1 4.44, cfg3 4.43 on an H100 SXM
at a 400 W power limit).  The step is bit-reproducible on a given GPU and build (fixed-order reductions, fixed-point warp
scatter), so this ratio does not vary from run to run; it moves only when the kernels' summation order changes, and any
such change is held to the bar here.  For this net the per-tensor rule is replaced by: median(err / floor) <= CHAOS_MEDIAN,
relative L2 error of every tensor <= CHAOS_L2, and the counts are reported.  Values (losses, disparities) keep
the strict 1e-4 bar.

Per-layer correctness at this size, DispResNet6's layers included, is established by the layer audit (audit_step below,
tests/layer_audit.py): every convolution, BatchNorm, upsample, cost-volume and feature-warp call of the timed cfg3 step is
checked against fp64 element by element, on its real inputs, within a derived per-element bound.  A per-op error of a
few per cent confined to one layer, which the chaos bar could not see, fails there.  The chaos bar stays as the
end-to-end check of the step against the oracle.

The per-tensor table is summarised on stdout and, when $CCB_PARITY_REPORT_DIR is set, written there as
parity_fullsize_<cfg>.json."""
import json
import os
import time
import torch
from tests.util import rel_err
from cc_b200 import synth, nn as cnn
from cc_b200.train_step import Trainer
from oracle import step as OS

OUT_TOL, LOSS_TOL, GRAD_TOL = 1e-4, 1e-4, 1e-3
FLOOR_FACTOR = 3.0
GRAD_TOL_HARD = 3e-3               # no gradient tensor of Pose / Mask / Flow may exceed this, whatever its floor says (H100: max 7.8e-4)
BETWEEN_FRAC = 0.05                # share of a net's tensors allowed between the bar and the cap (H100: none)
CHAOTIC_NETS = ('disp',)           # see the module docstring
CHAOS_MEDIAN, CHAOS_L2 = 5.0, 5e-2
# Pose / Mask / Flow gradients: bar 1e-3 (or 3 x floor); at most 5 % of a net's tensors may sit between the bar and the hard
# cap.  Measured at b4 256x832 on an H100 SXM (400 W power limit), cfg3: every Pose / Mask / Flow tensor under the bar (max
# 1.6e-5 / 2.7e-4 / 7.8e-4); the cap and the 5 % leave room for other GPUs and compilers, whose summation orders differ


def _flatten_aux(aux):
    out = {}
    for k, v in aux.items():
        if isinstance(v, (list, tuple)):
            for i, t in enumerate(v):
                out['%s[%d]' % (k, i)] = t
        elif torch.is_tensor(v):
            out[k] = v
    return out


def _oracle(cfg, P, tgt, refs, K, Kinv):
    for n in P:
        for t in P[n].values():
            t.grad = None
    loss, aux = OS.LOSS_FNS[cfg](P, tgt, refs, K, Kinv)
    loss.backward()
    vals = {'loss': loss.detach()}
    vals.update({k: v.detach() for k, v in _flatten_aux(aux).items()})
    grads = {}
    for n in P:
        for k, t in P[n].items():
            if t.requires_grad and t.grad is not None:
                grads['%s.%s' % (n, k)] = t.grad.detach()
    return vals, grads


def _params_to(P, device):
    return {n: {k: v.detach().to(device).requires_grad_(v.requires_grad) for k, v in d.items()} for n, d in P.items()}


def run(cfg, device, B=4, H=256, W=832, seed=50, with_floor=True, threads=None, report=True):
    """Returns the report dict; raises AssertionError when a tensor misses its bar."""
    if threads:
        torch.set_num_threads(threads)
    tgt, refs = synth.frames(B, H, W, seed=seed)
    K, Kinv = synth.intrinsics(B, H, W)
    P = OS.make_params(cfg)
    t0 = time.perf_counter()
    ovals, ograds = _oracle(cfg, P, tgt, refs, K, Kinv)
    t_cpu = time.perf_counter() - t0
    sd = {n: {k: v.detach().clone() for k, v in d.items()} for n, d in P.items()}

    tr = Trainer(cfg, device, state_dicts=sd)
    dt, dr, dK, dKi = tgt.to(device), [r.to(device) for r in refs], K.to(device), Kinv.to(device)
    loss, aux = tr.step(dt, dr, dK, dKi)
    cvals = {'loss': loss}
    cvals.update(_flatten_aux(aux))
    cgrads = {}
    for n in tr.nets:
        for k, p in tr.nets[n].named_parameters():
            if getattr(p, '_ccb_grad', None) is not None:
                cgrads['%s.%s' % (n, k)] = p._ccb_grad

    fvals, fgrads = {}, {}
    if with_floor and device.type == 'cuda':
        Pd = _params_to(P, device)
        fvals, fgrads = _oracle(cfg, Pd, dt, dr, dK, dKi)

    rows, bad = [], []
    for kind, oracle_d, ours_d, floor_d, tol in (('value', ovals, cvals, fvals, None), ('grad', ograds, cgrads, fgrads, GRAD_TOL)):
        for name, ref in oracle_d.items():
            if name not in ours_d:
                # a parameter the oracle trained and the product did not is a failure (occ decoders get no grad in either)
                if kind == 'grad' and ref.abs().max().item() > 0:
                    bad.append('%s: no gradient on the CUDA path' % name)
                continue
            bar = tol if tol is not None else (LOSS_TOL if ref.dim() == 0 else OUT_TOL)
            e = rel_err(ours_d[name], ref)
            fl = rel_err(floor_d[name], ref) if name in floor_d else None
            ok = e <= bar or (fl is not None and e <= FLOOR_FACTOR * fl)
            row = dict(kind=kind, name=name, numel=int(ref.numel()), err=e, floor=fl, bar=bar, ok=bool(ok))
            chaotic = kind == 'grad' and name.split('.')[0] in CHAOTIC_NETS and fl is not None
            if kind == 'grad':
                row['l2'] = float((ours_d[name].double().cpu() - ref.double().cpu()).norm() / ref.double().norm().clamp_min(1e-30))
            if chaotic:
                row['chaotic'] = True
                if row['l2'] > CHAOS_L2:
                    bad.append('grad %s: relative L2 error %.3e > %.1e (max-abs %.3e, floor %.3e)' % (name, row['l2'], CHAOS_L2, e, fl))
            elif kind == 'grad' and e > GRAD_TOL_HARD and not ok:
                bad.append('grad %s: rel err %.3e > hard cap %.1e (floor %s)' % (name, e, GRAD_TOL_HARD, 'n/a' if fl is None else '%.3e' % fl))
            elif kind == 'grad' and not ok:
                row['between_bar_and_cap'] = True           # counted below: a few per net at most
            elif not ok:
                bad.append('%s %s: rel err %.3e > %.1e (oracle GPU-vs-CPU floor %s)' % (kind, name, e, bar, 'n/a' if fl is None else '%.3e' % fl))
            rows.append(row)
    import statistics
    for net in sorted({r['name'].split('.')[0] for r in rows if r['kind'] == 'grad'}):
        n = sum(r['kind'] == 'grad' and r['name'].startswith(net + '.') for r in rows)
        k = sum(bool(r.get('between_bar_and_cap')) and r['name'].startswith(net + '.') for r in rows)
        if k > max(1, int(BETWEEN_FRAC * n)):
            bad.append('%s gradients: %d of %d tensors between the %.0e bar and the %.0e cap (allowed %.0f %%)' % (net, k, n, GRAD_TOL, GRAD_TOL_HARD, 100 * BETWEEN_FRAC))
    for net in CHAOTIC_NETS:
        ratios = [r['err'] / max(r['floor'], 1e-9) for r in rows if r.get('chaotic') and r['name'].startswith(net + '.')]
        if ratios and statistics.median(ratios) > CHAOS_MEDIAN:
            bad.append('%s gradients: median err / floor = %.2f > %.1f' % (net, statistics.median(ratios), CHAOS_MEDIAN))
    # 0/1 consensus targets are not in aux; masks are checked bit-exactly by the kernel-level full-size tests.
    rep = dict(cfg=cfg, B=B, H=H, W=W, seed=seed, device=str(device), oracle_cpu_s=t_cpu,
               bars=dict(loss=LOSS_TOL, outputs=OUT_TOL, grads=GRAD_TOL, floor_factor=FLOOR_FACTOR),
               n_values=sum(r['kind'] == 'value' for r in rows), n_grads=sum(r['kind'] == 'grad' for r in rows),
               max_value_err=max([r['err'] for r in rows if r['kind'] == 'value'] or [0.0]),
               max_grad_err=max([r['err'] for r in rows if r['kind'] == 'grad'] or [0.0]),
               max_value_floor=max([r['floor'] or 0.0 for r in rows if r['kind'] == 'value'] or [0.0]),
               max_grad_floor=max([r['floor'] or 0.0 for r in rows if r['kind'] == 'grad'] or [0.0]),
               n_over_bar=sum((r['err'] > r['bar']) for r in rows), n_fail=len(bad), rows=rows)
    per_net = {}
    for r in rows:
        if r['kind'] == 'grad':
            per_net.setdefault(r['name'].split('.')[0], []).append(r)
    rep['per_net'] = {}
    for net, rs in per_net.items():
        errs = sorted(r['err'] for r in rs)
        ratio = sorted(r['err'] / max(r['floor'] or 0.0, 1e-9) for r in rs)
        rep['per_net'][net] = dict(n=len(rs), err_median=errs[len(rs) // 2], err_max=errs[-1], over_1e3=sum(e > GRAD_TOL for e in errs),
                                   ratio_median=ratio[len(rs) // 2], ratio_p90=ratio[int(0.9 * len(rs))], l2_max=max(r['l2'] for r in rs))
    if report:
        summarise(rep)
        out = os.environ.get('CCB_PARITY_REPORT_DIR')
        if out:
            os.makedirs(out, exist_ok=True)
            tag = cfg if (B, H, W) == (4, 256, 832) else '%s_b%d_%dx%d' % (cfg, B, H, W)
            with open(os.path.join(out, 'parity_fullsize_%s.json' % tag), 'w') as f:
                json.dump(rep, f, indent=1)
    assert not bad, '%d tensors miss the parity bar:\n  ' % len(bad) + '\n  '.join(bad[:40])
    return rep


def summarise(rep):
    print('\n== parity %s b%d %dx%d on %s: %d values (max err %.2e, floor %.2e), %d parameter gradients (max err %.2e, floor %.2e); '
          '%d over bar, %d fail' % (rep['cfg'], rep['B'], rep['H'], rep['W'], rep['device'], rep['n_values'], rep['max_value_err'],
                                    rep['max_value_floor'], rep['n_grads'], rep['max_grad_err'], rep['max_grad_floor'],
                                    rep['n_over_bar'], rep['n_fail']))
    for net, d in rep.get('per_net', {}).items():
        print('   grads %-5s n=%3d  err median %.1e max %.1e  (> 1e-3: %d)   err/floor median %.1f p90 %.1f   rel-L2 max %.1e' % (
            net, d['n'], d['err_median'], d['err_max'], d['over_1e3'], d['ratio_median'], d['ratio_p90'], d['l2_max']))
    worst = sorted(rep['rows'], key=lambda r: -r['err'] / r['bar'])[:12]
    for r in worst:
        print('   %-5s %-44s err %.2e  floor %s  bar %.0e %s' % (r['kind'], r['name'], r['err'],
                                                                 'n/a     ' if r['floor'] is None else '%.2e' % r['floor'], r['bar'],
                                                                 '' if r['ok'] else 'FAIL'))


def _second_step(device, cfg, B, H, W, seed, flownet):
    """Trainer(cfg, flownet=flownet) from the oracle's weights (FlowNetC6: flownetc6_cases.step_flow_params, which keep
    its flows finite), one eager step (it records the weight-cache layouts, which then commit), then an unaudited second
    step from a snapshot that is restored.  -> (trainer, step arguments, loss and flat gradient of the second step)."""
    from tests import flownetc6_cases as FC6
    tgt, refs = synth.frames(B, H, W, seed=seed)
    K, Kinv = synth.intrinsics(B, H, W)
    P = OS.make_params(cfg)
    if flownet == 'FlowNetC6':
        P['flow'] = FC6.step_flow_params()
    sd = {n: {k: v.detach().clone() for k, v in d.items()} for n, d in P.items()}
    tr = Trainer(cfg, device, state_dicts=sd, flownet=flownet)
    args = (tgt.to(device), [r.to(device) for r in refs], K.to(device), Kinv.to(device))
    tr.step(*args)
    assert tr.wcache is not None and tr.wcache.committed
    snap = tr._snapshot()
    loss_ref = tr.step(*args)[0].clone()
    grad_ref = tr.opt.flat_g.clone()
    tr._restore(snap)
    torch.cuda.synchronize(device)
    return tr, args, loss_ref, grad_ref


def _audited_step(device, tr, args, loss_ref, grad_ref, audit):
    """The second step under `audit`, timed; its loss and flat gradient must equal the unaudited ones bit for bit."""
    t0 = time.perf_counter()
    with audit:
        loss = tr.step(*args)[0]
    torch.cuda.synchronize(device)
    print('   audited step: %.1f s (fp64 references included)' % (time.perf_counter() - t0))
    assert torch.equal(loss, loss_ref), (loss.item(), loss_ref.item())
    assert torch.equal(tr.opt.flat_g, grad_ref), 'the audit changed the flat gradient by %.3e' % (tr.opt.flat_g - grad_ref).abs().max().item()
    st = tr.wcache.stats()
    assert st['misses'] == 0 and st['hits'] > 0, st


def _tc_only(row):
    return bool(row.get('plans')) and all(p['path'] != 'ffma' for p in row['plans'])


def audit_step(device, cfg='cfg3', B=4, H=256, W=832, seed=50, flownet='Back2Future'):
    """The layer audit (tests/layer_audit.py) of the step the benchmark times, with either flow net: Trainer(cfg) from the
    oracle's weights, one eager step, then the SECOND eager step - committed cache, production IMPL_AUTO dispatch - with
    every layer call checked against fp64 element by element.
      * completeness: every Conv2d / ConvTranspose2d / BatchNorm2d module of the nets is audited forward and backward
        (Back2Future's occlusion decoders do not run in training, see build_nets); Back2Future's ten cost volumes and
        eight feature warps, or FlowNetC6's two dilated cost volumes (one per flow-net call) and nothing else;
      * non-interference: the audited step's loss and flat gradient equal, bit for bit, an unaudited second step from
        the same snapshot;
      * coverage, Back2Future: the coarsest cost volume (C = 192 on a 4x13 map: one tile per sample) runs corr_chunks =
        32 channel chunks, and the BatchNorm of DispResNet6's iconv1 shortcut reduces its 851968 values per channel in
        104 splits.  FlowNetC6: conv3_1 (473 input channels, a ragged last 4-channel chunk) and deconv4 (its data
        gradient an fprop with N = 1026 = 8 x 128 + 2) run the tensor-core kernels in both phases, a call with 1026
        channels is audited, and the plans include split-K tensor-core fprop / dgrad calls and weight gradients through
        padded rows.
    Measured on an H100 80GB HBM3 (700 W power limit), cfg3 b4 256x832: worst r per family in layer_audit.R_MEASURED;
    the audited step takes 2.0 s with Back2Future and 2.2-3.8 s with FlowNetC6 (wall time, fp64 references included).
    Returns the audit summary."""
    from tests import layer_audit as LA
    tr, args, loss_ref, grad_ref = _second_step(device, cfg, B, H, W, seed, flownet)
    audit = LA.LayerAudit(nets=tr.nets, tag='%s_b%d_%dx%d%s' % (cfg, B, H, W, '' if flownet == 'Back2Future' else '_' + flownet))
    _audited_step(device, tr, args, loss_ref, grad_ref, audit)

    rows = audit.rows
    want = {'%s.%s' % (n, k) for n, net in tr.nets.items() for k, m in net.named_modules()
            if isinstance(m, (cnn.Conv2d, cnn.ConvTranspose2d, cnn.BatchNorm2d)) and not k.startswith('decoder_occ')}
    for phase in ('fwd', 'bwd'):
        got = {r['name'] for r in rows if r['phase'] == phase and r['op'] in ('conv', 'convT', 'bn')}
        assert got == want, (phase, sorted(want - got)[:10], sorted(got - want)[:10])
    calls = dict(corr81=10, featwarp=8, corr441d=0) if flownet == 'Back2Future' else dict(corr81=0, featwarp=0, corr441d=2)
    for op, n in calls.items():
        for phase in ('fwd', 'bwd'):
            k = sum(r['op'] == op and r['phase'] == phase and r['name'].startswith('flow') for r in rows)
            assert k == n, (op, phase, k)
    assert not any(r['op'] == 'bn_eval' for r in rows)
    if flownet == 'Back2Future':
        h6, w6 = H // 64, W // 64
        assert LA.corr_chunks(B, 192, h6, w6) == 32
        assert {r['phase'] for r in rows if r['op'] == 'corr81' and r['shape'] == [B, 192, h6, w6] and r['chunks'] == 32} == {'fwd', 'bwd'}
    else:
        for name in ('flow.conv3_1.0', 'flow.deconv4.0'):            # the Conv2d / ConvTranspose2d of each block
            assert {r['phase'] for r in rows if r['name'] == name and _tc_only(r)} == {'fwd', 'bwd'}, \
                [(r['phase'], r['plans']) for r in rows if r['name'] == name]
        assert any(r['op'] in ('conv', 'convT') and 1026 in r['shape'][:2] for r in rows)
        plans = [p for r in rows for p in r.get('plans', ())]
        assert any(p['path'] == 'tc' and p['call'] != 'wgrad' and p['splits'] > 1 for p in plans)
        assert any(p['path'] == 'tc_padded' for p in plans)
    assert LA.bn_splits(B, H * W) == 104
    assert {r['phase'] for r in rows if r['op'] == 'bn' and r['name'] == 'disp.iconv1.0.downsample.1' and r['splits'] == 104} == {'fwd', 'bwd'}
    return audit.summary()


def loss_audit_step(device, cfg='cfg3', B=4, H=256, W=832, seed=50, flownet='Back2Future'):
    """The loss audit (tests/loss_audit.py) of the step the benchmark times, with either flow net, set up as audit_step:
    one eager step, then the second step with the weight cache committed, every loss-layer call checked against fp64
    element by element.
      * completeness: one rigid and one flow photometric call (forward and backward), four smoothness and two BCE calls
        (forward and backward), one consensus-target call, twelve pose2flow forwards, whichever the flow net; every
        level has partial tiles;
      * non-interference: the audited step's loss and flat gradient equal, bit for bit, an unaudited second step;
      * detectability: one dropped level-0 tile would put d_pose over its bound (the audit's tile_drop_r).
    Measured on an H100 80GB HBM3 (700 W power limit), cfg3 b4 256x832: worst r per output in loss_audit.R_MEASURED
    (the FlowNetC6 step's are no larger); the audited step takes 4.7-5.1 s with Back2Future and 7.1-7.3 s with FlowNetC6 (wall
    time, fp64 references included).
    Returns the audit summary."""
    from tests import loss_audit as LSA
    tr, args, loss_ref, grad_ref = _second_step(device, cfg, B, H, W, seed, flownet)
    audit = LSA.LossAudit(tag='%s_b%d_%dx%d%s' % (cfg, B, H, W, '' if flownet == 'Back2Future' else '_' + flownet))
    _audited_step(device, tr, args, loss_ref, grad_ref, audit)
    n = {}
    for r in audit.rows:
        n[(r['op'], r['phase'])] = n.get((r['op'], r['phase']), 0) + 1
    want = {('photo_rigid', 'fwd'): 1, ('photo_rigid', 'bwd'): 1, ('photo_flow', 'fwd'): 1, ('photo_flow', 'bwd'): 1,
            ('smooth', 'fwd'): 4, ('smooth', 'bwd'): 4, ('bce', 'fwd'): 2, ('bce', 'bwd'): 2, ('consensus', 'fwd'): 1,
            ('pose2flow', 'fwd'): 12}
    assert {k: v for k, v in n.items() if k[0] != 'pyramid'} == want, n
    assert n.get(('pyramid', 'fwd'), 0) > 0
    for r in audit.rows:
        if r['op'].startswith('photo') and r['phase'] == 'fwd':
            assert len(r['partial_tiles']) == 6 and all(r['partial_tiles']), r['partial_tiles']
    summ = audit.summary()
    # one dropped 64x20 tile of level 0, at the real proportion of a tile to ~2.1e5 pixels per (b, ref), is detected
    assert summ['photo_rigid']['tile_drop_r'] > LSA.R_OUT[('photo_rigid', 'd_pose')], summ['photo_rigid']['tile_drop_r']
    print('   audited calls: %d' % len(audit.rows))
    return summ


def seed_running_stats(nets, seed=31):
    """Every BatchNorm's running statistics set far from their defaults (0, 1): mean ~ N(0, 0.5^2), var ~ U[0.25, 4]; a
    kernel that ignored the mean, dropped eps or scaled by the variance would then miss the eval-mode bound."""
    g = torch.Generator().manual_seed(seed)
    n = 0
    for net in nets.values():
        for m in net.modules():
            if isinstance(m, cnn.BatchNorm2d):
                c = m.num_features
                m.running_mean.copy_(0.5 * torch.randn(c, generator=g))
                m.running_var.copy_(0.25 + 3.75 * torch.rand(c, generator=g))
                n += 1
    return n


# Conv2d / ConvTranspose2d / BatchNorm2d modules evaluate._flow_nets does not run, with the reason.  None: every module of
# the four nets runs in eval mode - DispResNet6 computes every disparity head (each feeds the next level), MaskNet6 is
# built with output_exp=True, and Back2Future(nlevels=6) runs its occlusion decoders outside training.
NOT_RUN_IN_EVAL = {}


def eval_nets(device, flownet='Back2Future'):
    """The four nets as the evaluation scripts load them: the oracle's weights, FlowNetC6 with step_flow_params."""
    from cc_b200 import models as CM
    from oracle import nets as ON
    from tests import flownetc6_cases as FC6
    nets = dict(disp=CM.DispResNet6(), pose=CM.PoseNetB6(nb_ref_imgs=4), mask=CM.MaskNet6(nb_ref_imgs=4, output_exp=True),
                flow=CM.Back2Future(nlevels=6) if flownet == 'Back2Future' else CM.FlowNetC6())
    sds = dict(disp=ON.disp_params(), pose=ON.pose_params(), mask=ON.mask_params(),
               flow=ON.flow_params() if flownet == 'Back2Future' else FC6.step_flow_params())
    for n, net in nets.items():
        net.load_state_dict({k: v.detach().clone() for k, v in sds[n].items()})
    return {n: net.to(device) for n, net in nets.items()}


def audit_eval_forwards(device, flownet='Back2Future', H=256, W=832, seed=75, report=True):
    """The layer audit of evaluate._flow_nets at B = 1 (test_flow.py / test_mask.py / submit_flow.py call the four nets
    so, in eval mode): every BatchNorm's running statistics seeded far from the defaults (seed_running_stats), then
      * non-interference: the audited outputs (mask, camera flow, flow-net flow) equal an unaudited run bit for bit;
      * completeness: every Conv2d / ConvTranspose2d / BatchNorm2d has a forward row (NOT_RUN_IN_EVAL lists the
        exceptions), every BatchNorm an eval-mode one (family bn_eval), and no call has a backward row;
      * the flow net's cost volumes: Back2Future's ten corr81 calls and eight feature warps, FlowNetC6's one corr441d.
    On an H100 80GB HBM3 (700 W power limit) at 256x832 the audited forwards take 0.4-0.6 s with Back2Future and 0.2 s with
    FlowNetC6 (wall time, fp64 references included).
    Returns the audit."""
    from cc_b200 import evaluate as CE
    from tests import layer_audit as LA
    nets = eval_nets(device, flownet)
    nbn = seed_running_stats(nets)
    tgt, refs = synth.frames(1, H, W, seed=seed)
    K, Kinv = synth.intrinsics(1, H, W)
    args = (tgt.to(device), [r.to(device) for r in refs], K.to(device), Kinv.to(device))
    order = ('disp', 'pose', 'mask', 'flow')
    with torch.no_grad():
        ref = [t.clone() for t in CE._flow_nets(*[nets[n] for n in order], *args)]
        audit = LA.LayerAudit(nets=nets, tag='eval_%s_b1_%dx%d' % (flownet, H, W), report=report)
        t0 = time.perf_counter()
        with audit:
            got = CE._flow_nets(*[nets[n] for n in order], *args)
        if device.type == 'cuda':
            torch.cuda.synchronize(device)
    print('   audited eval forwards: %.1f s (fp64 references included)' % (time.perf_counter() - t0))
    for what, a, b in zip(('emask', 'flow_cam', 'flow_fwd'), got, ref):
        assert torch.equal(a, b), '%s: the audit changed the output' % what
    rows = audit.rows
    assert all(r['phase'] == 'fwd' for r in rows)
    want = {'%s.%s' % (n, k) for n, net in nets.items() for k, m in net.named_modules()
            if isinstance(m, (cnn.Conv2d, cnn.ConvTranspose2d, cnn.BatchNorm2d))} - set(NOT_RUN_IN_EVAL)
    got_names = {r['name'] for r in rows if r['op'] in ('conv', 'convT', 'bn_eval')}
    assert got_names == want, (sorted(want - got_names)[:10], sorted(got_names - want)[:10])
    assert not any(r['op'] == 'bn' for r in rows)
    assert nbn > 0 and len({r['name'] for r in rows if r['op'] == 'bn_eval'}) == nbn
    calls = dict(corr81=10, featwarp=8, corr441d=0) if flownet == 'Back2Future' else dict(corr81=0, featwarp=0, corr441d=1)
    for op, n in calls.items():
        assert sum(r['op'] == op for r in rows) == n, (op, sum(r['op'] == op for r in rows))
    return audit


def _golden_rows(g, losses3, grads3, losses1, grads1):
    """rows (name, err, bar) of one implementation against tests/golden/step_small.npz.
    grads*: {net: {param name: grad}}."""
    from tests.util import key_with_stride, pick
    rows = []
    for k in ('loss_1', 'loss_2', 'loss_3', 'loss_4', 'loss_5', 'loss'):
        rows.append((k, rel_err(losses3[k], g[k]), LOSS_TOL))
    for nm in ('disp', 'pose', 'mask', 'flow'):
        gd = grads3[nm]
        gn = torch.sqrt(sum((t.double() ** 2).sum() for t in gd.values()))
        rows.append(('gnorm_' + nm, rel_err(gn, g['gnorm_' + nm]), GRAD_TOL))
        for key in g:
            if key.startswith('g_%s_' % nm):
                pname = key[len('g_%s_' % nm):].split('@')[0]
                _, st = key_with_stride(g, 'g_%s_%s' % (nm, pname))
                rows.append((key, rel_err(pick(gd[pname], st), g[key]), GRAD_TOL))
    rows.append(('cfg1_loss', rel_err(losses1['loss'], g['cfg1_loss']), LOSS_TOL))
    rows.append(('cfg1_l1', rel_err(losses1['loss_1'], g['cfg1_l1']), LOSS_TOL))
    rows.append(('cfg1_l3', rel_err(losses1['loss_3'], g['cfg1_l3']), LOSS_TOL))
    rows.append(('cfg1_g_disp_conv1.0.weight', rel_err(grads1['disp']['conv1.0.weight'], g['cfg1_g_disp_conv1.0.weight']), GRAD_TOL))
    gn = torch.sqrt(sum((t.double() ** 2).sum() for t in grads1['disp'].values()))
    rows.append(('cfg1_gnorm_disp', rel_err(gn, g['cfg1_gnorm_disp']), GRAD_TOL))
    rows.append(('cfg1_g_pose_pose_pred.bias', rel_err(grads1['pose']['pose_pred.bias'], g['cfg1_g_pose_pose_pred.bias']), GRAD_TOL))
    return rows


def golden_step_small(device, with_floor=True):
    """The CUDA step against tests/golden/step_small.npz: the reference's real train() body (train.py:454-509) run on the
    reference's own modules, B=2 64x128 - every loss term, the per-parameter gradients the fixture holds, gradient norms.
    Returns rows (name, err, floor, bar); floor = the oracle evaluated on `device` against the same fixture."""
    from tests.util import golden
    from cc_b200.train_step import loss_cfg3, loss_cfg1, build_nets
    g = golden('step_small')
    B, H, W = 2, 64, 128
    tgt, refs = synth.frames(B, H, W, seed=40)
    K, Kinv = synth.intrinsics(B, H, W)
    dt, dr, dK, dKi = tgt.to(device), [r.to(device) for r in refs], K.to(device), Kinv.to(device)
    P = OS.make_params('cfg3')
    sd = {n: {k: v.detach().clone() for k, v in d.items()} for n, d in P.items()}

    def ours(cfg, fn):
        nets = build_nets(cfg, device, state_dicts={n: sd[n] for n in OS.NETS_OF[cfg]})
        loss, aux = fn(nets, dt, dr, dK, dKi)
        loss.backward()
        losses = {k: v for k, v in aux.items() if k.startswith('loss_')}
        losses['loss'] = loss
        return losses, {n: {k: p.grad for k, p in nets[n].named_parameters() if p.grad is not None} for n in nets}

    def orac(cfg):
        Pd = _params_to({n: P[n] for n in OS.NETS_OF[cfg]}, device)
        loss, aux = OS.LOSS_FNS[cfg](Pd, dt, dr, dK, dKi)
        loss.backward()
        losses = {k: v for k, v in aux.items() if k.startswith('loss_')}
        losses['loss'] = loss
        return losses, {n: {k: t.grad for k, t in Pd[n].items() if t.requires_grad and t.grad is not None} for n in Pd}

    rows = _golden_rows(g, *ours('cfg3', loss_cfg3), *ours('cfg1', loss_cfg1))
    floor = {}
    if with_floor:
        floor = {n: e for n, e, _ in _golden_rows(g, *orac('cfg3'), *orac('cfg1'))}
    return [(n, e, floor.get(n), bar) for n, e, bar in rows]
