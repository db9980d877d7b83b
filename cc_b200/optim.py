"""Fused multi-tensor Adam over ONE flat fp32 buffer (SURVEY.md 2a K13 / O1).

The reference builds a single torch.optim.Adam over chain(all nets' parameters)
(train.py:307-310: lr, betas=(momentum, beta), weight_decay 0) and, under nn.DataParallel,
broadcasts 297 MB of parameters and reduces 297 MB of gradients through GPU0 every step.  Here all
trainable parameters are views into one flat buffer, all gradients views into another; a step is one
`ccb_adam_step_ranges` call, and data-parallel training all-reduces contiguous slices of the flat gradient
buffer (cc_b200/dist.py).

The order of the parameters inside the flat buffers is an internal detail (`relayout()` re-packs them in
gradient-completion order so that the data-parallel buckets are contiguous); checkpoints therefore use
torch.optim.Adam's own per-parameter `state_dict()` format, indexed by the order of the `params` argument
(= the reference's chain(disp, pose, mask, flow) order, train.py:307-310), and load either way.

Step groups (`groups=`, one per network) give each network its own step counter, as torch.optim.Adam's per-parameter
counts do when a network is fixed for a phase of training (train.py --fix-*: requires_grad = False, so Adam skips it).
`freeze()` names the groups the step skips: their parameters, moments and counters are not touched.  The step runs over
the maximal runs of active groups in the current flat layout; the device range table is rebuilt when the layout or the
frozen set changes, never per step."""
import torch
from . import _lib

ADAM_BLOCK = 256            # elements per block of the Adam kernel (misc_ops.cu)


class FlatAdam:
    def __init__(self, params, lr=2e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, groups=None):
        if weight_decay != 0:
            raise NotImplementedError('cc_b200.FlatAdam: weight_decay is 0 in the reference command line')
        self.params = [p for p in params if p.requires_grad]     # constructor order: the checkpoint index
        assert self.params, 'no trainable parameters'
        self.lr, self.betas, self.eps = lr, betas, eps
        self.numel = sum(p.numel() for p in self.params)
        self.grad_scale = 1.0
        self.flat_p = self.flat_g = self.exp_avg = self.exp_avg_sq = None
        if groups is None:
            self.groups = [list(self.params)]
        else:
            mine = {id(p) for p in self.params}
            self.groups = [[p for p in g if id(p) in mine] for g in groups]
            seen = [id(p) for g in self.groups for p in g]
            if len(seen) != len(set(seen)) or set(seen) != mine:
                raise ValueError('FlatAdam: groups must partition the parameters')
        self.group_of = {id(p): gi for gi, g in enumerate(self.groups) for p in g}
        self.frozen = frozenset()
        dev = self.params[0].device
        # group g: state[4g:4g+4] = step, 1-b1^t, sqrt(1-b2^t), unused
        self.state = torch.zeros(4 * len(self.groups), device=dev, dtype=torch.float32)
        self._pack(list(self.params), None)

    # ---- flat layout -------------------------------------------------------------------------------
    def _pack(self, order, old):
        """(Re)build the flat buffers with the parameters in `order`; `old` = {param: (m, v)} state to carry over."""
        dev = order[0].device
        n = self.numel
        flat_p = torch.empty(n, device=dev, dtype=torch.float32)
        flat_g = torch.zeros(n, device=dev, dtype=torch.float32)
        exp_avg = torch.zeros(n, device=dev, dtype=torch.float32)
        exp_avg_sq = torch.zeros(n, device=dev, dtype=torch.float32)
        off = 0
        self.offset = {}
        with torch.no_grad():
            for p in order:
                k = p.numel()
                flat_p[off:off + k].copy_(p.data.reshape(-1))
                if old is not None:
                    exp_avg[off:off + k].copy_(old[p][0].reshape(-1))
                    exp_avg_sq[off:off + k].copy_(old[p][1].reshape(-1))
                    flat_g[off:off + k].copy_(old[p][2].reshape(-1))
                p.data = flat_p[off:off + k].view_as(p)
                gview = flat_g[off:off + k].view_as(p)
                p.grad = gview                 # torch-produced grads accumulate in place into the flat buffer
                p._ccb_grad = gview            # cc_b200.nn backward kernels write here directly
                p._ccb_written = False
                self.offset[p] = (off, k)
                off += k
        self.order = list(order)
        self.flat_p, self.flat_g, self.exp_avg, self.exp_avg_sq = flat_p, flat_g, exp_avg, exp_avg_sq
        self._build_ranges()

    def _views(self, buf, p):
        off, k = self.offset[p]
        return buf[off:off + k].view_as(p)

    def relayout(self, order):
        """Re-pack the flat buffers with the parameters in `order` (a permutation of self.params), keeping
        values, gradients and Adam moments.  Used by the data-parallel bucket scheduler; must precede any CUDA-graph capture."""
        assert len(order) == len(self.params) and set(map(id, order)) == set(map(id, self.params))
        old = {p: (self._views(self.exp_avg, p).clone(), self._views(self.exp_avg_sq, p).clone(),
                   self._views(self.flat_g, p).clone()) for p in self.params}
        self._pack(list(order), old)

    # ---- step groups ---------------------------------------------------------------------------------
    def freeze(self, group_indices):
        """Set the groups step() skips (replacing the previous set).  Rebuilds the device range table: call it between
        steps, not inside a CUDA-graph capture."""
        frozen = frozenset(int(g) for g in group_indices)
        if not all(0 <= g < len(self.groups) for g in frozen):
            raise ValueError('FlatAdam.freeze: group indices %s out of range 0..%d' % (sorted(frozen), len(self.groups) - 1))
        if frozen != self.frozen:
            self.frozen = frozen
            self._build_ranges()

    def ranges(self):
        """[(offset, count, group)]: the maximal runs of one active group in the current flat layout."""
        runs = []
        for p in self.order:
            gi = self.group_of[id(p)]
            if gi in self.frozen:
                continue
            off, k = self.offset[p]
            if runs and runs[-1][2] == gi and runs[-1][0] + runs[-1][1] == off:
                runs[-1][1] += k
            else:
                runs.append([off, k, gi])
        return [tuple(r) for r in runs]

    def _build_ranges(self):
        """Device tables of ccb_adam_step_ranges: {offset, count, group, first_block} per range, active flag per group."""
        dev = self.flat_p.device
        table, nb = [], 0
        for off, k, gi in self.ranges():
            table += [off, k, gi, nb]
            nb += (k + ADAM_BLOCK - 1) // ADAM_BLOCK
        self._nranges, self._nblocks = len(table) // 4, nb
        self._range_table = torch.tensor(table or [0, 0, 0, 0], dtype=torch.int64).to(dev)
        self._active = torch.tensor([0 if g in self.frozen else 1 for g in range(len(self.groups))],
                                    dtype=torch.int32).to(dev)

    # ---- step ----------------------------------------------------------------------------------------
    def zero_grad(self, set_to_none=False):
        """`set_to_none` is accepted for torch compatibility and ignored: the gradients ARE the flat buffer."""
        self.flat_g.zero_()
        for p in self.params:
            p._ccb_written = False
            if p.grad is None:
                p.grad = p._ccb_grad

    def step(self):
        # Gradients are read from the flat buffer only.  If someone replaced p.grad (net.zero_grad(set_to_none=True)
        # followed by a torch-produced gradient installs a fresh tensor), fold that stray gradient in instead of
        # silently dropping it.
        for p in self.params:
            g = p.grad
            if g is not None and g.data_ptr() != p._ccb_grad.data_ptr():
                p._ccb_grad.add_(g)
                p.grad = p._ccb_grad
        _lib.call('ccb_adam_step_ranges', self.flat_p, self.flat_g, self.exp_avg, self.exp_avg_sq, self._range_table,
                  self._nranges, self._nblocks, self._active, len(self.groups), self.state, self.lr, self.betas[0],
                  self.betas[1], self.eps, self.grad_scale, self.flat_p)

    def group_steps(self):
        """Step count of every group (host copy)."""
        return [int(x) for x in self.state.view(-1, 4)[:, 0].tolist()]

    # ---- checkpoint: torch.optim.Adam's state_dict format (reference utils.py:55-63 saves optimizer.state_dict()) ----
    def state_dict(self):
        steps = self.state.view(-1, 4)[:, 0].cpu()
        state = {}
        for i, p in enumerate(self.params):
            step = steps[self.group_of[id(p)]]
            if float(step) > 0:                # a group that never stepped has no state, as in torch
                state[i] = {'step': step.clone(), 'exp_avg': self._views(self.exp_avg, p).detach().clone(),
                            'exp_avg_sq': self._views(self.exp_avg_sq, p).detach().clone()}
        group = {'lr': self.lr, 'betas': tuple(self.betas), 'eps': self.eps, 'weight_decay': 0, 'amsgrad': False,
                 'maximize': False, 'foreach': None, 'capturable': False, 'differentiable': False, 'fused': None,
                 'params': list(range(len(self.params)))}
        return {'state': state, 'param_groups': [group]}

    def load_state_dict(self, sd):
        """A group's counter is the largest step among its parameters that have state (0 when none has)."""
        steps = [0.0] * len(self.groups)
        if 'flat' in sd:                       # round-1 format of this class
            assert self.order == self.params, 'flat optimizer checkpoints predate relayout()'
            self.exp_avg.copy_(sd['exp_avg'])
            self.exp_avg_sq.copy_(sd['exp_avg_sq'])
            steps, g = [float(sd['step'])] * len(self.groups), sd
        else:
            g = sd['param_groups'][0]
            assert len(g['params']) == len(self.params), 'optimizer checkpoint has %d parameters, this model %d' % (
                len(g['params']), len(self.params))
            with torch.no_grad():
                for i, p in enumerate(self.params):
                    st = sd['state'].get(g['params'][i])
                    if st is None:
                        self._views(self.exp_avg, p).zero_()
                        self._views(self.exp_avg_sq, p).zero_()
                    else:
                        self._views(self.exp_avg, p).copy_(st['exp_avg'])
                        self._views(self.exp_avg_sq, p).copy_(st['exp_avg_sq'])
                        gi = self.group_of[id(p)]
                        steps[gi] = max(steps[gi], float(st['step']))
        self.state.zero_()
        self.state.view(-1, 4)[:, 0] = torch.tensor(steps, dtype=torch.float32)
        self.lr, self.betas, self.eps = g['lr'], tuple(g['betas']), g['eps']

    # ---- snapshot / restore (Trainer.capture warms up on real steps and must not train) --------------------------
    def snapshot(self):
        return (self.flat_p.clone(), self.exp_avg.clone(), self.exp_avg_sq.clone(), self.state.clone())

    def restore(self, snap):
        self.flat_p.copy_(snap[0]); self.exp_avg.copy_(snap[1]); self.exp_avg_sq.copy_(snap[2]); self.state.copy_(snap[3])
