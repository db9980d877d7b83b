"""Data-parallel plumbing: one process per GPU, the flat gradient buffer all-reduced over NCCL in a few
contiguous buckets that overlap the rest of the backward pass.

Replaces the reference's four nn.DataParallel wrappers (train.py:300-303), which scatter the batch,
replicate the modules and gather outputs to GPU0 every step and run every loss on GPU0.  Here each
rank runs the whole step (nets + losses) on its own b/N shard and the only exchange is
ncclAllReduce(sum) over the flat fp32 gradient buffer, averaged by the Adam kernel's
grad_scale = 1/world_size.

Semantics versus the reference (documented deviation):
  * BatchNorm batch statistics are per replica in the reference's DataParallel too - identical.
  * The losses are NOT: the reference gathers the net outputs to GPU0 and evaluates every loss over the
    FULL batch, so `oob_normalization_const = numel/valid.sum()` (loss_functions.py:48,103) and every
    `.mean()` are batch-global.  Here each rank normalises over its own shard and the gradients are then
    averaged: mean_r(oob_r * L_r) instead of oob_full * L_full.  The two agree when the valid fraction is
    the same on every shard and differ by the spread of valid fractions otherwise (SURVEY.md F7).  Exact
    equality would need an all-reduce of the 24 per-(level, ref) valid counts between the loss kernel and
    its finalize step, every step; that exchange is deliberately not on the path.

Overlap: GradBuckets learns, in one eager step, the order in which the parameter gradients are completed
during backward, re-packs the flat buffers in that order (FlatAdam.relayout) and cuts them into buckets
of ~BUCKET_MB; from then on every bucket's all-reduce is issued asynchronously (its own NCCL stream) the
moment its last gradient kernel has been enqueued, and the Adam step waits for all of them."""
import os
import torch
import torch.distributed as dist


def init_from_env(backend=None):
    """torchrun-style env (RANK / LOCAL_RANK / WORLD_SIZE / MASTER_*). Returns (rank, local_rank, world)."""
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        os.environ.setdefault('MASTER_PORT', '29500')
        if backend is None:
            backend = 'nccl' if torch.cuda.is_available() else 'gloo'
        if backend == 'nccl':
            torch.cuda.set_device(local)
            dist.init_process_group(backend, device_id=torch.device('cuda', local))
        else:
            dist.init_process_group(backend)
    return rank, local, world


def bind_to_gpu_numa(local_rank):
    """Pin this process to the CPUs next to its GPU (NVML's ideal affinity) so that pinned host batches are allocated on
    the GPU's NUMA node: a cross-socket H2D copy runs at a fraction of the PCIe rate (seen on the 2-GPU box: GPU1 sits
    on NUMA node 1).  Best effort: any failure leaves the affinity unchanged."""
    try:
        import pynvml
        pynvml.nvmlInit()
        vis = os.environ.get('CUDA_VISIBLE_DEVICES')
        idx = int(vis.split(',')[local_rank]) if vis and vis.split(',')[local_rank].isdigit() else local_rank
        pynvml.nvmlDeviceSetCpuAffinity(pynvml.nvmlDeviceGetHandleByIndex(idx))
        return True
    except Exception:
        return False


def world_size():
    return dist.get_world_size() if dist.is_initialized() else 1


def allreduce_grads(opt):
    """Sum the flat gradient buffer across ranks (one collective) and let Adam average it."""
    w = world_size()
    if w > 1:
        dist.all_reduce(opt.flat_g, op=dist.ReduceOp.SUM)
    opt.grad_scale = 1.0 / w


BUCKET_MB = float(os.environ.get('CCB_BUCKET_MB', '32'))


class _Bucket:
    __slots__ = ('lo', 'hi', 'need', 'have', 'work', 'sched')

    def __init__(self, sched, lo, hi, need):
        self.sched, self.lo, self.hi, self.need, self.have, self.work = sched, lo, hi, need, 0, None

    def note(self, p):
        self.have += 1
        if self.have == self.need and self.work is None:
            self.sched._fire(self)


class GradBuckets:
    """Overlapped gradient exchange for one FlatAdam.  Usage per step:
         opt.zero_grad(); buckets.begin(); loss.backward(); buckets.finish(); opt.step()
    The first `begin()/finish()` pair after construction is the LEARNING step (eager, one whole-buffer
    all-reduce at the end): it records the completion order of the directly-written gradients, after which
    `plan()` re-packs the optimiser and defines the buckets.  Every rank runs the same autograd graph, so the
    completion order - hence the collective order - is identical on every rank (asserted on the bucket table)."""

    def __init__(self, opt, bucket_mb=None, enabled=None):
        self.opt = opt
        self.world = world_size()
        self.enabled = (self.world > 1) if enabled is None else enabled
        self.bucket_floats = int((BUCKET_MB if bucket_mb is None else bucket_mb) * (1 << 20) / 4)
        self.buckets = None
        self.learning = False
        self._order = []
        opt.grad_scale = 1.0 / self.world

    # ---- learning ----------------------------------------------------------------------------------
    class _Recorder:
        def __init__(self, lst):
            self.lst = lst

        def note(self, p):
            self.lst.append(p)

    def begin(self):
        if not self.enabled:
            return
        if self.buckets is None:
            self.learning = True
            self._order = []
            rec = GradBuckets._Recorder(self._order)
            for p in self.opt.params:
                p._ccb_bucket = rec
                p._ccb_indirect = False
        else:
            for b in self.buckets:
                b.have, b.work = 0, None

    def plan(self):
        """After the learning step: relayout + bucket table."""
        opt = self.opt
        seen = set()
        done = []
        for p in self._order:
            if id(p) not in seen and not getattr(p, '_ccb_indirect', False):
                seen.add(id(p))
                done.append(p)
        fixed = {id(p) for p in opt.params if opt.group_of[id(p)] in opt.frozen}    # frozen groups: never exchanged
        done = [p for p in done if id(p) not in fixed]
        rest = [p for p in opt.params if id(p) not in seen and id(p) not in fixed]  # no direct gradient (unused /
        opt.relayout(done + rest + [p for p in opt.params if id(p) in fixed])       # torch-accumulated): tail
        end = sum(p.numel() for p in done + rest)                                    # the fixed parameters follow
        self.buckets = []
        lo, cnt, cur = 0, 0, 0
        for p in done:
            off, k = opt.offset[p]
            cur, cnt = off + k, cnt + 1
            if cur - lo >= self.bucket_floats:
                self.buckets.append(_Bucket(self, lo, cur, cnt))
                lo, cnt = cur, 0
        if cnt:
            self.buckets.append(_Bucket(self, lo, cur, cnt))
            lo = cur
        self.tail = (lo, end) if lo < end else None                 # reduced in finish(): zero or late gradients
        bi = 0
        for p in opt.params:
            p._ccb_bucket = None
        for p in done:
            off, _ = opt.offset[p]
            while off >= self.buckets[bi].hi:
                bi += 1
            p._ccb_bucket = self.buckets[bi]
        self.learning = False
        # every rank must have arrived at the same table (same autograd graph => same completion order)
        if self.world > 1:
            sig = torch.tensor([len(self.buckets)] + [b.hi for b in self.buckets][:62], dtype=torch.int64,
                               device=opt.flat_g.device if dist.get_backend() == 'nccl' else 'cpu')
            sig = torch.nn.functional.pad(sig, (0, 64 - sig.numel()))
            ref = sig.clone()
            dist.broadcast(ref, src=0)
            assert torch.equal(ref, sig), 'gradient buckets differ across ranks'

    # ---- steady state ------------------------------------------------------------------------------
    def _fire(self, b):
        if self.world > 1:
            b.work = dist.all_reduce(self.opt.flat_g[b.lo:b.hi], op=dist.ReduceOp.SUM, async_op=True)
        else:
            b.work = True

    def finish(self):
        if not self.enabled:
            return
        opt = self.opt
        if self.learning:
            if self.world > 1 and not opt.frozen:
                dist.all_reduce(opt.flat_g, op=dist.ReduceOp.SUM)
            elif self.world > 1:
                for off, k, _ in opt.ranges():          # the ranges Adam updates: frozen groups are not exchanged
                    dist.all_reduce(opt.flat_g[off:off + k], op=dist.ReduceOp.SUM)
            self.plan()
            return
        for b in self.buckets:
            if b.work is None:                       # a gradient did not show up this step (e.g. a frozen branch)
                self._fire(b)
        tail_work = None
        if self.tail is not None and self.world > 1:
            tail_work = dist.all_reduce(opt.flat_g[self.tail[0]:self.tail[1]], op=dist.ReduceOp.SUM, async_op=True)
        for b in self.buckets:
            if b.work is not True and b.work is not None:
                b.work.wait()
        if tail_work is not None:
            tail_work.wait()


def broadcast_params(opt, src=0):
    """Once at start-up (identical seeds make this a no-op in practice); never per step."""
    if world_size() > 1:
        dist.broadcast(opt.flat_p, src=src)


def max_over_ranks(value, device):
    t = torch.tensor([float(value)], device=device, dtype=torch.float64)
    if world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


def barrier():
    if world_size() > 1:
        dist.barrier()
