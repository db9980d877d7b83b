"""Training with fixed networks on the CPU simulator build: Adam over ranges with per-network step counters, FlatAdam
against torch.optim.Adam over training phases, the two-rank bucket exchange with a fixed network, and the photometric
loss's value-only and mask-gradient-free paths."""
import os
import sys
import pytest
import torch
import torch.multiprocessing as mp

from tests import frozen_cases as FC
from tests.util import sim_lib      # noqa: F401  (module fixture: the simulator library)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.usefixtures('sim_lib')


@pytest.mark.parametrize('case', [FC.case_adam_ranges_fp64, FC.case_flat_adam_phases, FC.case_load_missing_group_state,
                                  FC.case_photo_value_only], ids=lambda f: f.__name__)
def test_frozen_case(case):
    case(torch.device('cpu'))


def test_freeze_rejects_bad_groups():
    from cc_b200 import nn as cnn
    from cc_b200.optim import FlatAdam
    a, b = cnn.Conv2d(2, 3, 3), cnn.Conv2d(3, 1, 3)
    with pytest.raises(ValueError):
        FlatAdam(list(a.parameters()) + list(b.parameters()), groups=[list(a.parameters())])
    opt = FlatAdam(list(a.parameters()) + list(b.parameters()), groups=[list(a.parameters()), list(b.parameters())])
    with pytest.raises(ValueError):
        opt.freeze([2])
    opt.freeze([0, 1])
    assert opt.ranges() == []


def test_trainer_fixed_names():
    from cc_b200.train_step import Trainer
    with pytest.raises(ValueError):
        Trainer('cfg1', 'cpu', fixed=('disp', 'pose'))         # nothing left to train
    with pytest.raises(ValueError):
        Trainer('cfg1', 'cpu', fixed=('mask',))                # not a net of cfg1
    tr = Trainer('cfg1', 'cpu', fixed=('pose',))
    assert tr.fixed == ('pose',) and tr.opt.frozen == {1}
    assert not any(p.requires_grad for p in tr.nets['pose'].parameters())
    assert all(p.requires_grad for p in tr.nets['disp'].parameters()) and tr.nets['pose'].training
    tr.set_fixed(())
    assert tr.opt.frozen == set() and all(p.requires_grad for p in tr.nets['pose'].parameters())


# ---- two ranks, one network fixed ------------------------------------------------------------------------------------
def _fixed_worker(rank, world, port, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR='127.0.0.1',
                      MASTER_PORT=str(port))
    import build_sim
    from cc_b200 import _lib, dist as cdist, nn as cnn
    from cc_b200.optim import FlatAdam
    _lib.use_library(build_sim.build())
    cdist.init_from_env(backend='gloo')
    torch.manual_seed(0)
    A = torch.nn.Sequential(cnn.Conv2d(3, 6, 3, padding=1, act='relu'), cnn.Conv2d(6, 4, 3, padding=1, act='relu'))
    B = torch.nn.Sequential(cnn.Conv2d(4, 5, 3, padding=1, act='relu'), cnn.Conv2d(5, 2, 3, padding=1))
    opt = FlatAdam(list(A.parameters()) + list(B.parameters()), lr=1e-2, groups=[list(A.parameters()), list(B.parameters())])
    bk = cdist.GradBuckets(opt, bucket_mb=100 * 4 / (1 << 20))
    A.requires_grad_(False)                                # A fixed
    opt.freeze([0])
    a0 = [p.detach().clone() for p in A.parameters()]
    overlaps = []
    real = cdist.dist.all_reduce

    def logged(t, *args, **kw):
        base = opt.flat_g.data_ptr()
        if t.data_ptr() >= base and t.data_ptr() < base + 4 * opt.numel:
            lo = (t.data_ptr() - base) // 4
            hi = lo + t.numel()
            for p in A.parameters():
                off, k = opt.offset[p]
                if lo < off + k and off < hi:
                    overlaps.append((lo, hi, off, k))
        return real(t, *args, **kw)
    cdist.dist.all_reduce = logged
    try:
        for s in range(3):
            x = torch.randn(2, 3, 6, 7, generator=torch.Generator().manual_seed(100 * s + rank))
            opt.zero_grad(); bk.begin()
            (B(A(x)) ** 2).mean().backward()
            bk.finish(); opt.step()
    finally:
        cdist.dist.all_reduce = real
    a_same = all(torch.equal(p, q) for p, q in zip(A.parameters(), a0))
    fixed_tail = min(opt.offset[p][0] for p in A.parameters()) >= max(opt.offset[p][0] + opt.offset[p][1] for p in B.parameters())
    ret[rank] = (overlaps, a_same, fixed_tail, [p.detach().clone() for p in B.parameters()], opt.group_steps())
    cdist.barrier()
    torch.distributed.destroy_process_group()


def test_two_rank_fixed_net_is_never_exchanged():
    import build_sim
    build_sim.build()
    world = 2
    port = 33500 + (os.getpid() % 2000)
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_fixed_worker, args=(world, port, ret), nprocs=world, join=True)
    for r in range(world):
        overlaps, a_same, fixed_tail, _, steps = ret[r]
        assert overlaps == [], f'rank {r}: all-reduce touched the fixed net: {overlaps}'
        assert a_same, f'rank {r}: the fixed net moved'
        assert fixed_tail, f'rank {r}: the fixed net is not packed after the trained one'
        assert steps == [0, 3], steps
    assert all(torch.equal(p, q) for p, q in zip(ret[0][3], ret[1][3])), 'ranks disagree on the trained net'
