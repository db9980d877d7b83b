"""The N>1 path of cc_b200.dist on CPU: world_size-2 gloo, flat-gradient all-reduce + averaged Adam step.
(The kernels run through the CPU simulator build; what is under test is the host-side exchange logic.)"""
import os
import sys
import torch
import torch.multiprocessing as mp
from tests.util import sim_lib      # noqa: F401  (module fixture: the simulator library)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR='127.0.0.1',
                      MASTER_PORT=str(port))
    import build_sim
    from cc_b200 import _lib, dist as cdist, nn as cnn
    from cc_b200.optim import FlatAdam
    _lib.use_library(build_sim.build())
    r, _, w = cdist.init_from_env(backend='gloo')
    assert (r, w) == (rank, world)
    torch.manual_seed(0)                                   # identical init on every rank
    conv = cnn.Conv2d(3, 4, 3, padding=1)
    opt = FlatAdam(conv.parameters(), lr=1e-2)
    cdist.broadcast_params(opt)
    x = torch.randn(2, 3, 6, 7, generator=torch.Generator().manual_seed(100 + rank))   # different shard per rank
    opt.zero_grad()
    (conv(x) ** 2).mean().backward()
    local_g = opt.flat_g.clone()
    cdist.allreduce_grads(opt)
    summed = opt.flat_g.clone()
    opt.step()
    ret[rank] = (local_g, summed, opt.flat_p.clone(), opt.grad_scale)
    cdist.barrier()
    torch.distributed.destroy_process_group()


def test_two_rank_allreduce_and_step():
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))
    import build_sim
    build_sim.build()                       # build once in the parent so the workers only load it
    world = 2
    port = 29500 + (os.getpid() % 2000)
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
    g0, s0, p0, sc0 = ret[0]
    g1, s1, p1, sc1 = ret[1]
    assert sc0 == sc1 == 0.5
    assert torch.allclose(s0, g0 + g1, rtol=1e-6, atol=1e-8) and torch.equal(s0, s1)
    assert torch.equal(p0, p1)              # identical parameters after the averaged step
    # equals a single-process Adam step on the mean gradient
    sys.path.insert(0, ROOT)
    from oracle.step import Adam
    from cc_b200 import nn as cnn
    torch.manual_seed(0)
    conv = cnn.Conv2d(3, 4, 3, padding=1)
    flat = torch.cat([q.detach().reshape(-1) for q in conv.parameters()]).clone().requires_grad_(True)
    flat.grad = (g0 + g1) / 2
    o = Adam([flat], 1e-2)
    o.step()
    assert torch.allclose(flat.detach(), p0, rtol=1e-5, atol=1e-7)


def _bucket_worker(rank, world, port, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR='127.0.0.1',
                      MASTER_PORT=str(port))
    import build_sim
    from cc_b200 import _lib, dist as cdist, nn as cnn
    from cc_b200.optim import FlatAdam
    _lib.use_library(build_sim.build())
    cdist.init_from_env(backend='gloo')

    def make():
        torch.manual_seed(0)
        return torch.nn.Sequential(cnn.Conv2d(3, 6, 3, padding=1, act='relu'), cnn.Conv2d(6, 6, 3, padding=1, act='relu'),
                                   cnn.BatchNorm2d(6), cnn.Conv2d(6, 2, 3, padding=1))

    xs = [torch.randn(2, 3, 6, 7, generator=torch.Generator().manual_seed(100 * s + rank)) for s in range(3)]
    # (a) overlapped buckets (tiny bucket size => several buckets, relayout in completion order)
    net = make()
    opt = FlatAdam(net.parameters(), lr=1e-2)
    bk = cdist.GradBuckets(opt, bucket_mb=100 * 4 / (1 << 20))
    assert bk.enabled
    for x in xs:
        opt.zero_grad(); bk.begin()
        (net(x) ** 2).mean().backward()
        bk.finish(); opt.step()
    nb = len(bk.buckets)
    fired = [b.work is not None for b in bk.buckets]
    pa = {k: v.detach().clone() for k, v in net.state_dict().items()}
    sd = opt.state_dict()
    # (b) one all-reduce after backward (round-1 path)
    net2 = make()
    opt2 = FlatAdam(net2.parameters(), lr=1e-2)
    for x in xs:
        opt2.zero_grad()
        (net2(x) ** 2).mean().backward()
        cdist.allreduce_grads(opt2); opt2.step()
    pb = {k: v.detach().clone() for k, v in net2.state_dict().items()}
    # the first parameters in the re-packed flat buffer are the LAST layer's (their gradients complete first)
    first = opt.order[0]
    last_layer = [p for p in net[3].parameters()]
    ret[rank] = (nb, fired, pa, pb, any(first is q for q in last_layer), sd, opt2.state_dict())
    cdist.barrier()
    torch.distributed.destroy_process_group()


def test_two_rank_overlapped_buckets_match_single_allreduce():
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))
    import build_sim
    build_sim.build()
    world = 2
    port = 31500 + (os.getpid() % 2000)
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_bucket_worker, args=(world, port, ret), nprocs=world, join=True)
    for r in range(world):
        nb, fired, pa, pb, first_is_last_layer, sd, sd2 = ret[r]
        assert nb >= 3 and all(fired), (nb, fired)
        assert first_is_last_layer
        for k in pa:
            assert torch.allclose(pa[k], pb[k], rtol=1e-6, atol=1e-7), k
        # optimizer checkpoints are layout-independent (torch.optim.Adam format, constructor order)
        assert sd['param_groups'][0]['params'] == sd2['param_groups'][0]['params']
        for i in sd['state']:
            assert torch.allclose(sd['state'][i]['exp_avg'], sd2['state'][i]['exp_avg'], rtol=1e-5, atol=1e-8)
    # parameters identical on both ranks (BatchNorm running statistics are per replica, like DataParallel's)
    assert all(torch.equal(ret[0][2][k], ret[1][2][k]) for k in ret[0][2] if 'running' not in k and 'num_batches' not in k)


def test_flat_adam_checkpoint_roundtrip_with_torch_adam(sim_lib):
    """FlatAdam.state_dict() loads into torch.optim.Adam and back (reference utils.py:55-63 saves optimizer.state_dict())."""
    from cc_b200 import nn as cnn
    from cc_b200.optim import FlatAdam
    torch.manual_seed(1)
    net = torch.nn.Sequential(cnn.Conv2d(3, 4, 3, padding=1, act='relu'), cnn.Conv2d(4, 2, 3, padding=1))
    opt = FlatAdam(net.parameters(), lr=1e-2)
    x = torch.randn(2, 3, 5, 6)
    for _ in range(2):
        opt.zero_grad(); (net(x) ** 2).mean().backward(); opt.step()
    sd = opt.state_dict()
    ref = torch.optim.Adam([torch.nn.Parameter(p.detach().clone()) for p in net.parameters()], lr=1e-2)
    ref.load_state_dict(sd)                                      # torch accepts it
    opt.relayout(list(reversed(opt.params)))                       # layout change must not change the checkpoint
    sd2 = opt.state_dict()
    for i in sd['state']:
        assert torch.equal(sd['state'][i]['exp_avg_sq'], sd2['state'][i]['exp_avg_sq'])
    opt3 = FlatAdam([torch.nn.Parameter(p.detach().clone()) for p in net.parameters()], lr=5e-3)
    opt3.load_state_dict(ref.state_dict())                        # and back from torch
    assert opt3.lr == 1e-2 and abs(float(opt3.state[0]) - 2.0) < 1e-6
    for i, p in enumerate(opt3.params):
        assert torch.allclose(opt3._views(opt3.exp_avg, p), sd['state'][i]['exp_avg'])
    # a stray gradient installed by net.zero_grad(set_to_none=True) + a torch-produced grad is folded in, not dropped
    opt.zero_grad()
    p0 = opt.params[0]
    p0.grad = None
    p0.grad = torch.ones_like(p0)
    before = p0.detach().clone()
    opt.step()
    assert not torch.equal(before, p0.detach()) and p0.grad.data_ptr() == p0._ccb_grad.data_ptr()
