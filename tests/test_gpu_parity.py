"""Parity tests proper: the CUDA path (through cc_b200.* and the C ABI of libccb200.so) against the
oracle and the golden fixtures, on the H100."""
import pytest
import torch
from tests import kernel_cases as KC
from tests.util import conv_impl, device_lib      # noqa: F401  (device_lib: module fixture, the sm_90a library)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures('device_lib')]


@pytest.mark.parametrize('case', KC.ALL_CASES, ids=lambda f: f.__name__)
def test_case(case):
    case(torch.device('cuda:0'))
    torch.cuda.synchronize()


def test_full_size_rigid_loss_vs_cpu_oracle():
    """BASELINE.json size (b4, 256x832, 6 levels): product vs the CPU oracle; masks bit-exact."""
    KC.case_rigid_loss_oracle(torch.device('cuda:0'), B=4, H=256, W=832, NL=6, seed=5, robust=True,
                              oracle_device=torch.device('cpu'))
    KC.case_occlusion_and_valid_masks(torch.device('cuda:0'), B=4, H=256, W=832, NL=6, seed=5)


def test_warp_image_gradient_is_reproducible():
    """The image gradient of flow_warp / Back2Future's feature warp is a scatter; flows that pull many pixels onto a
    few source pixels make float atomics order-dependent.  Two runs must agree bit for bit (values: the parity cases),
    on both kernels (a warp per pixel for small many-channel maps, a thread per pixel otherwise); an inf in grad_out
    reaches only the source pixels it is scattered to."""
    from cc_b200 import inverse_warp as CW, nn as cnn
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(21)
    for (B, C, H, W) in ((2, 64, 48, 160), (2, 3, 128, 416)):
        img = torch.randn(B, C, H, W, generator=g).to(dev)
        ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing='ij')
        # every pixel is pulled to within ~1.5 px of one of a few centres: thousands of contributions per source pixel
        flow = torch.stack([(xs // 40) * 40 + 20 - xs, (ys // 24) * 24 + 12 - ys])[None].repeat(B, 1, 1, 1)
        flow = (flow + 1.5 * torch.rand(B, 2, H, W, generator=g)).to(dev)
        gout = torch.randn(B, C, H, W, generator=g).to(dev)
        for warp in (lambda x: CW.flow_warp(x, flow), lambda x: cnn.feat_warp(x, flow)):
            grads = []
            for _ in range(2):
                x = img.clone().requires_grad_(True)
                (warp(x) * gout).sum().backward()
                grads.append(x.grad)
            assert torch.equal(grads[0], grads[1]), (B, C, H, W)
            assert bool(torch.isfinite(grads[0]).all())
            ginf = gout.clone()
            ginf[0, 0, H // 2, W // 2] = float('inf')
            x = img.clone().requires_grad_(True)
            (warp(x) * ginf).sum().backward()
            bad = ~torch.isfinite(x.grad)
            assert 1 <= int(bad.sum()) <= 4 and bool(bad[0, 0].any()), int(bad.sum())


def test_full_size_properties():
    """Size-independent properties at full size: identity pose + huge depth => warp is the identity on
    interior pixels; zero flow samples at pixel centres - 0.5 (align_corners=False quirk, SURVEY F2)."""
    from cc_b200 import inverse_warp as CW, synth
    dev = torch.device('cuda:0')
    B, H, W = 4, 256, 832
    tgt, refs = synth.frames(B, H, W, seed=9)
    K, Kinv = synth.intrinsics(B, H, W)
    img, K, Kinv = refs[0].to(dev), K.to(dev), Kinv.to(dev)
    flow = torch.zeros(B, 2, H, W, device=dev)
    out = CW.flow_warp(img, flow)
    exp = torch.nn.functional.grid_sample(
        img, torch.stack(torch.meshgrid(torch.linspace(-1, 1, H, device=dev), torch.linspace(-1, 1, W, device=dev),
                                        indexing='ij')[::-1], -1)[None].expand(B, H, W, 2),
        align_corners=False)
    assert (out - exp).abs().max().item() < 1e-5
    # linearity of the backward in grad_out
    depth = synth.depths(B, H, W, 1, seed=2)[0][:, 0].to(dev).requires_grad_(True)
    pose = synth.poses(B, 4, seed=3)[:, 0].to(dev).requires_grad_(True)
    o = CW.inverse_warp(img, depth, pose, K, Kinv)
    g1 = torch.autograd.grad(o.sum(), [depth, pose], retain_graph=True)
    g2 = torch.autograd.grad((2.5 * o).sum(), [depth, pose])
    for a, b in zip(g1, g2):
        assert (2.5 * a - b).abs().max().item() <= 1e-5 * b.abs().max().item() + 1e-12


from tests import net_cases as NC   # noqa: E402


@pytest.mark.parametrize('case', NC.NET_CASES, ids=lambda f: f.__name__)
def test_net_case(case):
    case(torch.device('cuda:0'))
    torch.cuda.synchronize()


def test_conv_big_shapes():
    NC.case_conv_shapes(torch.device('cuda:0'), big=True)


from tests import step_cases as SC   # noqa: E402


def test_flat_adam():
    SC.case_flat_adam(torch.device('cuda:0'))


def test_adam_vs_fp64_per_element():
    SC.case_adam_fp64(torch.device('cuda:0'))


# cfg, B, H, W, bar of the eager losses of steps 0-2 against the CPU oracle (None: not run at full size); cfg2 takes cfg3's
# bar.  Measured on an H100 SXM (400 W power limit), worst step: cfg1 4.5e-5, cfg2 1.6e-5, cfg3 4.6e-5.  cfg1 runs at
# 128x416, where test_train_step_cfg1_vs_oracle sets its bar: at 64x128 the Adam steps amplify DispResNet6's chaotic
# gradient noise (the deepest BatchNorms see 2 values) from 2e-7 at step 0 to 2.8e-4 at step 2.
GRAPH_CASES = [('cfg1', 2, 128, 416, 2e-4), ('cfg2', 2, 64, 128, 1e-3), ('cfg3', 2, 64, 128, 1e-3), ('cfg3', 4, 256, 832, None)]


@pytest.mark.parametrize('cfg,B,H,W,loss_tol', GRAPH_CASES, ids=['%s-b%d-%dx%d' % c[:4] for c in GRAPH_CASES])
def test_train_step_graph_replay_vs_eager(cfg, B, H, W, loss_tol):
    """Trainer.capture() + replay() (what bench.py times) against eager Trainer.step(), bit for bit over three steps;
    Adam against fp64; losses against the oracle at the small size; the BASELINE size runs the benchmark's own split-K
    plans and weight-cache layouts."""
    SC.case_step_graph_vs_eager(torch.device('cuda:0'), cfg, B=B, H=H, W=W, loss_tol=loss_tol)


def test_conv_weight_cache():
    NC.case_conv_weight_cache(torch.device('cuda:0'))


def test_train_step_cfg1_vs_oracle():
    from cc_b200 import _lib
    with conv_impl(_lib.IMPL_FFMA):
        SC.case_step_cfg1(torch.device('cuda:0'), gtol=4e-3)
    with conv_impl(_lib.IMPL_AUTO):
        SC.case_step_cfg1(torch.device('cuda:0'), gtol=5e-2)


def test_conv_tensor_core_3xtf32():
    NC.case_conv_tc(torch.device('cuda:0'))


def test_conv_tma_family():
    """Named after the TMA-fed kernel family it was written for; those Blackwell kernels are gone, and the same thin / odd
    shapes now cross-check the wgmma kernels against the CUDA-core kernels and fp64 torch (net_cases.case_conv_tma_family)."""
    NC.case_conv_tma_family(torch.device('cuda:0'))


def test_alternate_nets():
    """All six alternate architectures (SURVEY N4) against the fixtures frozen from the reference's modules."""
    NC.case_alt_nets(torch.device('cuda:0'))


def test_conv_nhwc_slab():
    """Named after the channels-last slab kernel it was written for; that Blackwell kernel is gone, and the same network
    layer shapes now cross-check the wgmma kernels against the CUDA-core kernels and fp64 torch (net_cases.case_conv_nhwc)."""
    NC.case_conv_nhwc(torch.device('cuda:0'))


def test_joint_step_cfg3_vs_oracle():
    SC.case_step_cfg3(torch.device('cuda:0'))


def test_full_size_loss_layer_vs_cpu_oracle():
    """The flow-photometric, smoothness, BCE and consensus kernels at the BASELINE size (b4 256x832, 6 levels: 960+
    CTAs through the tile/prefix tables) against the CPU oracle."""
    KC.case_loss_layer_fullsize(torch.device('cuda:0'), B=4, H=256, W=832, NL=6, oracle_device=torch.device('cpu'))
    KC.case_consensus_fullsize(torch.device('cuda:0'), B=4, H=256, W=832, NL=6)


from tests import io_cases as IC   # noqa: E402


@pytest.mark.parametrize('case', IC.IO_CASES, ids=lambda f: f.__name__)
def test_io_case(case):
    case(torch.device('cuda:0'))


def test_io_full_size():
    IC.case_metrics_oracle_sizes(torch.device('cuda:0'))
    IC.case_input_pipeline_fullsize(torch.device('cuda:0'))


from tests import helper_cases as HC   # noqa: E402


@pytest.mark.parametrize('case', HC.HELPER_CASES, ids=lambda f: f.__name__)
def test_helper_case(case):
    case(torch.device('cuda:0'))


from tests import eval_cases as EC   # noqa: E402


@pytest.mark.parametrize('case', EC.EVAL_CASES, ids=lambda f: f.__name__)
def test_eval_case(case):
    """Evaluation cores (SURVEY N3: test_disp / test_pose / test_flow sample loops) against the oracle restatement."""
    case(torch.device('cuda:0'))


from tests import loss_audit as LSA   # noqa: E402


@pytest.mark.parametrize('opts', [{}] + LSA.SWEEP, ids=lambda o: '-'.join('%s=%s' % kv for kv in o.items()) or 'cfg3')
def test_loss_audit_options(opts):
    """The loss audit on the sm_90a build: the cfg3 loss layer at b2 64x128 and the template paths the step never takes
    (SSIM compiled out, powf, the oob term, border padding, quaternion poses, no masks, an 84x136 frame with 3 levels)."""
    o = dict(opts)
    kw = {k: o.pop(k) for k in ('H', 'W', 'NL') if k in o}
    with LSA.LossAudit(tag='gpu_' + ('_'.join(map(str, opts.values())) or 'cfg3')):
        LSA.cfg3_losses(torch.device('cuda:0'), opts=o, **kw)
    torch.cuda.synchronize()
