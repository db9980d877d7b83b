"""Oracle for FlowNetC6: a functional CPU fp32 restatement over a state_dict, the dilated correlation it needs, and the
oracle training step / flow evaluation with FlowNetC6 as the flow net.  TEST INFRASTRUCTURE.

* FlowNetC6  : reference models/FlowNetC6.py:32-164 (+ submodules.py:5-39); state_dict keys as the reference module's.
* correlate  : reference models/FlowNetC6.py:18-30.  PARITY UNPINNED, as for Back2Future's correlation (oracle/nets.py,
  SURVEY.md section 8c): the third-party spatial_correlation_sampler is absent from the reference, so its behaviour is
  restated from its documentation, with the dilation the FlowNetC6 call site asks for:
      out[b, ph, pw, y, x] = sum_c in1[b,c,y,x] * in2[b,c, y + d (ph - P//2), x + d (pw - P//2)]   (zero outside)
  with kernel_size=1, stride=1, padding=0, patch_size P=21, dilation_patch d=2; the first patch index is the vertical
  displacement.  At P=9, d=1 this is oracle.nets.spatial_correlation_sample.
* with_flownetc6(): while active, oracle.nets.flow_forward runs FlowNetC6 the way the reference's train.py:465-466 and
  test_flow.py:125 call it (flow_fwd = net(tgt, ref+), flow_bwd = net(tgt, ref-)), so the unchanged oracle.step and
  oracle.evaluate bodies give the --flownet FlowNetC6 step and evaluation."""
import contextlib
import torch
import torch.nn.functional as F
from oracle import nets as ON, step as OS

PATCH, DILATION = 21, 2
SLOPE = 0.1
NPARAMS = 39276490
# (name, in, out, kernel, stride) of the conv blocks (Conv2d + bias + LeakyReLU 0.1), registration order
CONVS = [('conv1', 3, 64, 7, 2), ('conv2', 64, 128, 5, 2), ('conv3', 128, 256, 5, 2), ('conv_redir', 256, 32, 1, 1),
         ('conv3_1', 473, 256, 3, 1), ('conv4', 256, 512, 3, 2), ('conv4_1', 512, 512, 3, 1), ('conv5', 512, 512, 3, 2),
         ('conv5_1', 512, 512, 3, 1), ('conv6', 512, 1024, 3, 2), ('conv6_1', 1024, 1024, 3, 1)]
DECONVS = [(5, 1024, 512), (4, 1026, 256), (3, 770, 128), (2, 386, 64), (1, 194, 32)]     # ConvT k4 s2 p1 + LeakyReLU
PREDICT_IN = {6: 1024, 5: 1026, 4: 770, 3: 386, 2: 194, 1: 98}                            # 3x3 -> 2, no activation


def spatial_correlation_sample(in1, in2, patch=PATCH, dilation=DILATION):
    """Restated third-party op (module docstring): [B,C,H,W] x2 -> [B,patch,patch,H,W]."""
    B, C, H, W = in1.shape
    r = (patch // 2) * dilation
    pad = F.pad(in2, (r, r, r, r))
    rows = []
    for ph in range(patch):
        y = ph * dilation
        rows.append(torch.stack([(in1 * pad[:, :, y:y + H, pw * dilation:pw * dilation + W]).sum(1) for pw in range(patch)], 1))
    return torch.stack(rows, 1)


def correlate(in1, in2):
    """Reference models/FlowNetC6.py:18-30: [B,441,H,W], divided by C (no activation)."""
    out = spatial_correlation_sample(in1, in2)
    b, ph, pw, h, w = out.size()
    return out.view(b, ph * pw, h, w) / in1.size(1)


def flownetc6_forward(p, x1, x2, training=True, div_flow=20):
    """Train mode: (flow1, ..., flow6), each div_flow * bilinear x2 of the head (full_res=True); eval mode: flow1."""
    spec = {name: (k, s) for name, _, _, k, s in CONVS}

    def conv(name, x):
        k, s = spec[name]
        return F.leaky_relu(F.conv2d(x, p[name + '.0.weight'], p[name + '.0.bias'], s, (k - 1) // 2), SLOPE)

    def tower(x):
        c1 = conv('conv1', x)
        c2 = conv('conv2', c1)
        return c1, c2, conv('conv3', c2)

    c1a, c2a, c3a = tower(x1)
    c3b = tower(x2)[2]
    corr = F.leaky_relu(correlate(c3a, c3b), SLOPE)
    c3_1 = conv('conv3_1', torch.cat((conv('conv_redir', c3a), corr), 1))
    c4 = conv('conv4_1', conv('conv4', c3_1))
    c5 = conv('conv5_1', conv('conv5', c4))
    c6 = conv('conv6_1', conv('conv6', c5))
    skips = {5: c5, 4: c4, 3: c3_1, 2: c2a, 1: c1a}
    pred = lambda n, t: F.conv2d(t, p['predict_flow%d.weight' % n], p['predict_flow%d.bias' % n], 1, 1)      # noqa: E731
    flows = {6: pred(6, c6)}
    feat = c6
    for n in range(5, 0, -1):
        dec = F.leaky_relu(F.conv_transpose2d(feat, p['deconv%d.0.weight' % n], p['deconv%d.0.bias' % n], stride=2, padding=1),
                           SLOPE)
        up = F.conv_transpose2d(flows[n + 1], p['upsampled_flow%d_to_%d.weight' % (n + 1, n)],
                                p['upsampled_flow%d_to_%d.bias' % (n + 1, n)], stride=2, padding=1)
        feat = torch.cat((skips[n], dec, up), 1)
        flows[n] = pred(n, feat)
    outs = [div_flow * F.interpolate(flows[n], scale_factor=2, mode='bilinear', align_corners=False) for n in range(1, 7)]
    return tuple(outs) if training else outs[0]


def _as_flow_forward(p, im_tar, im_refs, nlevels=6, training=True, with_occ=True):
    """oracle.nets.flow_forward's interface (im_refs = [I-, I+]) over FlowNetC6: train.py:465-466, test_flow.py:125."""
    if not training:
        return flownetc6_forward(p, im_tar, im_refs[1], training=False), None, None
    return list(flownetc6_forward(p, im_tar, im_refs[1])), list(flownetc6_forward(p, im_tar, im_refs[0])), None


@contextlib.contextmanager
def with_flownetc6():
    saved = ON.flow_forward
    ON.flow_forward = _as_flow_forward
    try:
        yield
    finally:
        ON.flow_forward = saved


def step_flow_params(seed=320, head_scale=0.05):
    """FlowNetC6 weights for step tests: synth.seeded_fill, the six predict_flow heads scaled by head_scale.
    Every output is 20 x a head upsampled, so the flows of the reference init (xavier, U[0,1) biases) or of seeded_fill
    alone are several pixels even on the 2x4 coarsest level of a 64x128 frame: every pixel of that level then samples
    outside the frame and the flow photometric loss is inf (in the reference as here).  Scaled heads keep the flows
    below a pixel there."""
    from cc_b200 import models as CM, synth
    sd = synth.seeded_fill(CM.FlowNetC6(), seed).state_dict()
    for k in sd:
        if k.startswith('predict_flow'):
            sd[k] = sd[k] * head_scale
    return sd


def make_params(cfg, requires_grad=True):
    """oracle.step.make_params with FlowNetC6 parameters (step_flow_params) for 'flow'."""
    P = OS.make_params(cfg, requires_grad)
    if 'flow' in P:
        P['flow'] = ON.clone_params(step_flow_params(), requires_grad=requires_grad)
    return P
