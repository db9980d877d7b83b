"""FlowNetC6 (the reference's second flow network, --flownet FlowNetC6) on the libccb200 kernels.
Reference: models/FlowNetC6.py:32-164 with models/submodules.py:5-39.  Same constructor, init_weights(), forward arity
`flow(x1, x2)`, train-mode 6-tuple (flow1 .. flow6, full resolution down to 1/32) / eval-mode flow1 and state_dict keys
(`conv1.0.weight`, `deconv5.0.bias`, `upsampled_flow6_to_5.weight`, ...), so reference checkpoints load.

The LeakyReLU(0.1) of every conv / deconv block runs in the convolution epilogue (a cnn.Fused placeholder keeps the
nn.Sequential index), the correlation's LeakyReLU in the cost-volume kernel (cc_b200.nn.corr441d).  H and W must be
multiples of 64: the reference concatenates the skips without cropping."""
import torch
import torch.nn as nn
from .. import nn as cnn

SLOPE = 0.1


def conv(in_planes, out_planes, kernel_size=3, stride=1):
    return nn.Sequential(cnn.Conv2d(in_planes, out_planes, kernel_size, stride=stride, padding=(kernel_size - 1) // 2,
                                    act='leaky', slope=SLOPE), cnn.Fused('leaky'))


def deconv(in_planes, out_planes):
    return nn.Sequential(cnn.ConvTranspose2d(in_planes, out_planes, 4, stride=2, padding=1, act='leaky', slope=SLOPE),
                         cnn.Fused('leaky'))


def predict_flow(in_planes):
    return cnn.Conv2d(in_planes, 2, 3, stride=1, padding=1)


class FlowNetC6(nn.Module):
    def __init__(self, nlevels=5, batchNorm=False, div_flow=20, full_res=True, pretrained=True):
        super().__init__()
        if batchNorm:
            raise NotImplementedError('cc_b200 FlowNetC6: batchNorm=True is not built (no reference caller uses it)')
        if not full_res:
            raise NotImplementedError('cc_b200 FlowNetC6: full_res=False is not built (no reference caller uses it)')
        self.batchNorm, self.div_flow, self.full_res = batchNorm, div_flow, full_res
        self.conv1 = conv(3, 64, kernel_size=7, stride=2)
        self.conv2 = conv(64, 128, kernel_size=5, stride=2)
        self.conv3 = conv(128, 256, kernel_size=5, stride=2)
        self.conv_redir = conv(256, 32, kernel_size=1, stride=1)
        self.conv3_1 = conv(473, 256)
        self.conv4 = conv(256, 512, stride=2)
        self.conv4_1 = conv(512, 512)
        self.conv5 = conv(512, 512, stride=2)
        self.conv5_1 = conv(512, 512)
        self.conv6 = conv(512, 1024, stride=2)
        self.conv6_1 = conv(1024, 1024)
        self.deconv5 = deconv(1024, 512)
        self.deconv4 = deconv(1026, 256)
        self.deconv3 = deconv(770, 128)
        self.deconv2 = deconv(386, 64)
        self.deconv1 = deconv(194, 32)
        for n, c in zip(range(6, 0, -1), (1024, 1026, 770, 386, 194, 98)):
            setattr(self, 'predict_flow%d' % n, predict_flow(c))
        for n in range(6, 1, -1):
            setattr(self, 'upsampled_flow%d_to_%d' % (n, n - 1), cnn.ConvTranspose2d(2, 2, 4, stride=2, padding=1))

    def init_weights(self):
        cnn.xavier_init_(self, bias_uniform=True)

    def forward(self, x1, x2):
        if x1.shape[-2] % 64 or x1.shape[-1] % 64:
            raise ValueError('FlowNetC6: H and W must be multiples of 64, got %dx%d' % tuple(x1.shape[-2:]))
        c1a = self.conv1(x1)
        c2a = self.conv2(c1a)
        c3a = self.conv3(c2a)
        c3b = self.conv3(self.conv2(self.conv1(x2)))
        corr = cnn.corr441d(c3a, c3b)                                   # LeakyReLU(0.1) fused
        c3_1 = self.conv3_1(torch.cat((self.conv_redir(c3a), corr), 1))
        c4 = self.conv4_1(self.conv4(c3_1))
        c5 = self.conv5_1(self.conv5(c4))
        c6 = self.conv6_1(self.conv6(c5))
        skips = {5: c5, 4: c4, 3: c3_1, 2: c2a, 1: c1a}
        flows = {6: self.predict_flow6(c6)}
        feat = c6
        for n in range(5, 0, -1):
            up = getattr(self, 'upsampled_flow%d_to_%d' % (n + 1, n))(flows[n + 1])
            feat = torch.cat((skips[n], getattr(self, 'deconv%d' % n)(feat), up), 1)
            flows[n] = getattr(self, 'predict_flow%d' % n)(feat)
        if not self.training:
            return self.div_flow * cnn.upsample2x(flows[1])
        return tuple(self.div_flow * cnn.upsample2x(flows[n]) for n in range(1, 7))
