"""The reference's alternate architectures (selectable through --dispnet / --posenet / --masknet, train.py:84-89) on
the libccb200 kernels - SURVEY.md row N4.  Same constructors, init_weights(), forward arity, train/eval outputs and
state_dict keys as the reference, so its checkpoints load; ReLU / sigmoid / residual adds run in the conv epilogues.

  DispNetS      models/DispNetS.py:40-133      plain encoder/decoder, 4 disparity scales
  DispNetS6     models/DispNetS6.py:40-137     the same with 6 scales
  DispResNetS6  models/DispResNetS6.py:97-194  DispResNet6 with 3-block encoders / 2-block iconvs from level 4 down
  PoseNet6      models/PoseNet6.py:19-62       PoseNetB6's trunk behind an extra 15->15 stride-2 conv
  PoseExpNet    models/PoseExpNet.py:18-94     SfMLearner's pose + explainability net (4 mask scales)
  MaskResNet6   models/MaskResNet6.py:67-160   residual encoder + MaskNet6's decoder

The alternate flow net, FlowNetC6 (--flownet, train.py:90), has its own module: FlowNetC6.py."""
import torch
import torch.nn as nn
from .. import nn as cnn
from .DispResNet6 import DispResNet6, BasicBlock, make_layer, downsample_conv, predict_disp, upconv, crop_like


def _conv_relu(cin, cout, k=3, stride=1):
    return nn.Sequential(cnn.Conv2d(cin, cout, k, stride=stride, padding=(k - 1) // 2, act='relu'), cnn.Fused())


def _deconv4(cin, cout):
    return nn.Sequential(cnn.ConvTranspose2d(cin, cout, 4, stride=2, padding=1, act='relu'), cnn.Fused())


class _DispNetPlain(nn.Module):
    """Shared body of DispNetS / DispNetS6: 7 two-conv stride-2 encoder stages, 7 (deconv, conv) decoder stages with skip
    concatenations, `nscales` sigmoid heads, the coarser disparity upsampled into the three finest decoder stages."""
    nscales = 4

    def __init__(self, alpha=10, beta=0.01):
        super().__init__()
        self.alpha, self.beta = alpha, beta
        cp = [32, 64, 128, 256, 512, 512, 512]
        ks = [7, 5, 3, 3, 3, 3, 3]
        cin = 3
        for n in range(1, 8):
            setattr(self, 'conv%d' % n, downsample_conv(cin, cp[n - 1], kernel_size=ks[n - 1]))
            cin = cp[n - 1]
        up = [512, 512, 256, 128, 64, 32, 16]
        ins = [cp[6]] + up[:6]
        for j, n in enumerate(range(7, 0, -1)):
            setattr(self, 'upconv%d' % n, upconv(ins[j], up[j]))
        iconv_in = {7: up[0] + cp[5], 6: up[1] + cp[4], 5: up[2] + cp[3], 4: up[3] + cp[2],
                    3: 1 + up[4] + cp[1], 2: 1 + up[5] + cp[0], 1: 1 + up[6]}
        for j, n in enumerate(range(7, 0, -1)):
            setattr(self, 'iconv%d' % n, _conv_relu(iconv_in[n], up[j]))
        for n in range(self.nscales, 0, -1):
            setattr(self, 'predict_disp%d' % n, predict_disp(up[7 - n]))

    def init_weights(self):
        cnn.xavier_init_(self)

    def _disp(self, n, feat):
        return self.alpha * getattr(self, 'predict_disp%d' % n)(feat) + self.beta

    def forward(self, x):
        c = [x]
        for n in range(1, 8):
            c.append(getattr(self, 'conv%d' % n)(c[-1]))
        disps = {}
        feat = c[7]
        for n in range(7, 0, -1):
            skip = c[n - 1]
            parts = [crop_like(getattr(self, 'upconv%d' % n)(feat), skip)]
            if n > 1:
                parts.append(skip)
            if n <= 3:
                parts.append(crop_like(cnn.upsample2x(disps[n + 1]), skip))
            feat = getattr(self, 'iconv%d' % n)(torch.cat(parts, 1))
            if n <= self.nscales:
                disps[n] = self._disp(n, feat)
        if self.training:
            return tuple(disps[n] for n in range(1, self.nscales + 1))
        return disps[1]


class DispNetS(_DispNetPlain):
    nscales = 4


class DispNetS6(_DispNetPlain):
    nscales = 6


class DispResNetS6(DispResNet6):
    """DispResNet6 with deeper stages from level 4 down (models/DispResNetS6.py:109-126)."""

    def __init__(self, alpha=10, beta=0.01):
        super().__init__(alpha, beta)
        cp = [32, 64, 128, 256, 512, 512, 512]
        up = [512, 512, 256, 128, 64, 32, 16]
        for n in range(4, 8):
            setattr(self, 'conv%d' % n, make_layer(cp[n - 2], BasicBlock, cp[n - 1], blocks=3, stride=2))
        iconv_in = {7: up[0] + cp[5], 6: up[1] + cp[4], 5: up[2] + cp[3], 4: up[3] + cp[2]}
        for n in range(7, 3, -1):
            setattr(self, 'iconv%d' % n, make_layer(iconv_in[n], BasicBlock, up[7 - n], blocks=2, stride=1))


class _PoseTrunk(nn.Module):
    def _build_trunk(self, nb_ref_imgs, first):
        planes = [16, 32, 64, 128, 256, 256, 256]
        ks = [7, 5, 3, 3, 3, 3, 3]
        cin = 3 * (1 + nb_ref_imgs)
        if first:
            self.conv0 = _conv_relu(cin, cin, 3, stride=2)
        for i in range(7):
            setattr(self, 'conv%d' % (i + 1), _conv_relu(cin, planes[i], ks[i], stride=2))
            cin = planes[i]
        self.pose_pred = cnn.Conv2d(planes[6], 6 * nb_ref_imgs, 1, padding=0)
        return planes

    def _pose(self, feat):
        pose = self.pose_pred(feat).mean(3).mean(2)
        return 0.01 * pose.view(pose.size(0), self.nb_ref_imgs, 6)

    def init_weights(self):
        cnn.xavier_init_(self)


class PoseNet6(_PoseTrunk):

    def __init__(self, nb_ref_imgs=2):
        super().__init__()
        self.nb_ref_imgs = nb_ref_imgs
        self._build_trunk(nb_ref_imgs, first=True)

    def forward(self, target_image, ref_imgs):
        assert(len(ref_imgs) == self.nb_ref_imgs)
        x = self.conv0(torch.cat([target_image] + list(ref_imgs), 1))
        for i in range(7):
            x = getattr(self, 'conv%d' % (i + 1))(x)
        return self._pose(x)


class PoseExpNet(_PoseTrunk):

    def __init__(self, nb_ref_imgs=2, output_exp=False):
        super().__init__()
        self.nb_ref_imgs, self.output_exp = nb_ref_imgs, output_exp
        planes = self._build_trunk(nb_ref_imgs, first=False)
        if output_exp:
            up = [256, 128, 64, 32, 16]
            ins = [planes[4]] + up[:4]
            for j, n in enumerate(range(5, 0, -1)):
                setattr(self, 'upconv%d' % n, _deconv4(ins[j], up[j]))
            for n in range(4, 0, -1):            # sigmoid applied functionally in the reference (:77-80): fused here
                setattr(self, 'predict_mask%d' % n, cnn.Conv2d(up[5 - n], nb_ref_imgs, 3, padding=1, act='sigmoid'))

    def forward(self, target_image, ref_imgs):
        assert(len(ref_imgs) == self.nb_ref_imgs)
        x = torch.cat([target_image] + list(ref_imgs), 1)
        c = [x]
        for i in range(7):
            c.append(getattr(self, 'conv%d' % (i + 1))(c[-1]))
        pose = self._pose(c[7])
        masks = [None] * 4
        if self.output_exp:
            feat = c[5]
            for n in range(5, 0, -1):
                feat = crop_like(getattr(self, 'upconv%d' % n)(feat), c[n - 1])
                if n <= 4:
                    masks[n - 1] = getattr(self, 'predict_mask%d' % n)(feat)
        if self.training:
            return masks, pose
        return masks[0], pose


class MaskResNet6(nn.Module):

    def __init__(self, nb_ref_imgs=4, output_exp=True):
        super().__init__()
        self.nb_ref_imgs, self.output_exp = nb_ref_imgs, output_exp
        planes = [16, 32, 64, 128, 256, 256]
        self.conv1 = _conv_relu(3 * (1 + nb_ref_imgs), planes[0], 7, stride=2)
        for n in range(2, 7):
            setattr(self, 'conv%d' % n, make_layer(planes[n - 2], BasicBlock, planes[n - 1], blocks=2, stride=2))
        if output_exp:
            up = [256, 256, 128, 64, 32, 16]
            dins = [planes[5]] + [up[j] + planes[4 - j] for j in range(5)]
            for j, n in enumerate(range(6, 0, -1)):
                setattr(self, 'deconv%d' % n, _deconv4(dins[j], up[j]))
            for j, n in enumerate(range(6, 0, -1)):
                setattr(self, 'pred_mask%d' % n, cnn.Conv2d(up[j], nb_ref_imgs, 3, padding=1, act='sigmoid'))

    def init_weights(self):
        cnn.xavier_init_(self)

    def init_mask_weights(self):
        """Reference MaskResNet6.py:107-120: re-initialise only the decoder + heads."""
        for m in self.modules():
            if isinstance(m, cnn.ConvTranspose2d):
                nn.init.xavier_uniform_(m.weight.data)
                if m.bias is not None:
                    m.bias.data.zero_()
        for n in range(1, 7):
            m = getattr(self, 'pred_mask%d' % n)
            nn.init.xavier_uniform_(m.weight.data)
            m.bias.data.zero_()

    def forward(self, target_image, ref_imgs):
        assert(len(ref_imgs) == self.nb_ref_imgs)
        x = torch.cat([target_image] + list(ref_imgs), 1)
        enc = []
        for n in range(1, 7):
            x = getattr(self, 'conv%d' % n)(x)
            enc.append(x)
        if not self.output_exp:
            return (None,) * 6 if self.training else None
        ups = [self.deconv6(enc[5])]
        for n in range(5, 0, -1):
            ups.append(getattr(self, 'deconv%d' % n)(torch.cat((ups[-1], enc[n - 1]), 1)))
        masks = [getattr(self, 'pred_mask%d' % n)(ups[6 - n]) for n in range(1, 7)]
        if self.training:
            return tuple(masks)
        return masks[0]
