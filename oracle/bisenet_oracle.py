"""BiSeNet restated op for op on the CPU in fp32 (torch), from a state dict.

Reference: /root/reference/facelib/parsing/bisenet.py (ConvBNReLU, BiSeNetOutput, AttentionRefinementModule, ContextPath,
FeatureFusionModule, BiSeNet.forward :120-140) and facelib/parsing/resnet.py (ResNet18).  tests/test_oracle_bisenet.py checks
it bit for bit against the unmodified reference class.
"""
from collections import OrderedDict

import torch
import torch.nn.functional as F

from codeformer_b200.bisenet import bisenet_spec


def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + '.running_mean'], sd[p + '.running_var'], sd[p + '.weight'], sd[p + '.bias'], False, 0.1, 1e-5)


def _cbr(x, sd, p, pad=1):
    """ConvBNReLU: conv (no bias), BatchNorm, ReLU."""
    return F.relu(_bn(F.conv2d(x, sd[p + '.conv.weight'], None, 1, pad), sd, p + '.bn'))


def resnet18(sd, x):
    """ResNet18 of resnet.py: returns feat8, feat16, feat32."""
    p = 'cp.resnet.'
    x = F.relu(_bn(F.conv2d(x, sd[p + 'conv1.weight'], None, 2, 3), sd, p + 'bn1'))
    x = F.max_pool2d(x, 3, 2, 1)
    feats = []
    for li in range(4):
        for b in range(2):
            q = f'{p}layer{li + 1}.{b}.'
            s = 2 if (b == 0 and li > 0) else 1
            r = F.relu(_bn(F.conv2d(x, sd[q + 'conv1.weight'], None, s, 1), sd, q + 'bn1'))
            r = _bn(F.conv2d(r, sd[q + 'conv2.weight'], None, 1, 1), sd, q + 'bn2')
            sc = _bn(F.conv2d(x, sd[q + 'downsample.0.weight'], None, s), sd, q + 'downsample.1') if q + 'downsample.0.weight' in sd else x
            x = F.relu(sc + r)
        feats.append(x)
    return feats[1], feats[2], feats[3]


def arm_attention(sd, p, feat):
    """AttentionRefinementModule's attention vector [B,C,1,1] of its ConvBNReLU output."""
    a = F.avg_pool2d(feat, feat.size()[2:])
    return torch.sigmoid(_bn(F.conv2d(a, sd[p + '.conv_atten.weight']), sd, p + '.bn_atten'))


def arm(sd, p, x):
    feat = _cbr(x, sd, p + '.conv')
    return torch.mul(feat, arm_attention(sd, p, feat))


def context_path(sd, x):
    feat8, feat16, feat32 = resnet18(sd, x)
    h8, w8 = feat8.size()[2:]
    h16, w16 = feat16.size()[2:]
    h32, w32 = feat32.size()[2:]
    avg = F.avg_pool2d(feat32, feat32.size()[2:])
    avg = _cbr(avg, sd, 'cp.conv_avg', pad=0)
    avg_up = F.interpolate(avg, (h32, w32), mode='nearest')
    feat32_sum = arm(sd, 'cp.arm32', feat32) + avg_up
    feat32_up = _cbr(F.interpolate(feat32_sum, (h16, w16), mode='nearest'), sd, 'cp.conv_head32')
    feat16_sum = arm(sd, 'cp.arm16', feat16) + feat32_up
    feat16_up = _cbr(F.interpolate(feat16_sum, (h8, w8), mode='nearest'), sd, 'cp.conv_head16')
    return feat8, feat16_up, feat32_up


def ffm_attention(sd, feat):
    """FeatureFusionModule's attention vector [B,C,1,1] of its convblk output."""
    a = F.avg_pool2d(feat, feat.size()[2:])
    return torch.sigmoid(F.conv2d(F.relu(F.conv2d(a, sd['ffm.conv1.weight'])), sd['ffm.conv2.weight']))


def ffm(sd, fsp, fcp):
    feat = _cbr(torch.cat([fsp, fcp], dim=1), sd, 'ffm.convblk', pad=0)
    return torch.mul(feat, ffm_attention(sd, feat)) + feat


def head(sd, p, x):
    return F.conv2d(_cbr(x, sd, p + '.conv'), sd[p + '.conv_out.weight'])


def forward(sd, x):
    """x [B,3,H,W] fp32 -> (out, out16, out32), each [B,num_class,H,W]."""
    h, w = x.size()[2:]
    feat_res8, feat_cp8, feat_cp16 = context_path(sd, x)
    feat_fuse = ffm(sd, feat_res8, feat_cp8)
    outs = (head(sd, 'conv_out', feat_fuse), head(sd, 'conv_out16', feat_cp8), head(sd, 'conv_out32', feat_cp16))
    return tuple(F.interpolate(o, (h, w), mode='bilinear', align_corners=True) for o in outs)


def random_bisenet_state_dict(seed=1, num_class=19, head_bias=(2.0, 1.0, 1.0, 0.5)):
    """Seeded parameters with activations of order 1 through the network: conv weights N(0, 2/fan_in) (the ReLU gain),
    BatchNorm gamma U(0.5, 1) (bn2 / downsample U(0.3, 0.6), so that residual sums stay of order 1), running_var U(0.5, 1.5),
    running_mean / beta 0.1 N.  The attention convs are N(0, 0.5/fan_in), so their sigmoids stay away from 0 and 1.  The
    head ``conv_out.conv_out`` adds ``head_bias`` to the logits of classes 0, 1, 14, 2 through its weights on a constant
    direction, so several classes -- of both mask values -- cover real parts of a face."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    for name, (shape, dtype) in bisenet_spec(num_class).items():
        if dtype == torch.int64:
            t = torch.tensor(100, dtype=torch.int64)
        elif len(shape) == 4:
            fan_in = shape[1] * shape[2] * shape[3]
            gain = 0.5 if ('atten' in name or name.startswith('ffm.conv')) else 2.0
            t = torch.randn(shape, generator=g) * (gain / fan_in) ** 0.5
        elif name.endswith('running_var'):
            t = 0.5 + torch.rand(shape, generator=g)
        elif name.endswith('.weight'):
            lo, hi = (0.3, 0.6) if ('bn2' in name or 'downsample.1' in name) else (0.5, 1.0)
            t = lo + (hi - lo) * torch.rand(shape, generator=g)
        else:
            t = 0.1 * torch.randn(shape, generator=g)
        sd[name] = t
    # the head's input is a ReLU output, positive on average: a bias along the all-ones direction of the 256 channels
    w = sd['conv_out.conv_out.weight']
    for cls, b in zip((0, 1, 14, 2), head_bias):
        w[cls] += b / w.shape[1]
    return sd
