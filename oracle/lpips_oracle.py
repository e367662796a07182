"""torch fp32 restatement (CPU) of LPIPS-VGG, lpips 0.1 ``LPIPS(net='vgg', version='0.1', lpips=True, spatial=False)``, of
basicsr's ``LPIPSLoss`` (basicsr/losses/losses.py:257-282) and of the two uint8 conventions the package scores images in.

The lpips package is restated from its published definition (ScalingLayer, the five torchvision ``vgg16().features``
slices, normalize_tensor, the 1x1 ``lin`` layers, spatial_average); the backbone is torchvision's own module, built with
``weights=None``.  tests/test_oracle_lpips.py pins the slices against torchvision and the reference's ``LPIPSLoss`` against
this class bit for bit.
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn
import torchvision

SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
CHANNELS = (64, 128, 256, 512, 512)
SLICES = ((0, 4), (4, 9), (9, 16), (16, 23), (23, 30))


class ScalingLayer(nn.Module):
    def __init__(self):
        super().__init__()
        self.register_buffer('shift', torch.Tensor(SHIFT)[None, :, None, None])
        self.register_buffer('scale', torch.Tensor(SCALE)[None, :, None, None])

    def forward(self, inp):
        return (inp - self.shift) / self.scale


class Vgg16(nn.Module):
    """torchvision vgg16().features in the five lpips slices; forward -> [relu1_2, relu2_2, relu3_3, relu4_3, relu5_3]."""

    def __init__(self):
        super().__init__()
        features = torchvision.models.vgg16(weights=None).features
        for s, (a, b) in enumerate(SLICES, 1):
            sl = nn.Sequential()
            for x in range(a, b):
                sl.add_module(str(x), features[x])
            setattr(self, f'slice{s}', sl)

    def forward(self, x):
        out = []
        for s in range(1, 6):
            x = getattr(self, f'slice{s}')(x)
            out.append(x)
        return out


class NetLinLayer(nn.Module):
    def __init__(self, chn_in, chn_out=1):
        super().__init__()
        self.model = nn.Sequential(nn.Dropout(), nn.Conv2d(chn_in, chn_out, 1, stride=1, padding=0, bias=False))

    def forward(self, x):
        return self.model(x)


def normalize_tensor(in_feat, eps=1e-10):
    norm_factor = torch.sqrt(torch.sum(in_feat ** 2, dim=1, keepdim=True))
    return in_feat / (norm_factor + eps)


def spatial_average(in_tens, keepdim=True):
    return in_tens.mean([2, 3], keepdim=keepdim)


class LPIPS(nn.Module):
    """lpips.LPIPS(net='vgg', version='0.1', lpips=True, spatial=False) with random backbone and lin weights (load a state
    dict); the keyword arguments of the lpips constructor that select other forms are not restated."""

    def __init__(self, net='vgg', spatial=False, **kwargs):
        super().__init__()
        assert net == 'vgg' and not spatial
        self.scaling_layer = ScalingLayer()
        self.L = 5
        self.net = Vgg16()
        self.lin0, self.lin1, self.lin2, self.lin3, self.lin4 = (NetLinLayer(c) for c in CHANNELS)
        self.lins = nn.ModuleList([self.lin0, self.lin1, self.lin2, self.lin3, self.lin4])
        self.eval()

    def forward(self, in0, in1, retPerLayer=False, normalize=False):
        if normalize:
            in0 = 2 * in0 - 1
            in1 = 2 * in1 - 1
        outs0, outs1 = self.net.forward(self.scaling_layer(in0)), self.net.forward(self.scaling_layer(in1))
        diffs = [(normalize_tensor(outs0[k]) - normalize_tensor(outs1[k])) ** 2 for k in range(self.L)]
        res = [spatial_average(self.lins[k](diffs[k]), keepdim=True) for k in range(self.L)]
        val = 0
        for k in range(self.L):
            val += res[k]
        return (val, res) if retPerLayer else val


def random_lpips_state_dict(seed=1):
    """Seeded lpips-layout parameters: He-scaled conv weights N(0, 2 / fan_in), so activations stay of order 1 through the
    13 ReLU layers, biases 0.01 N, lin weights U(0, 2 / C) (lpips keeps them >= 0); the ScalingLayer constants."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    for k, v in LPIPS().state_dict().items():
        if k.startswith('scaling_layer.'):
            t = v.clone()
        elif k.startswith('lins.'):
            t = sd['lin' + k[len('lins.'):]]
        elif k.startswith('lin'):
            t = torch.rand(v.shape, generator=g) * (2.0 / v.shape[1])
        elif k.endswith('.bias'):
            t = 0.01 * torch.randn(v.shape, generator=g)
        else:
            t = torch.randn(v.shape, generator=g) * (2.0 / (v.shape[1] * 9)) ** 0.5
        sd[k] = t
    return sd


class LPIPSLoss(nn.Module):
    """basicsr's LPIPSLoss (losses.py:257-282) on the restated LPIPS."""

    def __init__(self, loss_weight=1.0, use_input_norm=True, range_norm=False):
        super().__init__()
        self.perceptual = LPIPS(net='vgg', spatial=False).eval()
        self.loss_weight = loss_weight
        self.use_input_norm = use_input_norm
        self.range_norm = range_norm
        if self.use_input_norm:
            self.register_buffer('mean', torch.Tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1))
            self.register_buffer('std', torch.Tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1))

    def forward(self, pred, target):
        if self.range_norm:
            pred = (pred + 1) / 2
            target = (target + 1) / 2
        if self.use_input_norm:
            pred = (pred - self.mean) / self.std
            target = (target - self.mean) / self.std
        return self.loss_weight * self.perceptual(target.contiguous(), pred.contiguous()).mean()


# ---- uint8 conventions -----------------------------------------------------------------------------------------------
def im2tensor(image, imtype=np.uint8, cent=1., factor=255. / 2.):
    """lpips.im2tensor: an RGB HWC image -> [1,3,H,W] float32 in [-1, 1] (float64 arithmetic, then the cast)."""
    return torch.Tensor((image / factor - cent)[:, :, :, np.newaxis].transpose((3, 2, 0, 1)))


def codeformer_tensor(bgr):
    """The training pipeline's image tensor of a uint8 BGR HWC image: img2tensor(img / 255., bgr2rgb=True) (float64
    division, float32 cast) and normalize(0.5, 0.5) -> [1,3,H,W] in [-1, 1]."""
    t = torch.from_numpy(np.ascontiguousarray((bgr / 255.).astype(np.float32)[:, :, ::-1])).permute(2, 0, 1)[None]
    return (t - 0.5) / 0.5


def input_tensor(bgr, convention):
    """The fp32 RGB tensor ``LPIPS.forward`` receives for a uint8 BGR image: 'lpips' im2tensor of the RGB image (forward
    with normalize=False), 'codeformer' the training tensor (LPIPSLoss(use_input_norm=True, range_norm=True) on it)."""
    if convention == 'lpips':
        return im2tensor(np.ascontiguousarray(bgr[:, :, ::-1]))
    if convention == 'codeformer':
        return codeformer_tensor(bgr)
    raise ValueError(convention)


def stem_input(bgr, convention):
    """What conv1_1 sees for a uint8 BGR image: the convention's tensor through its chain and the ScalingLayer."""
    x = input_tensor(bgr, convention)
    if convention == 'codeformer':
        x = (x + 1) / 2
        x = (x - torch.Tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)) / torch.Tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    return ScalingLayer()(x)


def u8_table(convention):
    """[3][256]: stem_input of every byte value, by RGB channel."""
    ramp = np.repeat(np.arange(256, dtype=np.uint8)[None, :, None], 3, axis=2)      # [1,256,3], every channel = u
    return stem_input(ramp, convention)[0, :, 0, :]


def distance_u8(lp, ref_bgr, cand_bgr, convention='lpips'):
    """LPIPS of two uint8 BGR HWC images in a convention (the value ``lpips_distance`` computes)."""
    a, b = input_tensor(ref_bgr, convention), input_tensor(cand_bgr, convention)
    if convention == 'codeformer':
        loss = LPIPSLoss(use_input_norm=True, range_norm=True)
        loss.perceptual = lp
        return loss(b, a)
    return lp(a, b).view(())
