"""torch fp32 restatement (CPU) of pytorch-fid's ``InceptionV3(output_blocks=[3], use_fid_inception=True)`` -- the FID network
BasicSR vendors as ``basicsr/archs/inception.py`` -- and the patched torchvision model it is defined by.

``reference_model(sd)`` builds torchvision's ``Inception3(num_classes=1008, aux_logits=False, init_weights=False)`` with the FID
blocks (the pool branches of InceptionA / C / E_1 are ``avg_pool2d(3, 1, 1, count_include_pad=False)``, that of E_2 is
``max_pool2d(3, 1, 1)``) in the wrapper's ``blocks`` layout.  ``forward(sd, x, ...)`` restates the same network op for op from
a state dict.  tests/test_oracle_fid.py holds the two bit for bit.
"""
from collections import OrderedDict

import torch
import torch.nn as nn
import torch.nn.functional as F
from torchvision.models import inception as tvi


class FIDInceptionA(tvi.InceptionA):
    def forward(self, x):
        b1 = self.branch1x1(x)
        b5 = self.branch5x5_2(self.branch5x5_1(x))
        b3 = self.branch3x3dbl_3(self.branch3x3dbl_2(self.branch3x3dbl_1(x)))
        bp = self.branch_pool(F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False))
        return torch.cat([b1, b5, b3, bp], 1)


class FIDInceptionC(tvi.InceptionC):
    def forward(self, x):
        b1 = self.branch1x1(x)
        b7 = self.branch7x7_3(self.branch7x7_2(self.branch7x7_1(x)))
        bd = x
        for m in (self.branch7x7dbl_1, self.branch7x7dbl_2, self.branch7x7dbl_3, self.branch7x7dbl_4, self.branch7x7dbl_5):
            bd = m(bd)
        bp = self.branch_pool(F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False))
        return torch.cat([b1, b7, bd, bp], 1)


class FIDInceptionE(tvi.InceptionE):
    def __init__(self, in_channels, max_pool):
        super().__init__(in_channels)
        self.max_pool = max_pool

    def forward(self, x):
        b1 = self.branch1x1(x)
        b3 = self.branch3x3_1(x)
        b3 = torch.cat([self.branch3x3_2a(b3), self.branch3x3_2b(b3)], 1)
        bd = self.branch3x3dbl_2(self.branch3x3dbl_1(x))
        bd = torch.cat([self.branch3x3dbl_3a(bd), self.branch3x3dbl_3b(bd)], 1)
        if self.max_pool:      # FIDInceptionE_2
            bp = F.max_pool2d(x, kernel_size=3, stride=1, padding=1)
        else:                  # FIDInceptionE_1
            bp = F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False)
        return torch.cat([b1, b3, bd, self.branch_pool(bp)], 1)


def torchvision_model():
    """torchvision's Inception3 with the FID blocks, torchvision names (the layout of the FID weight file)."""
    m = tvi.Inception3(num_classes=1008, aux_logits=False, init_weights=False)
    m.Mixed_5b = FIDInceptionA(192, pool_features=32)
    m.Mixed_5c = FIDInceptionA(256, pool_features=64)
    m.Mixed_5d = FIDInceptionA(288, pool_features=64)
    m.Mixed_6b = FIDInceptionC(768, channels_7x7=128)
    m.Mixed_6c = FIDInceptionC(768, channels_7x7=160)
    m.Mixed_6d = FIDInceptionC(768, channels_7x7=160)
    m.Mixed_6e = FIDInceptionC(768, channels_7x7=192)
    m.Mixed_7b = FIDInceptionE(1280, max_pool=False)
    m.Mixed_7c = FIDInceptionE(2048, max_pool=True)
    return m.eval()


class Wrapper(nn.Module):
    """pytorch-fid's InceptionV3 wrapper with output_blocks=[3]: ``blocks`` and forward -> [pool3]."""

    def __init__(self, net, resize_input=True, normalize_input=True):
        super().__init__()
        self.resize_input, self.normalize_input = resize_input, normalize_input
        self.blocks = nn.ModuleList([
            nn.Sequential(net.Conv2d_1a_3x3, net.Conv2d_2a_3x3, net.Conv2d_2b_3x3, nn.MaxPool2d(kernel_size=3, stride=2)),
            nn.Sequential(net.Conv2d_3b_1x1, net.Conv2d_4a_3x3, nn.MaxPool2d(kernel_size=3, stride=2)),
            nn.Sequential(net.Mixed_5b, net.Mixed_5c, net.Mixed_5d, net.Mixed_6a, net.Mixed_6b, net.Mixed_6c, net.Mixed_6d,
                          net.Mixed_6e),
            nn.Sequential(net.Mixed_7a, net.Mixed_7b, net.Mixed_7c, nn.AdaptiveAvgPool2d(output_size=(1, 1)))])

    def forward(self, x):
        if self.resize_input:
            x = F.interpolate(x, size=(299, 299), mode='bilinear', align_corners=False)
        if self.normalize_input:
            x = 2 * x - 1
        for block in self.blocks:
            x = block(x)
        return [x]


def reference_model(sd=None, resize_input=True, normalize_input=True):
    """The patched torchvision model in the wrapper's layout, loaded with the wrapper-named state dict ``sd`` (if given)."""
    m = Wrapper(torchvision_model(), resize_input, normalize_input).eval()
    if sd is not None:
        m.load_state_dict(sd)
    return m


def random_fid_state_dict(seed):
    """Seeded wrapper-named weights: He-normal convs and BatchNorm statistics near the identity, so that activations stay of
    order 1 through all 94 ReLU convs."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    for k, v in reference_model().state_dict().items():
        if k.endswith('num_batches_tracked'):
            sd[k] = torch.zeros((), dtype=torch.int64)
        elif k.endswith('conv.weight'):
            sd[k] = torch.randn(v.shape, generator=g) * (2.0 / (v.shape[1] * v.shape[2] * v.shape[3])) ** 0.5
        elif k.endswith('bn.weight'):
            sd[k] = 1 + 0.1 * torch.randn(v.shape, generator=g)
        elif k.endswith('bn.bias'):
            sd[k] = 0.1 * torch.randn(v.shape, generator=g)
        elif k.endswith('running_mean'):
            sd[k] = 0.1 * torch.randn(v.shape, generator=g)
        else:
            sd[k] = 0.5 + torch.rand(v.shape, generator=g)
    return sd


def torchvision_names(sd):
    """The wrapper-named dict renamed to torchvision's names (the FID weight file's layout), plus an fc layer to ignore."""
    tv = torchvision_model()
    wrapper = Wrapper(tv)
    ids = {id(m): name for name, m in tv.named_modules()}
    rename = {}
    for name, m in wrapper.named_modules():
        if id(m) in ids and ids[id(m)]:
            rename[name] = ids[id(m)]
    out = OrderedDict()
    for k, v in sd.items():
        mod, leaf = k.rsplit('.', 1)
        head = max((p for p in rename if mod == p or mod.startswith(p + '.')), key=len)
        out[rename[head] + mod[len(head):] + '.' + leaf] = v
    out['fc.weight'] = torch.zeros(1008, 2048)
    out['fc.bias'] = torch.zeros(1008)
    return out


# ---- the same network restated from the state dict ----
def _basic(sd, p, x, stride=1, padding=0):
    x = F.conv2d(x, sd[p + '.conv.weight'], None, stride, padding)
    x = F.batch_norm(x, sd[p + '.bn.running_mean'], sd[p + '.bn.running_var'], sd[p + '.bn.weight'], sd[p + '.bn.bias'],
                     False, 0.1, 0.001)
    return F.relu(x)


def _avg(x):
    return F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False)


def _block_a(sd, p, x):
    b1 = _basic(sd, p + '.branch1x1', x)
    b5 = _basic(sd, p + '.branch5x5_2', _basic(sd, p + '.branch5x5_1', x), padding=2)
    b3 = _basic(sd, p + '.branch3x3dbl_1', x)
    b3 = _basic(sd, p + '.branch3x3dbl_3', _basic(sd, p + '.branch3x3dbl_2', b3, padding=1), padding=1)
    return torch.cat([b1, b5, b3, _basic(sd, p + '.branch_pool', _avg(x))], 1)


def _block_b(sd, p, x):
    b3 = _basic(sd, p + '.branch3x3', x, stride=2)
    bd = _basic(sd, p + '.branch3x3dbl_2', _basic(sd, p + '.branch3x3dbl_1', x), padding=1)
    bd = _basic(sd, p + '.branch3x3dbl_3', bd, stride=2)
    return torch.cat([b3, bd, F.max_pool2d(x, kernel_size=3, stride=2)], 1)


def _block_c(sd, p, x):
    b1 = _basic(sd, p + '.branch1x1', x)
    b7 = _basic(sd, p + '.branch7x7_1', x)
    b7 = _basic(sd, p + '.branch7x7_2', b7, padding=(0, 3))
    b7 = _basic(sd, p + '.branch7x7_3', b7, padding=(3, 0))
    bd = _basic(sd, p + '.branch7x7dbl_1', x)
    for i, pad in ((2, (3, 0)), (3, (0, 3)), (4, (3, 0)), (5, (0, 3))):
        bd = _basic(sd, f'{p}.branch7x7dbl_{i}', bd, padding=pad)
    return torch.cat([b1, b7, bd, _basic(sd, p + '.branch_pool', _avg(x))], 1)


def _block_d(sd, p, x):
    b3 = _basic(sd, p + '.branch3x3_2', _basic(sd, p + '.branch3x3_1', x), stride=2)
    b7 = _basic(sd, p + '.branch7x7x3_1', x)
    b7 = _basic(sd, p + '.branch7x7x3_2', b7, padding=(0, 3))
    b7 = _basic(sd, p + '.branch7x7x3_3', b7, padding=(3, 0))
    b7 = _basic(sd, p + '.branch7x7x3_4', b7, stride=2)
    return torch.cat([b3, b7, F.max_pool2d(x, kernel_size=3, stride=2)], 1)


def _block_e(sd, p, x, max_pool):
    b1 = _basic(sd, p + '.branch1x1', x)
    b3 = _basic(sd, p + '.branch3x3_1', x)
    b3 = torch.cat([_basic(sd, p + '.branch3x3_2a', b3, padding=(0, 1)), _basic(sd, p + '.branch3x3_2b', b3, padding=(1, 0))], 1)
    bd = _basic(sd, p + '.branch3x3dbl_2', _basic(sd, p + '.branch3x3dbl_1', x), padding=1)
    bd = torch.cat([_basic(sd, p + '.branch3x3dbl_3a', bd, padding=(0, 1)), _basic(sd, p + '.branch3x3dbl_3b', bd, padding=(1, 0))], 1)
    pool = F.max_pool2d(x, kernel_size=3, stride=1, padding=1) if max_pool else _avg(x)
    return torch.cat([b1, b3, bd, _basic(sd, p + '.branch_pool', pool)], 1)


def input_stage(x, resize_input=True, normalize_input=True):
    if resize_input:
        x = F.interpolate(x, size=(299, 299), mode='bilinear', align_corners=False)
    if normalize_input:
        x = 2 * x - 1
    return x


def forward(sd, x, resize_input=True, normalize_input=True):
    """pool3 [B,2048,1,1] of fp32 NCHW x, op for op as the wrapper computes it."""
    x = input_stage(x, resize_input, normalize_input)
    x = _basic(sd, 'blocks.0.0', x, stride=2)
    x = _basic(sd, 'blocks.0.1', x)
    x = _basic(sd, 'blocks.0.2', x, padding=1)
    x = F.max_pool2d(x, kernel_size=3, stride=2)
    x = _basic(sd, 'blocks.1.0', x)
    x = _basic(sd, 'blocks.1.1', x)
    x = F.max_pool2d(x, kernel_size=3, stride=2)
    for i in range(3):
        x = _block_a(sd, f'blocks.2.{i}', x)
    x = _block_b(sd, 'blocks.2.3', x)
    for i in range(4, 8):
        x = _block_c(sd, f'blocks.2.{i}', x)
    x = _block_d(sd, 'blocks.3.0', x)
    x = _block_e(sd, 'blocks.3.1', x, False)
    x = _block_e(sd, 'blocks.3.2', x, True)
    return F.adaptive_avg_pool2d(x, (1, 1))


def u8_to_tensor(images_bgr):
    """uint8 HWC BGR [B,H,W,3] (numpy or tensor) -> fp32 NCHW RGB in [0, 1], as ToTensor computes it."""
    x = torch.as_tensor(images_bgr)
    return x.flip(-1).permute(0, 3, 1, 2).float().div(255)
