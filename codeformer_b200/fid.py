"""Fréchet Inception Distance on libcfb200: the FID Inception-v3 on the conv engine, for restored faces, fidelity sweeps and
whole images.

``InceptionV3`` mirrors pytorch-fid's ``InceptionV3(output_blocks=[3], use_fid_inception=True)``, which BasicSR vendors as
``basicsr/archs/inception.py``: the same wrapper state dict (``blocks.0.0.conv.weight``, ..., BatchNorm buffers included) and
``forward(x)`` -> ``[pool3]`` with the ``resize_input`` / ``normalize_input`` flags.  ``load_fid_inception_weights`` maps the
torchvision-named FID weight file (``pt_inception-2015-12-05-6726825d.pth``) into it.

Statistics and distance follow pytorch-fid / BasicSR: ``fid_statistics`` is the mean and ``np.cov(features, rowvar=False)`` of
the float32 pool3 features, computed in float64 on the device; ``frechet_distance`` evaluates
``|mu_a - mu_b|^2 + tr(sigma_a) + tr(sigma_b) - 2 tr(sqrtm(sigma_a sigma_b))`` on the device, the trace term as the sum of
``sqrt(max(lambda, 0))`` over the eigenvalues of ``sigma_a^1/2 sigma_b sigma_a^1/2``; ``calculate_fid`` is BasicSR's host
formula with scipy.  Inference only, pool3 only, no CPU fallback.
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .native import NativeNet

FEATURES = 2048
DEFAULT_MAX_BATCH = 32

# torchvision Inception3 module -> the wrapper's block prefix
TORCHVISION_BLOCKS = OrderedDict([
    ('Conv2d_1a_3x3', 'blocks.0.0'), ('Conv2d_2a_3x3', 'blocks.0.1'), ('Conv2d_2b_3x3', 'blocks.0.2'),
    ('Conv2d_3b_1x1', 'blocks.1.0'), ('Conv2d_4a_3x3', 'blocks.1.1'),
    ('Mixed_5b', 'blocks.2.0'), ('Mixed_5c', 'blocks.2.1'), ('Mixed_5d', 'blocks.2.2'), ('Mixed_6a', 'blocks.2.3'),
    ('Mixed_6b', 'blocks.2.4'), ('Mixed_6c', 'blocks.2.5'), ('Mixed_6d', 'blocks.2.6'), ('Mixed_6e', 'blocks.2.7'),
    ('Mixed_7a', 'blocks.3.0'), ('Mixed_7b', 'blocks.3.1'), ('Mixed_7c', 'blocks.3.2')])


def _block_convs(kind, cin, arg=None):
    """(branch name, cin, cout, kh, kw) of torchvision's Inception blocks, in registration order."""
    if kind == 'A':
        return [('branch1x1', cin, 64, 1, 1), ('branch5x5_1', cin, 48, 1, 1), ('branch5x5_2', 48, 64, 5, 5),
                ('branch3x3dbl_1', cin, 64, 1, 1), ('branch3x3dbl_2', 64, 96, 3, 3), ('branch3x3dbl_3', 96, 96, 3, 3),
                ('branch_pool', cin, arg, 1, 1)]
    if kind == 'B':
        return [('branch3x3', cin, 384, 3, 3), ('branch3x3dbl_1', cin, 64, 1, 1), ('branch3x3dbl_2', 64, 96, 3, 3),
                ('branch3x3dbl_3', 96, 96, 3, 3)]
    if kind == 'C':
        c7 = arg
        return [('branch1x1', cin, 192, 1, 1), ('branch7x7_1', cin, c7, 1, 1), ('branch7x7_2', c7, c7, 1, 7),
                ('branch7x7_3', c7, 192, 7, 1), ('branch7x7dbl_1', cin, c7, 1, 1), ('branch7x7dbl_2', c7, c7, 7, 1),
                ('branch7x7dbl_3', c7, c7, 1, 7), ('branch7x7dbl_4', c7, c7, 7, 1), ('branch7x7dbl_5', c7, 192, 1, 7),
                ('branch_pool', cin, 192, 1, 1)]
    if kind == 'D':
        return [('branch3x3_1', cin, 192, 1, 1), ('branch3x3_2', 192, 320, 3, 3), ('branch7x7x3_1', cin, 192, 1, 1),
                ('branch7x7x3_2', 192, 192, 1, 7), ('branch7x7x3_3', 192, 192, 7, 1), ('branch7x7x3_4', 192, 192, 3, 3)]
    return [('branch1x1', cin, 320, 1, 1), ('branch3x3_1', cin, 384, 1, 1), ('branch3x3_2a', 384, 384, 1, 3),
            ('branch3x3_2b', 384, 384, 3, 1), ('branch3x3dbl_1', cin, 448, 1, 1), ('branch3x3dbl_2', 448, 384, 3, 3),
            ('branch3x3dbl_3a', 384, 384, 1, 3), ('branch3x3dbl_3b', 384, 384, 3, 1), ('branch_pool', cin, 192, 1, 1)]


def inception_convs():
    """(torchvision module path, wrapper prefix, cin, cout, kh, kw) of the 94 BasicConv2d, in the wrapper's order."""
    out = [('Conv2d_1a_3x3', 'blocks.0.0', 3, 32, 3, 3), ('Conv2d_2a_3x3', 'blocks.0.1', 32, 32, 3, 3),
           ('Conv2d_2b_3x3', 'blocks.0.2', 32, 64, 3, 3), ('Conv2d_3b_1x1', 'blocks.1.0', 64, 80, 1, 1),
           ('Conv2d_4a_3x3', 'blocks.1.1', 80, 192, 3, 3)]
    plan = [('Mixed_5b', 'A', 192, 32), ('Mixed_5c', 'A', 256, 64), ('Mixed_5d', 'A', 288, 64), ('Mixed_6a', 'B', 288, None),
            ('Mixed_6b', 'C', 768, 128), ('Mixed_6c', 'C', 768, 160), ('Mixed_6d', 'C', 768, 160), ('Mixed_6e', 'C', 768, 192),
            ('Mixed_7a', 'D', 768, None), ('Mixed_7b', 'E', 1280, None), ('Mixed_7c', 'E', 2048, None)]
    for name, kind, cin, arg in plan:
        for br, ci, co, kh, kw in _block_convs(kind, cin, arg):
            out.append((f'{name}.{br}', f'{TORCHVISION_BLOCKS[name]}.{br}', ci, co, kh, kw))
    return out


def fid_inception_spec():
    """state_dict keys -> (shape, dtype) of pytorch-fid's InceptionV3(output_blocks=[3]), in its order."""
    spec = OrderedDict()
    for _, p, cin, cout, kh, kw in inception_convs():
        spec[p + '.conv.weight'] = ((cout, cin, kh, kw), torch.float32)
        for leaf in ('weight', 'bias', 'running_mean', 'running_var'):
            spec[f'{p}.bn.{leaf}'] = ((cout,), torch.float32)
        spec[p + '.bn.num_batches_tracked'] = ((), torch.int64)
    return spec


def _init(name, entry, g):
    """Placeholder weights until load_fid_inception_weights (or ``model_path``): seeded He-normal convs and nn.BatchNorm2d's
    initial state (weight 1, bias 0, running mean 0, running var 1)."""
    shape, dtype = entry
    if dtype == torch.int64:
        return torch.zeros(shape, dtype=torch.int64)
    if name.endswith('conv.weight'):
        fan_in = shape[1] * shape[2] * shape[3]
        return nn.Parameter(torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5, requires_grad=False)
    if name.endswith('bn.weight'):
        return nn.Parameter(torch.ones(shape), requires_grad=False)
    if name.endswith('bn.bias'):
        return nn.Parameter(torch.zeros(shape), requires_grad=False)
    if name.endswith('running_mean'):
        return torch.zeros(shape)
    return torch.ones(shape)


def _cuda(x, fn):
    if not (torch.is_tensor(x) and x.is_cuda):
        raise RuntimeError(f'{fn}: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
    return x


class InceptionV3(NativeNet):
    """pytorch-fid's InceptionV3 for FID (pool3 features) on the wgmma conv engine, fp32 parity (split-fp16 operands).  The
    input stage, Conv2d_1a, the pools and the statistics are SIMT kernels of the package (fid.cu)."""

    def __init__(self, output_blocks=(3,), resize_input=True, normalize_input=True, requires_grad=False,
                 use_fid_inception=True, model_path=None):
        if sorted(output_blocks) != [3]:
            raise NotImplementedError(f'codeformer_b200.InceptionV3 builds output_blocks=[3] (pool3) only, got {output_blocks}')
        if not use_fid_inception:
            raise NotImplementedError('codeformer_b200.InceptionV3 builds the FID Inception (use_fid_inception=True) only')
        if requires_grad:
            raise NotImplementedError('codeformer_b200.InceptionV3 is inference-only (requires_grad=False)')
        super().__init__('fid', (), fid_inception_spec(), _init)
        self.resize_input, self.normalize_input = bool(resize_input), bool(normalize_input)
        self.output_blocks, self.last_needed_block = [3], 3
        if model_path is not None:
            self.load_fid_inception_weights(torch.load(model_path, map_location='cpu'))
        self.eval()

    def load_fid_inception_weights(self, sd):
        """Load a torchvision-named FID Inception state dict (``Conv2d_1a_3x3.conv.weight``, ``Mixed_5b.branch1x1.bn.*``, ...;
        ``pt_inception-2015-12-05-6726825d.pth``); ``fc.*`` is ignored."""
        mapped = {}
        for tv, p, *_ in inception_convs():
            for leaf in ('conv.weight', 'bn.weight', 'bn.bias', 'bn.running_mean', 'bn.running_var', 'bn.num_batches_tracked'):
                if f'{tv}.{leaf}' in sd:
                    mapped[f'{p}.{leaf}'] = sd[f'{tv}.{leaf}']
        missing, unexpected = self.load_state_dict(mapped, strict=False)
        missing = [k for k in missing if not k.endswith('num_batches_tracked')]
        if missing or unexpected:
            raise KeyError(f'load_fid_inception_weights: missing {missing[:4]}, unexpected {unexpected[:4]}')
        return self

    def _workspace(self, batch, h, w, device, resize=True):
        need = _lib.load().cfb_fid_workspace_bytes(self._handle(), batch, h, w, int(resize))
        if need < 0:
            _lib.check(1, 'cfb_fid_workspace_bytes')
        if self._ws is None or self._ws.numel() < need or self._ws.device != device:
            object.__setattr__(self, '_ws', None)
            object.__setattr__(self, '_ws', torch.empty(int(need), dtype=torch.uint8, device=device))
        return self._ws

    def _run(self, x, u8, resize, normalize, max_batch):
        """x: contiguous CUDA fp32 [B,3,H,W] or uint8 [B,H,W,3] -> [B,2048] float32, launches of at most max_batch images."""
        if int(max_batch) < 1:
            raise ValueError('InceptionV3: max_batch must be >= 1')
        lib, dev, B = _lib.load(), x.device, x.shape[0]
        H, W = (x.shape[1], x.shape[2]) if u8 else (x.shape[2], x.shape[3])
        if not resize and (H < 75 or W < 75):
            raise ValueError(f'InceptionV3: without resize_input the images must be at least 75 x 75, got {H} x {W}')
        feat = torch.empty((B, FEATURES), dtype=torch.float32, device=dev)
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            for i in range(0, B, int(max_batch)):
                m = min(int(max_batch), B - i)
                ws = self._workspace(m, H, W, dev, resize)
                if u8:
                    st = lib.cfb_fid_forward_u8(self._net, _lib.ptr(x[i:i + m]), m, H, W, _lib.ptr(feat[i:]), _lib.ptr(ws),
                                                ws.numel(), _lib.stream(dev))
                else:
                    st = lib.cfb_fid_forward(self._net, _lib.ptr(x[i:i + m]), m, H, W, int(resize), int(normalize),
                                             _lib.ptr(feat[i:]), _lib.ptr(ws), ws.numel(), _lib.stream(dev))
                _lib.check(st, 'cfb_fid_forward')
        return feat

    def forward(self, x, max_batch=DEFAULT_MAX_BATCH):
        """x: fp32 CUDA [B,3,H,W] RGB (in [0, 1] with normalize_input, in [-1, 1] without) -> [pool3 [B,2048,1,1]].  An image
        with a NaN in a value the first conv reads gets NaN features, as in torch."""
        _cuda(x, 'InceptionV3.forward')
        if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != 3:
            raise RuntimeError(f'InceptionV3.forward: expected float32 [B,3,H,W], got {x.dtype} {tuple(x.shape)}')
        feat = self._run(x.contiguous(), False, self.resize_input, self.normalize_input, max_batch)
        return [feat.view(-1, FEATURES, 1, 1)]

    def forward_u8(self, images, max_batch=DEFAULT_MAX_BATCH):
        """images: CUDA uint8 HWC BGR [B,H,W,3] -> [B,2048] float32: pytorch-fid's path for image files (RGB, ToTensor's v / 255,
        resize to 299, 2x - 1) fused into the first conv; equal to ``cfb_fid_input`` then ``forward`` with both flags off."""
        _cuda(images, 'InceptionV3.forward_u8')
        if images.dtype != torch.uint8:
            raise NotImplementedError(f'InceptionV3.forward_u8: only uint8 images are supported, got {images.dtype}')
        if images.dim() != 4 or images.shape[-1] != 3:
            raise RuntimeError(f'InceptionV3.forward_u8: expected [B,H,W,3], got {tuple(images.shape)}')
        return self._run(images.contiguous(), True, True, True, max_batch)


def fid_input(x, resize=True, normalize=True):
    """The input stage alone: fp32 CUDA [B,3,H,W] or uint8 CUDA HWC BGR [B,H,W,3] -> fp32 [B,3,299,299] (resize) or [B,3,H,W]."""
    _cuda(x, 'fid_input')
    u8 = x.dtype == torch.uint8
    if not (u8 and x.dim() == 4 and x.shape[-1] == 3) and not (x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3):
        raise RuntimeError(f'fid_input: expected uint8 [B,H,W,3] or float32 [B,3,H,W], got {x.dtype} {tuple(x.shape)}')
    x = x.contiguous()
    B, H, W = (x.shape[0], x.shape[1], x.shape[2]) if u8 else (x.shape[0], x.shape[2], x.shape[3])
    oh, ow = (299, 299) if resize else (H, W)
    out = torch.empty((B, 3, oh, ow), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().cfb_fid_input(_lib.ptr(x), int(u8), B, H, W, int(resize), int(normalize), _lib.ptr(out),
                                             _lib.stream(x.device)), 'cfb_fid_input')
    return out


def _device_u8(img, fn, device):
    if isinstance(img, np.ndarray):
        if img.dtype != np.uint8:
            raise NotImplementedError(f'{fn}: only uint8 images are supported, got {img.dtype}')
        return torch.from_numpy(np.ascontiguousarray(img)).to(device)
    if not torch.is_tensor(img):
        raise TypeError(f'{fn}: expected a numpy array or a tensor, got {type(img).__name__}')
    if img.dtype != torch.uint8:
        raise NotImplementedError(f'{fn}: only uint8 images are supported, got {img.dtype}')
    return img.to(device)


def _default_device(*xs):
    for x in xs:
        if torch.is_tensor(x) and x.is_cuda:
            return x.device
    return torch.device('cuda', torch.cuda.current_device())


def inception_features(images, net, max_batch=DEFAULT_MAX_BATCH):
    """pool3 features (float32, on the device) of uint8 HWC BGR images through ``net.forward_u8``:

    * faces [B,H,W,3] (numpy, host or CUDA tensor): [B,2048];
    * a fidelity sweep [B,K,H,W,3] (``CodeFormer.forward_u8_sweep``): [K,B,2048], one feature set per weight;
    * a list of HWC images of any sizes (``restore_images`` results): [N,2048] in list order; images of one size share
      launches.

    A feature vector does not depend on the batch it was computed in."""
    fn = 'inception_features'
    if isinstance(images, (list, tuple)):
        dev = _default_device(*images)
        imgs = [_device_u8(x, fn, dev) for x in images]
        out = torch.empty((len(imgs), FEATURES), dtype=torch.float32, device=dev)
        groups = OrderedDict()
        for i, x in enumerate(imgs):
            if x.dim() != 3 or x.shape[-1] != 3:
                raise ValueError(f'{fn}: image {i} must be [H,W,3], got {tuple(x.shape)}')
            groups.setdefault(tuple(x.shape), []).append(i)
        for idx in groups.values():
            feat = net.forward_u8(torch.stack([imgs[i] for i in idx]), max_batch)
            out[torch.tensor(idx, device=dev)] = feat
        return out
    x = _device_u8(images, fn, _default_device(images))
    if x.dim() == 4 and x.shape[-1] == 3:
        return net.forward_u8(x, max_batch)
    if x.dim() == 5 and x.shape[-1] == 3:
        B, K = x.shape[0], x.shape[1]
        feat = net.forward_u8(x.transpose(0, 1).reshape(K * B, *x.shape[2:]), max_batch)
        return feat.view(K, B, FEATURES)
    raise ValueError(f'{fn}: expected [B,H,W,3], [B,K,H,W,3] or a list of [H,W,3] images, got {tuple(x.shape)}')


def fid_statistics(features):
    """(mu [D], sigma [D,D]) in float64 on the device: the mean and ``np.cov(features, rowvar=False)`` of float32 CUDA features
    [N,D] (N >= 2, D a multiple of 64).  Every sum runs over the rows in order: the result depends only on the matrix."""
    fn = 'fid_statistics'
    _cuda(features, fn)
    if features.dtype != torch.float32 or features.dim() != 2:
        raise RuntimeError(f'{fn}: expected float32 [N,D], got {features.dtype} {tuple(features.shape)}')
    N, D = features.shape
    if N < 2:
        raise ValueError(f'{fn}: at least 2 feature vectors are needed for a covariance, got {N}')
    if D % 64 != 0 or D == 0:
        raise ValueError(f'{fn}: the feature width must be a multiple of 64, got {D}')
    x = features.contiguous()
    if x.data_ptr() % 16:          # the kernels read rows as float4
        x = x.clone()
    mu = torch.empty(D, dtype=torch.float64, device=x.device)
    sigma = torch.empty((D, D), dtype=torch.float64, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().cfb_fid_stats(_lib.ptr(x), N, D, _lib.ptr(mu), _lib.ptr(sigma), _lib.stream(x.device)),
                   'cfb_fid_stats')
    return mu, sigma


def _stats_on(stats, device, fn):
    mu, sigma = stats
    mu = torch.as_tensor(mu, dtype=torch.float64).to(device)
    sigma = torch.as_tensor(sigma, dtype=torch.float64).to(device)
    if mu.dim() != 1 or sigma.shape != (mu.shape[0], mu.shape[0]):
        raise ValueError(f'{fn}: expected mu [D] and sigma [D,D], got {tuple(mu.shape)} and {tuple(sigma.shape)}')
    return mu, sigma


def frechet_distance(stats_a, stats_b):
    """FID of two (mu, sigma) pairs (numpy arrays or tensors), in float64 on the device:
    ``|mu_a - mu_b|^2 + tr(sigma_a) + tr(sigma_b) - 2 sum sqrt(max(lambda, 0))`` over the eigenvalues lambda of
    ``sigma_a^1/2 sigma_b sigma_a^1/2`` (the eigenvalues of sigma_a sigma_b, so the sum is tr(sqrtm(sigma_a sigma_b)));
    sigma_a^1/2 comes from ``torch.linalg.eigh`` with negative eigenvalues clamped to 0.  Returns a Python float."""
    fn = 'frechet_distance'
    dev = _default_device(*stats_a, *stats_b)
    mu1, s1 = _stats_on(stats_a, dev, fn)
    mu2, s2 = _stats_on(stats_b, dev, fn)
    if mu1.shape != mu2.shape:
        raise ValueError(f'{fn}: the statistics have different widths, {mu1.shape[0]} and {mu2.shape[0]}')
    w, v = torch.linalg.eigh(s1)
    r = (v * w.clamp_min(0).sqrt()) @ v.T
    m = r @ s2 @ r
    lam = torch.linalg.eigvalsh((m + m.T) * 0.5)
    diff = mu1 - mu2
    return float(diff.dot(diff) + torch.trace(s1) + torch.trace(s2) - 2 * lam.clamp_min(0).sqrt().sum())


def _sqrtm(a):
    from scipy import linalg
    try:
        return linalg.sqrtm(a, disp=False)[0]
    except TypeError:             # scipy releases without the disp argument
        return linalg.sqrtm(a)


def calculate_fid(mu1, sigma1, mu2, sigma2, eps=1e-6):
    """BasicSR's calculate_fid (basicsr/metrics/fid.py) on the host with scipy: the drop-in, and the reference of
    ``frechet_distance``.  A non-finite sqrtm retries with eps * I added to both covariances; an imaginary diagonal beyond 1e-3
    raises ValueError."""
    mu1, mu2 = np.atleast_1d(mu1), np.atleast_1d(mu2)
    sigma1, sigma2 = np.atleast_2d(sigma1), np.atleast_2d(sigma2)
    assert mu1.shape == mu2.shape, 'Two mean vectors have different lengths'
    assert sigma1.shape == sigma2.shape, 'Two covariances have different dimensions'
    diff = mu1 - mu2
    covmean = _sqrtm(sigma1.dot(sigma2))
    if not np.isfinite(covmean).all():
        print(f'Product of cov matrices is singular. Adding {eps} to diagonal of cov estimates')
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = _sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            m = np.max(np.abs(covmean.imag))
            raise ValueError(f'Imaginary component {m}')
        covmean = covmean.real
    return diff @ diff + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean)


def fid_scores(candidates, reference_stats, net, max_batch=DEFAULT_MAX_BATCH):
    """FID of restored sets against reference statistics (mu, sigma), e.g. of the ground-truth faces or a published
    ``inception_FFHQ_512`` file:

    * a fidelity sweep [B,K,H,W,3]: float64 [K], one FID per weight;
    * a list of K lists of images (``restore_images_sweep`` results, ``candidates[k][i]``): [K];
    * one set, [B,H,W,3] or a list of images: float64 [1]."""
    if isinstance(candidates, (list, tuple)) and len(candidates) and isinstance(candidates[0], (list, tuple)):
        feats = [inception_features(list(c), net, max_batch) for c in candidates]
    else:
        f = inception_features(candidates, net, max_batch)
        feats = list(f) if f.dim() == 3 else [f]
    return torch.tensor([frechet_distance(fid_statistics(f), reference_stats) for f in feats], dtype=torch.float64)
