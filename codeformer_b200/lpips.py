"""LPIPS-VGG on libcfb200: the perceptual distance of restored faces, fidelity sweeps and whole images.

``LPIPS`` mirrors ``lpips.LPIPS(net='vgg', version='0.1', lpips=True, spatial=False)`` of the lpips 0.1 package, the
perceptual term of basicsr's ``LPIPSLoss`` (basicsr/losses/losses.py:257-282) that every CodeFormer training config uses: the
same ``state_dict`` (``scaling_layer``, ``net.slice1..5`` with torchvision's ``vgg16().features`` indices, ``lin0..4`` and
the same five weights again as ``lins.0..4``) and ``forward(in0, in1, retPerLayer, normalize)``.  ``LPIPSLoss`` is the
basicsr class, for evaluation.  ``lpips_distance`` scores uint8 faces, sweeps and lists of whole images, each reference's
features computed once however many candidates it has.

Semantics: ScalingLayer ``(x - shift) / scale``; VGG-16 relu1_2, relu2_2, relu3_3, relu4_3, relu5_3; per layer
``f / (sqrt(sum_c f^2) + 1e-10)`` of both images, ``(f0 - f1)^2``, the 1x1 ``lin_k`` and the mean over H x W; the value is
the sum over the layers.  Inference only, no CPU fallback; ``version='0.0'``, ``lpips=False``, ``spatial=True`` and the
AlexNet / SqueezeNet backbones are not built.
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .native import NativeNet

# torchvision vgg16().features: (index, cin, cout) of the 13 convs, and the conv count that ends each lpips slice
VGG16_CONVS = ((0, 3, 64), (2, 64, 64), (5, 64, 128), (7, 128, 128), (10, 128, 256), (12, 256, 256), (14, 256, 256),
               (17, 256, 512), (19, 512, 512), (21, 512, 512), (24, 512, 512), (26, 512, 512), (28, 512, 512))
SLICE_ENDS = (4, 9, 16, 23, 30)          # features[0:4], [4:9], [9:16], [16:23], [23:30]
CHANNELS = (64, 128, 256, 512, 512)      # relu1_2 .. relu5_3
SHIFT = (-.030, -.088, -.188)            # lpips ScalingLayer
SCALE = (.458, .448, .450)
CONVENTIONS = {'lpips': 0, 'codeformer': 1}
NORMALIZE, RANGE_NORM, INPUT_NORM = 1, 2, 4      # the fp32 input transforms (cfb_lpips_forward's xform)
WORKSPACE_BUDGET = 4 << 30               # bytes of workspace one launch may use; a single larger group still runs alone
DEFAULT_MAX_BATCH = 32                   # groups (one reference and its candidates) per launch


def _slice_of(index):
    return next(s for s, end in enumerate(SLICE_ENDS, 1) if index < end)


def lpips_spec():
    """state_dict keys -> (shape, dtype) of lpips.LPIPS(net='vgg', version='0.1'), in its order.  ``lins`` is a ModuleList
    over the ``lin0..4`` modules, so their weights are listed twice.  The lpips weight file ``weights/v0.1/vgg.pth`` holds
    the ``lin*`` keys only (lpips loads it with ``strict=False``)."""
    spec = OrderedDict()
    spec['scaling_layer.shift'] = ((1, 3, 1, 1), torch.float32)
    spec['scaling_layer.scale'] = ((1, 3, 1, 1), torch.float32)
    for idx, cin, cout in VGG16_CONVS:
        p = f'net.slice{_slice_of(idx)}.{idx}'
        spec[p + '.weight'] = ((cout, cin, 3, 3), torch.float32)
        spec[p + '.bias'] = ((cout,), torch.float32)
    for prefix in ('lin{}', 'lins.{}'):
        for k, c in enumerate(CHANNELS):
            spec[prefix.format(k) + '.model.1.weight'] = ((1, c, 1, 1), torch.float32)
    return spec


def _init(name, entry, g):
    """ScalingLayer constants; seeded He-normal conv weights with zero biases (torchvision's VGG initialisation) and
    non-negative lin weights.  Real weights come from load_vgg16_features and load_state_dict (or ``model_path``)."""
    shape, _ = entry
    if name.startswith('scaling_layer.'):
        return torch.tensor(SHIFT if name.endswith('shift') else SCALE, dtype=torch.float32).view(shape)
    if name.endswith('.bias'):
        return nn.Parameter(torch.zeros(shape), requires_grad=False)
    if name.startswith('lin'):
        return nn.Parameter(torch.rand(shape, generator=g) / shape[1], requires_grad=False)
    std = (2.0 / (shape[0] * 9)) ** 0.5
    return nn.Parameter(torch.randn(shape, generator=g) * std, requires_grad=False)


def _cuda(x, fn):
    if not (torch.is_tensor(x) and x.is_cuda):
        raise RuntimeError(f'{fn}: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
    return x


class LPIPS(NativeNet):
    """Parameter holder with lpips' ``state_dict`` and ``forward`` on the wgmma conv engine (fp32 parity: split-fp16
    operands).  conv1_1 and the head are SIMT kernels of the package (lpips.cu)."""

    def __init__(self, net='vgg', version='0.1', lpips=True, spatial=False, model_path=None):
        if net != 'vgg':
            raise NotImplementedError(f"codeformer_b200.LPIPS builds net='vgg' (got {net!r})")
        if version != '0.1':
            raise NotImplementedError(f"codeformer_b200.LPIPS builds version='0.1' (got {version!r})")
        if not lpips:
            raise NotImplementedError('codeformer_b200.LPIPS builds lpips=True (the learned linear layers)')
        if spatial:
            raise NotImplementedError('codeformer_b200.LPIPS builds spatial=False (no distance maps)')
        spec = OrderedDict((k, v) for k, v in lpips_spec().items() if not k.startswith('lins.'))
        super().__init__('lpips', (), spec, _init)
        self.lins = nn.ModuleList([getattr(self, f'lin{k}') for k in range(5)])
        self.pnet_type, self.version, self.lpips, self.spatial, self.L = net, version, True, False, 5
        object.__setattr__(self, 'last_launch_images', [])
        if model_path is not None:
            self.load_state_dict(torch.load(model_path, map_location='cpu'), strict=False)
        self.eval()

    def load_vgg16_features(self, sd):
        """Load a torchvision ``vgg16`` state dict (``features.<i>.weight`` / ``.bias``, e.g. ``vgg16-397923af.pth``) into
        ``net.slice*``; the classifier keys are ignored."""
        mapped = {}
        for idx, _, _ in VGG16_CONVS:
            for leaf in ('weight', 'bias'):
                mapped[f'net.slice{_slice_of(idx)}.{idx}.{leaf}'] = sd[f'features.{idx}.{leaf}']
        missing, unexpected = self.load_state_dict(mapped, strict=False)
        assert not unexpected
        return self

    def _workspace(self, batch, h, w, group, device):
        need = _lib.load().cfb_lpips_workspace_bytes(self._handle(), batch, h, w, group)
        if need < 0:
            _lib.check(1, 'cfb_lpips_workspace_bytes')
        if self._ws is None or self._ws.numel() < need or self._ws.device != device:
            object.__setattr__(self, '_ws', None)
            object.__setattr__(self, '_ws', torch.empty(int(need), dtype=torch.uint8, device=device))
        return self._ws

    def _groups_per_launch(self, B, G, H, W, max_batch):
        per_group = _lib.load().cfb_lpips_workspace_bytes(self._handle(), 1, H, W, G)
        if per_group < 0:
            _lib.check(1, 'cfb_lpips_workspace_bytes')
        return max(1, min(B, int(max_batch), WORKSPACE_BUDGET // max(int(per_group), 1)))

    def _launch(self, ref, cand, G, mode, u8, max_batch=DEFAULT_MAX_BATCH):
        """ref [B,...] and cand [B*G,...] (contiguous, one device) -> val [B*G], per-layer [B*G,5]; one launch per chunk of
        groups that stays under WORKSPACE_BUDGET."""
        lib = _lib.load()
        dev, B = ref.device, ref.shape[0]
        H, W = (ref.shape[1], ref.shape[2]) if u8 else (ref.shape[2], ref.shape[3])
        if H < 16 or W < 16:
            raise ValueError(f'LPIPS: images must be at least 16 x 16 (relu5_3 is at 1/16 of the input), got {H} x {W}')
        if int(max_batch) < 1:
            raise ValueError('LPIPS: max_batch must be >= 1')
        val = torch.empty(B * G, dtype=torch.float32, device=dev)
        layers = torch.empty((B * G, 5), dtype=torch.float32, device=dev)
        launches = []
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            if B:
                n = self._groups_per_launch(B, G, H, W, max_batch)
                fn = lib.cfb_lpips_forward_u8 if u8 else lib.cfb_lpips_forward
                for i in range(0, B, n):
                    m = min(n, B - i)
                    ws = self._workspace(m, H, W, G, dev)
                    _lib.check(fn(self._net, _lib.ptr(ref[i:i + m]), _lib.ptr(cand[i * G:(i + m) * G]), m, H, W, G, mode,
                                  _lib.ptr(val[i * G:]), _lib.ptr(layers[i * G:]), _lib.ptr(ws), ws.numel(), _lib.stream(dev)),
                               'cfb_lpips_forward')
                    launches.append(m * (1 + G))
        object.__setattr__(self, 'last_launch_images', launches)
        return val, layers

    def _check_f32(self, in0, in1, fn):
        for x in (in0, in1):
            _cuda(x, fn)
            if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != 3:
                raise RuntimeError(f'{fn}: expected float32 [N,3,H,W], got {x.dtype} {tuple(x.shape)}')
        if in0.shape != in1.shape or in0.device != in1.device:
            raise RuntimeError(f'{fn}: the two inputs differ in shape or device: {tuple(in0.shape)}, {tuple(in1.shape)}')

    def _pairs(self, in0, in1, mode):
        self._check_f32(in0, in1, 'LPIPS.forward')
        return self._launch(in0.contiguous(), in1.contiguous(), 1, mode, False)

    def forward(self, in0, in1, retPerLayer=False, normalize=False):
        """in0, in1: fp32 CUDA [N,3,H,W] RGB in [-1, 1] (in [0, 1] with ``normalize=True``) -> [N,1,1,1]; with
        ``retPerLayer`` also the list of the five layers' [N,1,1,1] values, as lpips returns them."""
        val, layers = self._pairs(in0, in1, NORMALIZE if normalize else 0)
        N = in0.shape[0]
        val = val.view(N, 1, 1, 1)
        if retPerLayer:
            return val, [layers[:, k].reshape(N, 1, 1, 1) for k in range(5)]
        return val

    def forward_u8(self, ref, cand, convention='lpips', max_batch=DEFAULT_MAX_BATCH):
        """ref: CUDA uint8 HWC BGR [B,H,W,3]; cand: [B,H,W,3] (one candidate each) or [B,K,H,W,3] (a sweep) -> float32 [B]
        or [B,K].  ``convention`` 'lpips' (lpips.im2tensor of the RGB image) or 'codeformer' (the training pipeline's
        tensors through LPIPSLoss(use_input_norm=True, range_norm=True)); equal to ``forward`` on those tensors bit for bit.
        Each reference's features are computed once."""
        fn = 'LPIPS.forward_u8'
        if convention not in CONVENTIONS:
            raise ValueError(f'{fn}: convention must be one of {sorted(CONVENTIONS)}, got {convention!r}')
        for x in (ref, cand):
            _cuda(x, fn)
            if x.dtype != torch.uint8:
                raise NotImplementedError(f'{fn}: only uint8 images are supported, got {x.dtype}')
        if (ref.dim() != 4 or ref.shape[-1] != 3 or cand.dim() not in (4, 5) or cand.shape[0] != ref.shape[0]
                or tuple(cand.shape[-3:]) != tuple(ref.shape[1:]) or cand.device != ref.device):
            raise RuntimeError(f'{fn}: expected ref [B,H,W,3] and cand [B,H,W,3] or [B,K,H,W,3] on one device, got '
                               f'{tuple(ref.shape)} and {tuple(cand.shape)}')
        B, sweep = ref.shape[0], cand.dim() == 5
        K = cand.shape[1] if sweep else 1
        cand = cand.reshape(B * K, *cand.shape[-3:]).contiguous()
        val, _ = self._launch(ref.contiguous(), cand, K, CONVENTIONS[convention], True, max_batch)
        return val.view(B, K) if sweep else val


class LPIPSLoss(nn.Module):
    """basicsr's LPIPSLoss (losses.py:257-282) for evaluation: ``forward(pred, target)`` = ``loss_weight`` * the mean LPIPS of
    (target, pred) after the optional ``range_norm`` ((x + 1) / 2) and ``use_input_norm`` (ImageNet mean / std).  There is no
    backward: with grad enabled, an input that requires grad raises instead of giving a loss without a gradient."""

    def __init__(self, loss_weight=1.0, use_input_norm=True, range_norm=False):
        super().__init__()
        self.perceptual = LPIPS(net='vgg', spatial=False).eval()
        self.loss_weight = loss_weight
        self.use_input_norm = use_input_norm
        self.range_norm = range_norm
        if self.use_input_norm:       # the constants the device chain applies (cfb_lpips_forward's input_norm)
            self.register_buffer('mean', torch.Tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1))
            self.register_buffer('std', torch.Tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1))

    def train(self, mode=True):
        if mode:
            raise RuntimeError('codeformer_b200.LPIPSLoss is evaluation-only (no backward); call .eval()')
        return super().train(False)

    def forward(self, pred, target):
        if torch.is_grad_enabled() and any(torch.is_tensor(x) and x.requires_grad for x in (pred, target)):
            raise RuntimeError('codeformer_b200.LPIPSLoss has no backward; evaluate it under torch.no_grad() or on inputs '
                               'that do not require grad')
        mode = (RANGE_NORM if self.range_norm else 0) | (INPUT_NORM if self.use_input_norm else 0)
        val, _ = self.perceptual._pairs(target, pred, mode)
        return self.loss_weight * val.view(-1, 1, 1, 1).mean()


def _device_u8(img, fn, device):
    """A uint8 numpy array or CUDA tensor -> CUDA tensor; other dtypes raise NotImplementedError."""
    if isinstance(img, np.ndarray):
        if img.dtype != np.uint8:
            raise NotImplementedError(f'{fn}: only uint8 images are supported, got {img.dtype}')
        return torch.from_numpy(np.ascontiguousarray(img)).to(device)
    if not torch.is_tensor(img):
        raise TypeError(f'{fn}: expected a numpy array or a CUDA tensor, got {type(img).__name__}')
    _cuda(img, fn)
    if img.dtype != torch.uint8:
        raise NotImplementedError(f'{fn}: only uint8 images are supported, got {img.dtype}')
    return img


def _lists(restored, reference, net, convention, max_batch):
    fn = 'lpips_distance'
    sweep = len(restored) > 0 and isinstance(restored[0], (list, tuple))
    rows = list(restored) if sweep else [restored]
    if not isinstance(reference, (list, tuple)) or any(len(r) != len(reference) for r in rows):
        raise ValueError(f'{fn}: restored must be a list of len(reference) images, or a list of such lists')
    dev = next((x.device for x in [*reference, *[y for r in rows for y in r]] if torch.is_tensor(x) and x.is_cuda),
               torch.device('cuda', torch.cuda.current_device()))
    refs = [_device_u8(g, fn, dev) for g in reference]
    out = torch.empty((len(rows), len(refs)), dtype=torch.float32, device=dev)
    groups = {}
    for i, g in enumerate(refs):
        if g.dim() != 3 or g.shape[-1] != 3:
            raise ValueError(f'{fn}: reference image {i} must be [H,W,3], got {tuple(g.shape)}')
        cands = []
        for k, row in enumerate(rows):
            r = _device_u8(row[i], fn, dev)
            if tuple(r.shape) != tuple(g.shape):
                raise ValueError(f'{fn}: restored image {i} has shape {tuple(r.shape)}, its reference {tuple(g.shape)}')
            cands.append(r)
        groups.setdefault(tuple(g.shape), []).append((i, g, cands))
    for members in groups.values():            # one call per shape; the references' K candidates form one group each
        ref = torch.stack([m[1] for m in members])
        cand = torch.stack([torch.stack(m[2]) for m in members])
        val = net.forward_u8(ref, cand, convention, max_batch)          # [n, K]
        idx = torch.tensor([m[0] for m in members], device=dev)
        out[:, idx] = val.t()
    return out if sweep else out[0]


def lpips_distance(restored, reference, net, convention='lpips', max_batch=DEFAULT_MAX_BATCH):
    """LPIPS of restored uint8 BGR images against their references, as float32 CUDA tensors:

    * ``restored`` [B,H,W,3] against ``reference`` [B,H,W,3]: [B];
    * a fidelity sweep ``restored`` [B,K,H,W,3] (``CodeFormer.forward_u8_sweep``) against ``reference`` [B,H,W,3]: [B,K],
      the shape ``identity_similarity`` and ``psnr_ssim`` return; each reference's features are computed once per face;
    * lists of HWC images of any sizes (``restore_images`` results): a list of N against a list of N references gives [N];
      a list of K such lists (``restore_images_sweep`` results, ``restored[k][i]``) gives [K,N].  Images of one shape are
      scored together, in launches that stay under ``WORKSPACE_BUDGET`` (a single larger pair runs alone).

    ``net`` is an ``LPIPS``; ``convention`` 'lpips' or 'codeformer' (``LPIPS.forward_u8``); ``max_batch`` bounds the
    references per launch.  Images are numpy arrays or CUDA tensors, uint8 only.  A value does not depend on the batch."""
    if isinstance(restored, (list, tuple)):
        return _lists(restored, reference, net, convention, max_batch)
    fn = 'lpips_distance'
    dev = restored.device if torch.is_tensor(restored) and restored.is_cuda else (
        reference.device if torch.is_tensor(reference) and reference.is_cuda else torch.device('cuda', torch.cuda.current_device()))
    a, b = _device_u8(restored, fn, dev), _device_u8(reference, fn, dev)
    if b.dim() != 4 or a.dim() not in (4, 5) or a.shape[0] != b.shape[0] or tuple(a.shape[-3:]) != tuple(b.shape[1:]):
        raise ValueError(f'{fn}: expected restored [B,H,W,3] or [B,K,H,W,3] and reference [B,H,W,3], got {tuple(a.shape)} and '
                         f'{tuple(b.shape)}')
    return net.forward_u8(b, a, convention, max_batch)
