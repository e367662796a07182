"""ResNetArcFace on libcfb200: identity embeddings of faces, to score restored faces and fidelity sweeps against their inputs.

Mirrors ``ResNetArcFace('IRBlock', layers, use_se=False)`` of /root/reference/basicsr/archs/arcface_arch.py:171-245 (the
identity network of basicsr/models/codeformer_model.py): same constructor and ``state_dict`` (181 entries for ``[2,2,2,2]``,
BatchNorm counters included, so a GFPGAN-style ``arcface_resnet18.pth`` loads strictly) and ``forward(x) -> [B,512]`` on the
gray 128 x 128 input.  ``forward_u8`` takes the uint8 BGR 512 x 512 faces themselves, with the caller's normalisation and
``gray_resize_for_identity`` (codeformer_model.py:131-135) fused.  ``identity_similarity`` scores restored faces, or a
sweep's candidates, against their inputs.  No CPU fallback; inference only.
"""
from collections import OrderedDict

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from .native import NativeNet
from .registry import ARCH_REGISTRY


def arcface_spec(layers=(2, 2, 2, 2)):
    """state_dict keys -> (shape, dtype) of the reference ResNetArcFace('IRBlock', layers, use_se=False), in registration order."""
    spec = OrderedDict()

    def bn(name, c):
        for k in ('weight', 'bias', 'running_mean', 'running_var'):
            spec[f'{name}.{k}'] = ((c,), torch.float32)
        spec[name + '.num_batches_tracked'] = ((), torch.int64)

    spec['conv1.weight'] = ((64, 1, 3, 3), torch.float32)
    bn('bn1', 64)
    spec['prelu.weight'] = ((1,), torch.float32)
    inplanes = 64
    for li, nb in enumerate(layers):
        planes = 64 << li
        for b in range(nb):
            p = f'layer{li + 1}.{b}'
            stride = 2 if (b == 0 and li > 0) else 1
            bn(p + '.bn0', inplanes)
            spec[p + '.conv1.weight'] = ((inplanes, inplanes, 3, 3), torch.float32)
            bn(p + '.bn1', inplanes)
            spec[p + '.prelu.weight'] = ((1,), torch.float32)
            spec[p + '.conv2.weight'] = ((planes, inplanes, 3, 3), torch.float32)
            bn(p + '.bn2', planes)
            if b == 0 and (stride != 1 or inplanes != planes):
                spec[p + '.downsample.0.weight'] = ((planes, inplanes, 1, 1), torch.float32)
                bn(p + '.downsample.1', planes)
            inplanes = planes
    bn('bn4', 512)
    spec['fc5.weight'] = ((512, 512 * 8 * 8), torch.float32)
    spec['fc5.bias'] = ((512,), torch.float32)
    bn('bn5', 512)
    return spec


def arcface_init(name, entry, g):
    """The reference's initialisation (arcface_arch.py:203-212): xavier-normal conv and linear weights, BatchNorm (1, 0) with
    running statistics (0, 1), linear bias 0; PReLU's default slope 0.25."""
    shape, dtype = entry
    leaf = name.rsplit('.', 1)[-1]
    if dtype == torch.int64:
        return torch.tensor(0, dtype=torch.long)
    if leaf in ('running_mean', 'running_var'):
        return torch.zeros(shape) if leaf == 'running_mean' else torch.ones(shape)
    if name.endswith('prelu.weight'):
        return nn.Parameter(torch.full(shape, 0.25))
    if len(shape) >= 2:
        rf = shape[2] * shape[3] if len(shape) == 4 else 1
        std = (2.0 / (shape[1] * rf + shape[0] * rf)) ** 0.5
        return nn.Parameter(torch.randn(shape, generator=g) * std)
    return nn.Parameter(torch.ones(shape) if leaf == 'weight' else torch.zeros(shape))


def random_arcface_state_dict(layers=(2, 2, 2, 2), seed=1):
    """Seeded parameters with activations of order 1 through the network (tests and benchmarks: no ArcFace checkpoint is
    needed): conv / linear weights N(0, 1/fan_in), BatchNorm gamma U(0.5, 1), beta and running_mean 0.1 N, running_var
    U(0.5, 1.5), PReLU slopes U(0.1, 0.3), fc5 bias 0.1 N."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    for name, (shape, dtype) in arcface_spec(layers).items():
        if dtype == torch.int64:
            t = torch.tensor(100, dtype=torch.int64)
        elif len(shape) >= 2:
            fan_in = 1
            for d in shape[1:]:
                fan_in *= d
            t = torch.randn(shape, generator=g) / fan_in ** 0.5
        elif name.endswith('prelu.weight'):
            t = 0.1 + 0.2 * torch.rand(shape, generator=g)
        elif name.endswith('running_var'):
            t = 0.5 + torch.rand(shape, generator=g)
        elif name.endswith('.weight'):
            t = 0.5 + 0.5 * torch.rand(shape, generator=g)
        else:
            t = 0.1 * torch.randn(shape, generator=g)
        sd[name] = t
    return sd


@ARCH_REGISTRY.register()
class ResNetArcFace(NativeNet):
    """Parameter holder with the reference's ``state_dict`` and ``forward`` on the wgmma conv engine (fp32 parity: split-fp16
    operands).  Only ``block='IRBlock'`` with ``use_se=False`` is built, the form of the checkpoints in use."""

    def __init__(self, block='IRBlock', layers=(2, 2, 2, 2), use_se=True):
        if block != 'IRBlock':
            raise NotImplementedError(f"codeformer_b200.ResNetArcFace builds block='IRBlock' (got {block!r})")
        if use_se:
            raise NotImplementedError('codeformer_b200.ResNetArcFace builds use_se=False (the SE blocks are not built)')
        layers = tuple(int(n) for n in layers)
        if len(layers) != 4 or min(layers) < 1:
            raise ValueError(f'ResNetArcFace: layers must be four block counts >= 1, got {layers}')
        super().__init__('arcface', layers, arcface_spec(layers), arcface_init)
        self.layers, self.use_se, self.inplanes = layers, False, 512
        self.eval()

    def _workspace(self, batch, device):
        need = _lib.load().cfb_arcface_workspace_bytes(self._handle(), batch)
        if need < 0:
            _lib.check(1, 'cfb_arcface_workspace_bytes')
        if self._ws is None or self._ws.numel() < need or self._ws.device != device:
            object.__setattr__(self, '_ws', None)
            object.__setattr__(self, '_ws', torch.empty(int(need), dtype=torch.uint8, device=device))
        return self._ws

    def _run(self, x, u8):
        lib = _lib.load()
        dev, B = x.device, x.shape[0]
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            emb = torch.empty((B, 512), dtype=torch.float32, device=dev)
            if B:
                ws = self._workspace(B, dev)
                fn = lib.cfb_arcface_forward_u8 if u8 else lib.cfb_arcface_forward
                _lib.check(fn(self._net, _lib.ptr(x), _lib.ptr(emb), B, _lib.ptr(ws), ws.numel(), _lib.stream(dev)),
                           'cfb_arcface_forward')
        return emb

    def forward(self, x):
        """x: fp32 CUDA [B,1,128,128] (the gray identity input) -> embeddings [B,512] (arcface_arch.py:229-245)."""
        if not (torch.is_tensor(x) and x.is_cuda):
            raise RuntimeError('ResNetArcFace.forward: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
        if x.dtype != torch.float32 or x.dim() != 4 or tuple(x.shape[1:]) != (1, 128, 128):
            raise RuntimeError(f'ResNetArcFace.forward: expected float32 [B,1,128,128], got {x.dtype} {tuple(x.shape)}')
        return self._run(x.contiguous(), False)

    def forward_u8(self, faces):
        """faces: CUDA uint8 HWC BGR [N,512,512,3] -> embeddings [N,512]: ``forward`` of the gray identity input the caller
        would build (img2tensor(face / 255.), normalize(0.5, 0.5), gray_resize_for_identity), bit for bit."""
        if not (torch.is_tensor(faces) and faces.is_cuda and faces.dtype == torch.uint8 and faces.dim() == 4
                and tuple(faces.shape[1:]) == (512, 512, 3)):
            raise RuntimeError('ResNetArcFace.forward_u8: expected a CUDA uint8 [N,512,512,3] tensor')
        return self._run(faces.contiguous(), True)


def identity_similarity(arcface, faces, restored, max_batch=64):
    """Cosine similarity of the ArcFace embeddings of restored faces to those of their inputs.

    ``faces``: CUDA uint8 [B,512,512,3] BGR (the cropped inputs); ``restored``: [B,512,512,3] (one restored face each) or a
    sweep's [B,K,512,512,3] (``CodeFormer.forward_u8_sweep``).  Returns float32 [B] or [B,K] on the device, equal to
    ``F.cosine_similarity`` of the embeddings.  The B + B*K faces go through ``arcface.forward_u8`` in chunks of at most
    ``max_batch``."""
    if not (torch.is_tensor(faces) and faces.dim() == 4 and tuple(faces.shape[1:]) == (512, 512, 3)):
        raise RuntimeError(f'identity_similarity: faces must be [B,512,512,3], got {tuple(getattr(faces, "shape", ()))}')
    if not (torch.is_tensor(restored) and restored.dim() in (4, 5) and tuple(restored.shape[-3:]) == (512, 512, 3)
            and restored.shape[0] == faces.shape[0]):
        raise RuntimeError('identity_similarity: restored must be [B,512,512,3] or [B,K,512,512,3] with the B of faces, got '
                           f'{tuple(getattr(restored, "shape", ()))}')
    if int(max_batch) < 1:
        raise ValueError('identity_similarity: max_batch must be >= 1')
    B = faces.shape[0]
    K = restored.shape[1] if restored.dim() == 5 else 1
    flat = restored.reshape(B * K, 512, 512, 3)
    total, mb = B + B * K, int(max_batch)
    emb = torch.empty((total, 512), dtype=torch.float32, device=faces.device)
    for i in range(0, total, mb):          # one batch over [faces; restored], chunked
        j = min(total, i + mb)
        parts = []
        if i < B:
            parts.append(faces[i:min(j, B)])
        if j > B:
            parts.append(flat[max(i, B) - B:j - B])
        chunk = parts[0] if len(parts) == 1 else torch.cat(parts)
        emb[i:j] = arcface.forward_u8(chunk)
    e_in, e_out = emb[:B], emb[B:].view(B, K, 512)
    sims = torch.stack([F.cosine_similarity(e_out[:, k].contiguous(), e_in, dim=-1) for k in range(K)], dim=1)
    return sims if restored.dim() == 5 else sims[:, 0]
