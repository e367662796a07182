"""ParseNet on libcfb200 (SURVEY.md section 8 row f3): the face-parsing network of the paste-back step.

Mirrors ``ParseNet`` of /root/reference/facelib/parsing/parsenet.py:140-194 as built by ``init_parsing_model('parsenet')``
(/root/reference/facelib/parsing/__init__.py:13: ``ParseNet(in_size=512, out_size=512, parsing_ch=19)``) and used by
``FaceRestoreHelper.paste_faces_to_input_image`` (/root/reference/facelib/utils/face_restoration_helper.py:457-487): same
constructor, same ``state_dict`` (238 entries incl. the BatchNorm buffers -- a reference checkpoint loads strictly), same
``forward(x) -> (out_mask, out_img)``.  The arithmetic is ``cfb_parsenet_forward`` (CUDA); eval-mode BatchNorm is folded into
the conv weights when the native copy is prepared.  ``face_parse_mask`` is the caller's step right after the network
(argmax over the 19 classes + MASK_COLORMAP) on the device.  No CPU fallback; inference only (BatchNorm uses running stats).
"""
import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .native import NativeNet, Precision


def parsenet_plan(in_size=512, out_size=512, min_feat_size=32, base_ch=64, res_depth=10, ch_range=(32, 256)):
    """(prefix, kind, cin, cout) of every ResidualBlock in registration order (parsenet.py:151-181); kind none/down/up."""
    min_ch, max_ch = ch_range
    clip = lambda x: max(min_ch, min(x, max_ch))      # noqa: E731
    min_feat_size = min(in_size, min_feat_size)
    down_steps = int(np.log2(in_size // min_feat_size))
    up_steps = int(np.log2(out_size // min_feat_size))
    plan, head = [], base_ch
    for i in range(down_steps):
        plan.append((f'encoder.{i + 1}', 'down', clip(head), clip(head * 2)))
        head *= 2
    for i in range(res_depth):
        plan.append((f'body.{i}', 'none', clip(head), clip(head)))
    for i in range(up_steps):
        plan.append((f'decoder.{i}', 'up', clip(head), clip(head // 2)))
        head //= 2
    return plan, clip(head)


def parsenet_spec(in_size=512, out_size=512, min_feat_size=32, base_ch=64, parsing_ch=19, res_depth=10, ch_range=(32, 256)):
    """state_dict keys -> (shape, dtype) of the reference ParseNet, in registration order."""
    from collections import OrderedDict
    spec = OrderedDict()

    def conv(p, cin, cout, bias):
        spec[p + '.conv2d.weight'] = ((cout, cin, 3, 3), torch.float32)
        if bias:
            spec[p + '.conv2d.bias'] = ((cout,), torch.float32)

    def bn(p, c):
        for k in ('weight', 'bias', 'running_mean', 'running_var'):
            spec[f'{p}.norm.norm.{k}'] = ((c,), torch.float32)
        spec[f'{p}.norm.norm.num_batches_tracked'] = ((), torch.int64)

    plan, head = parsenet_plan(in_size, out_size, min_feat_size, base_ch, res_depth, ch_range)
    conv('encoder.0', 3, base_ch, True)
    for prefix, kind, cin, cout in plan:
        if kind != 'none' or cin != cout:
            conv(prefix + '.shortcut_func', cin, cout, True)
        conv(prefix + '.conv1', cin, cout, False)
        bn(prefix + '.conv1', cout)
        conv(prefix + '.conv2', cout, cout, False)
        bn(prefix + '.conv2', cout)
    conv('out_img_conv', head, 3, True)
    conv('out_mask_conv', head, parsing_ch, True)
    return spec


def random_parsenet_state_dict(spec, seed=1):
    """Seeded parameters that exercise every term: filters U(+-1/sqrt(fan_in)), BatchNorm weight 1+0.1N, bias / running_mean
    0.1N, running_var U(0.5, 1.5)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, (shape, dtype) in spec.items():
        if dtype == torch.int64:
            t = torch.tensor(100, dtype=torch.int64)
        elif len(shape) == 4:
            fan_in = shape[1] * shape[2] * shape[3]
            t = (torch.rand(shape, generator=g) * 2 - 1) / fan_in ** 0.5
        elif name.endswith('running_var'):
            t = 0.5 + torch.rand(shape, generator=g)
        elif name.endswith('norm.weight'):
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        else:
            t = 0.1 * torch.randn(shape, generator=g)
        sd[name] = t
    return sd


def _parsenet_init(name, entry, g):
    """The reference's default initialisation: BatchNorm (1, 0) with running stats (0, 1), filters U(+-1/sqrt(fan_in)),
    conv biases 0."""
    shape, dtype = entry
    leaf = name.rsplit('.', 1)[-1]
    if dtype == torch.int64:
        return torch.tensor(0, dtype=torch.long)
    if leaf in ('running_mean', 'running_var'):
        return torch.zeros(shape) if leaf == 'running_mean' else torch.ones(shape)
    if len(shape) == 4:
        fan_in = shape[1] * shape[2] * shape[3]
        return nn.Parameter((torch.rand(shape, generator=g) * 2 - 1) / fan_in ** 0.5)
    return nn.Parameter(torch.ones(shape) if name.endswith('norm.weight') else torch.zeros(shape))


class ParseNet(Precision, NativeNet):
    """Parameter holder with the reference's ``state_dict`` + ``forward`` on the wgmma conv engine.  ``set_precision('fp16')``
    covers the shortcut, conv1 and conv2 of every encoder, body and decoder block; encoder.0 and the two heads stay fp32 in
    both precisions."""

    def __init__(self, in_size=128, out_size=128, min_feat_size=32, base_ch=64, parsing_ch=19, res_depth=10,
                 relu_type='LeakyReLU', norm_type='bn', ch_range=[32, 256]):
        if relu_type.lower() != 'leakyrelu' or norm_type.lower() != 'bn':
            raise NotImplementedError("codeformer_b200 builds ParseNet with relu_type='LeakyReLU', norm_type='bn' (the shipped model)")
        super().__init__('parsenet', (in_size, out_size, min_feat_size, base_ch, parsing_ch, res_depth, int(ch_range[0]), int(ch_range[1])),
                         parsenet_spec(in_size, out_size, min_feat_size, base_ch, parsing_ch, res_depth, tuple(ch_range)), _parsenet_init)
        self.res_depth, self.parsing_ch = res_depth, parsing_ch
        self.in_size, self.min_feat_size = in_size, min_feat_size

    def forward(self, x, return_img=True):
        """x [B,3,H,W] fp32 CUDA -> (out_mask [B,parsing_ch,H,W], out_img [B,3,H,W])  (parsenet.py:188-194)."""
        if not (torch.is_tensor(x) and x.is_cuda):
            raise RuntimeError('ParseNet.forward: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
        if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != 3:
            raise RuntimeError(f'ParseNet.forward: expected float32 [B,3,H,W], got {x.dtype} {tuple(x.shape)}')
        lib = _lib.load()
        x = x.contiguous()
        B, _, H, W = x.shape
        dev = x.device
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            mask = torch.empty((B, self.parsing_ch, H, W), dtype=torch.float32, device=dev)
            img = torch.empty((B, 3, H, W), dtype=torch.float32, device=dev) if return_img else None
            ws = self._workspace(B, H, W, dev)
            _lib.check(lib.cfb_parsenet_forward(self._net, _lib.ptr(x), _lib.ptr(mask), _lib.ptr(img), B, H, W, _lib.ptr(ws),
                                                ws.numel(), _lib.stream(dev)), 'cfb_parsenet_forward')
        return mask, img

    def masks_u8(self, faces):
        """The parse step of paste_faces_to_input_image:458-468 straight from uint8 faces: CUDA uint8 [N,H,W,3] BGR ->
        (classes, mask), CUDA uint8 [N,H,W] each -- byte-equal to ``face_parse_mask(self(x)[0])`` with x the normalised
        input of the same faces (``cfb_parsenet_masks_u8``: no fp32 input, logits or out_img in between).  H and W must be
        multiples of 2^down_steps (in_size / min_feat_size) and at least twice that."""
        if not (torch.is_tensor(faces) and faces.is_cuda):
            raise RuntimeError('ParseNet.masks_u8: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
        if faces.dtype != torch.uint8 or faces.dim() != 4 or faces.shape[3] != 3:
            raise RuntimeError(f'ParseNet.masks_u8: expected uint8 [N,H,W,3] BGR faces, got {faces.dtype} {tuple(faces.shape)}')
        N, H, W, _ = faces.shape
        div = 2 ** int(np.log2(self.in_size // min(self.in_size, self.min_feat_size)))
        if H % div or W % div or H < 2 * div or W < 2 * div:
            raise RuntimeError(f'ParseNet.masks_u8: H and W must be multiples of {div} and at least {2 * div}, got {H}x{W}')
        lib = _lib.load()
        faces = faces.contiguous()
        dev = faces.device
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            cls = torch.empty((N, H, W), dtype=torch.uint8, device=dev)
            mask = torch.empty((N, H, W), dtype=torch.uint8, device=dev)
            if N:
                ws = self._workspace(N, H, W, dev)
                _lib.check(lib.cfb_parsenet_masks_u8(self._net, _lib.ptr(faces), _lib.ptr(cls), _lib.ptr(mask), N, H, W, _lib.ptr(ws),
                                                     ws.numel(), _lib.stream(dev)), 'cfb_parsenet_masks_u8')
        return cls, mask


def face_parse_mask(out_mask):
    """``out.argmax(dim=1)`` + the MASK_COLORMAP lookup of face_restoration_helper.py:463-468 on the device:
    logits [B,19,H,W] -> (classes uint8 [B,H,W], mask uint8 [B,H,W] with 255 on the face classes 1..13 and 15)."""
    if not (torch.is_tensor(out_mask) and out_mask.is_cuda and out_mask.dtype == torch.float32 and out_mask.dim() == 4):
        raise RuntimeError('face_parse_mask expects the CUDA float32 logits [B,C,H,W] of ParseNet')
    lib = _lib.load()
    out_mask = out_mask.contiguous()
    B, C, H, W = out_mask.shape
    with torch.cuda.device(out_mask.device):
        cls = torch.empty((B, H, W), dtype=torch.uint8, device=out_mask.device)
        mask = torch.empty((B, H, W), dtype=torch.uint8, device=out_mask.device)
        _lib.check(lib.cfb_parse_argmax(_lib.ptr(out_mask), _lib.ptr(cls), _lib.ptr(mask), B, C, H * W,
                                        _lib.stream(out_mask.device)), 'cfb_parse_argmax')
    return cls, mask


def init_parsing_model(model_name='parsenet', half=False, device='cuda', model_path=None):
    """``facelib.parsing.init_parsing_model('parsenet')`` (facelib/parsing/__init__.py:8-23) without the download: pass the
    checkpoint path (``parsing_parsenet.pth``) or load the state dict yourself."""
    if model_name != 'parsenet':
        raise NotImplementedError(f'{model_name} is not built (SURVEY.md section 8 f3 names ParseNet)')
    model = ParseNet(in_size=512, out_size=512, parsing_ch=19)
    if model_path is not None:
        model.load_state_dict(torch.load(model_path, map_location='cpu'), strict=True)
    return model.eval().to(device)
