"""BiSeNet on libcfb200: the light face-parsing network of the paste-back step (facelib's own default parser).

Mirrors ``BiSeNet(num_class)`` of /root/reference/facelib/parsing/bisenet.py:104-140 (ResNet-18 context path,
facelib/parsing/resnet.py) as built by ``init_parsing_model('bisenet')``: same constructor and ``state_dict`` (191 entries for
19 classes, BatchNorm buffers included, so ``parsing_bisenet.pth`` loads strictly) and ``forward(x) -> (out, out16, out32)``.
``masks_u8`` gives the parse masks of ``FaceRestoreHelper.paste_faces_to_input_image`` (face_restoration_helper.py:457-468)
straight from uint8 faces.  Eval-mode BatchNorm is folded into the convs when the native copy is prepared.  No CPU fallback;
inference only.
"""
from collections import OrderedDict

import torch
import torch.nn as nn

from . import _lib
from .native import NativeNet


def bisenet_spec(num_class=19):
    """state_dict keys -> (shape, dtype) of the reference BiSeNet(num_class), in registration order."""
    spec = OrderedDict()

    def conv(name, cin, cout, k):
        spec[name + '.weight'] = ((cout, cin, k, k), torch.float32)

    def bn(name, c):
        for k in ('weight', 'bias', 'running_mean', 'running_var'):
            spec[f'{name}.{k}'] = ((c,), torch.float32)
        spec[name + '.num_batches_tracked'] = ((), torch.int64)

    def cbr(name, cin, cout, k):
        conv(name + '.conv', cin, cout, k)
        bn(name + '.bn', cout)

    conv('cp.resnet.conv1', 3, 64, 7)
    bn('cp.resnet.bn1', 64)
    cin = 64
    for li, cout in enumerate((64, 128, 256, 512)):
        for b in range(2):
            p = f'cp.resnet.layer{li + 1}.{b}'
            conv(p + '.conv1', cin, cout, 3); bn(p + '.bn1', cout)
            conv(p + '.conv2', cout, cout, 3); bn(p + '.bn2', cout)
            if cin != cout:
                conv(p + '.downsample.0', cin, cout, 1); bn(p + '.downsample.1', cout)
            cin = cout
    for name, c in (('cp.arm16', 256), ('cp.arm32', 512)):
        cbr(name + '.conv', c, 128, 3)
        conv(name + '.conv_atten', 128, 128, 1)
        bn(name + '.bn_atten', 128)
    cbr('cp.conv_head32', 128, 128, 3)
    cbr('cp.conv_head16', 128, 128, 3)
    cbr('cp.conv_avg', 512, 128, 1)
    cbr('ffm.convblk', 256, 256, 1)
    conv('ffm.conv1', 256, 64, 1)
    conv('ffm.conv2', 64, 256, 1)
    for name, cin, mid in (('conv_out', 256, 256), ('conv_out16', 128, 64), ('conv_out32', 128, 64)):
        cbr(name + '.conv', cin, mid, 3)
        conv(name + '.conv_out', mid, num_class, 1)
    return spec


def _bisenet_init(name, entry, g):
    """PyTorch's default initialisation, which the reference keeps: filters U(+-1/sqrt(fan_in)), BatchNorm (1, 0) with
    running statistics (0, 1)."""
    shape, dtype = entry
    leaf = name.rsplit('.', 1)[-1]
    if dtype == torch.int64:
        return torch.tensor(0, dtype=torch.long)
    if leaf in ('running_mean', 'running_var'):
        return torch.zeros(shape) if leaf == 'running_mean' else torch.ones(shape)
    if len(shape) == 4:
        fan_in = shape[1] * shape[2] * shape[3]
        return nn.Parameter((torch.rand(shape, generator=g) * 2 - 1) / fan_in ** 0.5)
    return nn.Parameter(torch.ones(shape) if leaf == 'weight' else torch.zeros(shape))


class BiSeNet(NativeNet):
    """Parameter holder with the reference's ``state_dict`` + ``forward`` on the wgmma conv engine (fp32 only)."""

    def __init__(self, num_class):
        if not 1 <= int(num_class) <= 64:
            raise NotImplementedError(f'codeformer_b200 builds BiSeNet with 1..64 classes, got {num_class}')
        super().__init__('bisenet', (int(num_class),), bisenet_spec(int(num_class)), _bisenet_init)
        self.num_class = int(num_class)

    @staticmethod
    def _check_size(owner, H, W):
        if H % 32 or W % 32 or H < 32 or W < 32:
            raise RuntimeError(f'{owner}: H and W must be positive multiples of 32, got {H}x{W}')

    def forward(self, x, return_feat=False):
        """x [B,3,H,W] fp32 CUDA -> (out, out16, out32), each [B,num_class,H,W] fp32 (bisenet.py:120-140).  H and W must be
        multiples of 32: then every nearest resize of the context path is an exact x2 or a broadcast of a 1 x 1 map."""
        if return_feat:
            raise NotImplementedError('codeformer_b200.BiSeNet returns (out, out16, out32) only (return_feat=True is not built)')
        if not (torch.is_tensor(x) and x.is_cuda):
            raise RuntimeError('BiSeNet.forward: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
        if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != 3:
            raise RuntimeError(f'BiSeNet.forward: expected float32 [B,3,H,W], got {x.dtype} {tuple(x.shape)}')
        B, _, H, W = x.shape
        self._check_size('BiSeNet.forward', H, W)
        lib = _lib.load()
        x = x.contiguous()
        dev = x.device
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            outs = [torch.empty((B, self.num_class, H, W), dtype=torch.float32, device=dev) for _ in range(3)]
            if B:
                ws = self._workspace(B, H, W, dev)
                _lib.check(lib.cfb_bisenet_forward(self._net, _lib.ptr(x), *(_lib.ptr(o) for o in outs), B, H, W, _lib.ptr(ws),
                                                   ws.numel(), _lib.stream(dev)), 'cfb_bisenet_forward')
        return tuple(outs)

    def masks_u8(self, faces):
        """The parse step of paste_faces_to_input_image:458-468 straight from uint8 faces: CUDA uint8 [N,H,W,3] BGR ->
        (classes, mask), CUDA uint8 [N,H,W] each -- byte-equal to ``face_parse_mask(self(x)[0])`` with x the normalised
        input of the same faces (``cfb_bisenet_masks_u8``: the upsampling of ``out`` is fused with the argmax, and out16 /
        out32 are not computed).  H and W must be multiples of 32."""
        if not (torch.is_tensor(faces) and faces.is_cuda):
            raise RuntimeError('BiSeNet.masks_u8: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
        if faces.dtype != torch.uint8 or faces.dim() != 4 or faces.shape[3] != 3:
            raise RuntimeError(f'BiSeNet.masks_u8: expected uint8 [N,H,W,3] BGR faces, got {faces.dtype} {tuple(faces.shape)}')
        N, H, W, _ = faces.shape
        self._check_size('BiSeNet.masks_u8', H, W)
        lib = _lib.load()
        faces = faces.contiguous()
        dev = faces.device
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            cls = torch.empty((N, H, W), dtype=torch.uint8, device=dev)
            mask = torch.empty((N, H, W), dtype=torch.uint8, device=dev)
            if N:
                ws = self._workspace(N, H, W, dev)
                _lib.check(lib.cfb_bisenet_masks_u8(self._net, _lib.ptr(faces), _lib.ptr(cls), _lib.ptr(mask), N, H, W, _lib.ptr(ws),
                                                    ws.numel(), _lib.stream(dev)), 'cfb_bisenet_masks_u8')
        return cls, mask
