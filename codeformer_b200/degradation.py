"""Synthetic degradations on the GPU: the corruption chain of FFHQBlindDataset (basicsr/data/ffhq_blind_dataset.py:210-240),
which makes CodeFormer's evaluation pairs, for batches of uint8 faces.

  sample_degradations   the host draw of every face's parameters, consuming ``random`` and ``np.random`` in the dataset's
                        order (random.choices, the kernel's uniforms, scale, noise sigma, randn, JPEG quality), so the same
                        seeds give the same parameters bit for bit
  degrade_faces         the chain on the device: 41 x 41 Gaussian blur (BORDER_REFLECT_101), INTER_LINEAR to int(S // scale),
                        Gaussian noise and clip, JPEG at int(q), INTER_LINEAR back to ``in_size``, clip(round(x * 255))
  jpeg_roundtrip        cv2.imdecode(cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, q]), 1) on the device, byte for byte

Exactness (include/cfb200.h, cfb_degrade_faces): the blur is the float64 direct correlation in a fixed order, rounded once to
float32 (cv2's own filter2D filters a 41 x 41 kernel by DFT, whose error is about 3e-8 on [0, 1] images); every later stage
follows cv2's and libjpeg-turbo's arithmetic exactly, so from the same blurred image the uint8 result is cv2's byte for byte.
Motion blur, flips, colour jitter, gray conversion and inpainting masks are training augmentations and are not part of it.
"""
import math
import random

import numpy as np
import torch

from . import _lib

STAGE2_RANGES = dict(blur_sigma=(1, 15), downsample_range=(4, 30), noise_range=(0, 20), jpeg_range=(30, 80))
STAGE3_RANGES = dict(blur_sigma=(0.1, 10), downsample_range=(1, 12), noise_range=(0, 15), jpeg_range=(60, 100))


def _gaussian_kernel(ksize, p, r, q):
    """The bivariate Gaussian density exp(-(p x^2 + 2 r x y + q y^2) / 2) on the integer offsets -k//2 .. k//2 (x along
    columns, y along rows), normalised to sum 1; [[p, r], [r, q]] is the inverse covariance."""
    off = np.arange(ksize, dtype=np.float64) - ksize // 2
    x, y = off[None, :], off[:, None]
    k = np.exp(-0.5 * (p * x * x + 2. * r * x * y + q * y * y))
    return k / k.sum()


def _draw_kernel(kind, ksize, sigma_range, np_rng):
    """Sigmas (and for 'aniso' a rotation) drawn as the dataset's sampler draws them, and the kernel.  The covariance is
    sigma^2 I, or diag(sigma_x^2, sigma_y^2) rotated by theta, R D R^T; its inverse R D^-1 R^T has the entries below."""
    if kind == 'iso':
        sx = np_rng.uniform(sigma_range[0], sigma_range[1])
        sy, theta = sx, 0.
        k = _gaussian_kernel(ksize, 1. / (sx * sx), 0., 1. / (sx * sx))
    elif kind == 'aniso':
        sx = np_rng.uniform(sigma_range[0], sigma_range[1])
        sy = np_rng.uniform(sigma_range[0], sigma_range[1])
        theta = np_rng.uniform(-math.pi, math.pi)
        c, s_ = math.cos(theta), math.sin(theta)
        ix, iy = 1. / (sx * sx), 1. / (sy * sy)
        k = _gaussian_kernel(ksize, c * c * ix + s_ * s_ * iy, c * s_ * (ix - iy), s_ * s_ * ix + c * c * iy)
    else:
        raise NotImplementedError(f'sample_degradations: kernel type {kind!r} is not supported (iso, aniso)')
    return sx, sy, theta, k / np.sum(k)          # the dataset's sampler normalises the normalised kernel once more


def sample_degradations(n, gt_size=512, in_size=512, kernel_list=('iso', 'aniso'), kernel_prob=(0.5, 0.5), blur_kernel_size=41,
                        blur_sigma=(1, 15), downsample_range=(4, 30), noise_range=(0, 20), jpeg_range=(30, 80), py_rng=random,
                        np_rng=np.random):
    """Draw the degradation parameters of ``n`` faces as FFHQBlindDataset does (defaults: CodeFormer_stage2.yml).

    Returns a list of dicts with ``kernel_type``, ``sigma_x``, ``sigma_y``, ``rotation`` (0 for iso), ``kernel`` (float64
    [k, k]), ``scale``, ``size`` = int(gt_size // scale), ``noise_sigma`` and ``noise`` (float32 [size, size, 3], already
    multiplied by the sigma; both None without ``noise_range``) and ``quality`` = int(q) (None without ``jpeg_range``).
    ``py_rng`` / ``np_rng`` are the ``random`` and ``np.random`` modules or objects with their methods."""
    if in_size > gt_size:
        raise ValueError(f'sample_degradations: in_size {in_size} exceeds gt_size {gt_size}')
    if blur_kernel_size % 2 != 1:
        raise ValueError('sample_degradations: the blur kernel size must be odd')
    for kind in kernel_list:
        if kind not in ('iso', 'aniso'):
            raise NotImplementedError(f'sample_degradations: kernel type {kind!r} is not supported (iso, aniso)')
    out = []
    for _ in range(n):
        kind = py_rng.choices(list(kernel_list), list(kernel_prob))[0]
        sx, sy, theta, k = _draw_kernel(kind, blur_kernel_size, blur_sigma, np_rng)
        scale = np_rng.uniform(downsample_range[0], downsample_range[1])
        size = int(gt_size // scale)
        p = dict(kernel_type=kind, sigma_x=sx, sigma_y=sy, rotation=theta, kernel=k, scale=scale, size=size,
                 noise_sigma=None, noise=None, quality=None)
        if noise_range is not None:
            p['noise_sigma'] = np_rng.uniform(noise_range[0] / 255., noise_range[1] / 255.)
            p['noise'] = np.float32(np_rng.randn(size, size, 3)) * p['noise_sigma']
        if jpeg_range is not None:
            p['quality'] = int(np_rng.uniform(jpeg_range[0], jpeg_range[1]))
        out.append(p)
    return out


def _u8_faces(x, fn):
    if isinstance(x, np.ndarray):
        if x.dtype != np.uint8:
            raise NotImplementedError(f'{fn}: dtype {x.dtype} is not supported (uint8 BGR)')
        x = torch.from_numpy(np.ascontiguousarray(x)).to(torch.device('cuda', torch.cuda.current_device()))
    elif not torch.is_tensor(x):
        raise TypeError(f'{fn}: expected a numpy array or a CUDA tensor, got {type(x).__name__}')
    if not x.is_cuda:
        raise RuntimeError(f'{fn}: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
    if x.dtype != torch.uint8:
        raise NotImplementedError(f'{fn}: dtype {x.dtype} is not supported (uint8 BGR)')
    if x.dim() != 4 or x.shape[3] != 3:
        raise ValueError(f'{fn}: expected uint8 BGR images [B,H,W,3], got shape {tuple(x.shape)}')
    return x.contiguous()


def _workspace(nbytes, dev, what):
    if nbytes < 0:
        _lib.check(1, what)
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=dev)


def degrade_faces(gt, params=None, in_size=512, **ranges):
    """Degrade uint8 BGR faces ``gt`` [B, S, S, 3] (numpy or CUDA) with the FFHQBlindDataset chain.

    ``params``: the list ``sample_degradations`` returns, one entry per face; when None it is drawn here with
    ``gt_size=S``, ``in_size`` and ``ranges`` (the keyword arguments of ``sample_degradations``).  Returns ``(lq, params)``:
    lq uint8 BGR [B, in_size, in_size, 3] on the device -- clip(round(x * 255)) of the dataset's float result, ready for
    ``CodeFormer.forward_u8`` / ``forward_u8_sweep``.  All faces run in one launch per stage, whatever their sizes and
    qualities."""
    x = _u8_faces(gt, 'degrade_faces')
    B, S, S2, _ = x.shape
    if S != S2:
        raise ValueError(f'degrade_faces: faces must be square, got {S}x{S2}')
    in_size = int(in_size)
    if not 1 <= in_size <= S:
        raise ValueError(f'degrade_faces: in_size {in_size} must be in 1..gt_size ({S})')
    if params is None:
        params = sample_degradations(B, gt_size=S, in_size=in_size, **ranges)
    elif ranges:
        raise ValueError('degrade_faces: give either params or sampling ranges, not both')
    if len(params) != B:
        raise ValueError(f'degrade_faces: {len(params)} parameter sets for {B} faces')
    lq, _, _ = _run(x, params, in_size, debug=False)
    return lq, params


def _run(x, params, in_size, debug):
    B, S = x.shape[0], x.shape[1]
    dev = x.device
    ks = {p['kernel'].shape[0] for p in params}
    if len(ks) > 1:
        raise ValueError('degrade_faces: every face needs the same blur kernel size')
    ks = ks.pop() if ks else 1
    sizes = np.array([int(p['size']) for p in params], np.int32)
    if B and (sizes.min() < 1 or sizes.max() > S):
        raise ValueError(f'degrade_faces: small sizes must be in 1..{S}')
    qual = np.array([0 if p['quality'] is None else int(p['quality']) for p in params], np.int32)
    if any(p['quality'] is not None and not 1 <= int(p['quality']) <= 100 for p in params):
        raise ValueError('degrade_faces: JPEG quality must be in 1..100')
    offs = np.full(B, -1, np.int64)
    fields, at = [], 0
    for b, p in enumerate(params):
        if p['noise'] is not None:
            nz = np.asarray(p['noise'], np.float32)
            if nz.shape != (sizes[b], sizes[b], 3):
                raise ValueError(f'degrade_faces: noise of face {b} has shape {nz.shape}, expected {(sizes[b], sizes[b], 3)}')
            offs[b] = at
            at += nz.size
            fields.append(nz.ravel())
    lib = _lib.load()
    lq = torch.empty((B, in_size, in_size, 3), dtype=torch.uint8, device=dev)
    packed = int((sizes.astype(np.int64) ** 2 * 3).sum())
    stage_a = torch.empty(max(packed, 1), dtype=torch.float32, device=dev) if debug else None
    pre = torch.zeros(max(packed, 1), dtype=torch.uint8, device=dev) if debug else None
    if B == 0:
        return lq, stage_a, pre
    kern = torch.from_numpy(np.stack([np.asarray(p['kernel'], np.float64) for p in params])).to(dev)
    noise = torch.from_numpy(np.concatenate(fields)).to(dev) if fields else None
    with torch.cuda.device(dev):
        ws = _workspace(lib.cfb_degrade_workspace_bytes(B, S, sizes.ctypes.data, qual.ctypes.data), dev,
                        'cfb_degrade_workspace_bytes')
        args = [_lib.ptr(x), B, S, _lib.ptr(kern), ks, sizes.ctypes.data, qual.ctypes.data, _lib.ptr(noise), offs.ctypes.data,
                in_size, _lib.ptr(lq), _lib.ptr(ws), ws.numel()]
        if debug:
            _lib.check(lib.cfb_debug_degrade_faces(*args, _lib.ptr(stage_a), _lib.ptr(pre), _lib.stream(dev)),
                       'cfb_debug_degrade_faces')
        else:
            _lib.check(lib.cfb_degrade_faces(*args, _lib.stream(dev)), 'cfb_degrade_faces')
    return lq, stage_a, pre


def jpeg_roundtrip(images, quality):
    """cv2.imdecode(cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, q]), 1) of each uint8 BGR image of ``images``
    [B, H, W, 3] (numpy or CUDA), byte for byte (libjpeg-turbo's baseline 4:2:0 with its islow DCTs), on the device.
    ``quality``: one int 1..100 or one per image.  Returns a uint8 CUDA tensor of the same shape."""
    x = _u8_faces(images, 'jpeg_roundtrip')
    B, H, W, _ = x.shape
    q = np.broadcast_to(np.asarray(quality, np.int64), (B,)).astype(np.int32).copy()
    if B and (q.min() < 1 or q.max() > 100):
        raise ValueError('jpeg_roundtrip: quality must be in 1..100')
    out = torch.empty_like(x)
    if B == 0:
        return out
    lib = _lib.load()
    with torch.cuda.device(x.device):
        ws = _workspace(lib.cfb_jpeg_workspace_bytes(B, H, W), x.device, 'cfb_jpeg_workspace_bytes')
        _lib.check(lib.cfb_jpeg_roundtrip(_lib.ptr(x), _lib.ptr(out), B, H, W, q.ctypes.data, _lib.ptr(ws), ws.numel(),
                                          _lib.stream(x.device)), 'cfb_jpeg_roundtrip')
    return out
