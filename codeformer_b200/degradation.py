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

Colorization and inpainting inputs (``COLORIZATION_OPTIONS``, ``INPAINTING_OPTIONS``; cfb_degrade_faces_color): the dataset's
colour shift, cv2's gray conversion and torchvision's brightness / contrast / saturation / hue jitter run on the chain's float
image (or gt / 255 without corruption) before its single rounding, each with the reference's float32 arithmetic, so the
bytes are the dataset's from the same float image.  The one exception is the contrast mean: the device takes the exact mean
of the face's gray to one float32 rounding, where torch's CPU sum differs from it in the last bits (include/cfb200.h).  The
brush strokes are drawn with Pillow on the host, as the dataset draws them, and masked pixels become 255.  Motion blur and
flips are training augmentations and are not part of it.
"""
import math
import random

import numpy as np
import torch

from . import _lib

STAGE2_RANGES = dict(blur_sigma=(1, 15), downsample_range=(4, 30), noise_range=(0, 20), jpeg_range=(30, 80))
STAGE3_RANGES = dict(blur_sigma=(0.1, 10), downsample_range=(1, 12), noise_range=(0, 15), jpeg_range=(60, 100))
# options/CodeFormer_colorization.yml: the stage-2 chain, then the colour shift, gray and torchvision jitter stages
COLORIZATION_OPTIONS = dict(STAGE2_RANGES, color_jitter_prob=0.3, color_jitter_shift=20, gray_prob=0.01,
                            color_jitter_pt_prob=0.3)
# options/CodeFormer_inpainting.yml: no corruption, white brush strokes on the ground truth
INPAINTING_OPTIONS = dict(use_corrupt=False, gen_inpaint_mask=True)

# torchvision ColorJitter ops in FFHQBlindDataset.color_jitter_pt's numbering (the values torch.randperm(4) permutes)
JITTER_OPS = ('brightness', 'contrast', 'saturation', 'hue')


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


def _draw_strokes(S, np_rng):
    """The random draws of brush_stroke_mask (basicsr/data/data_util.py:310-362) on an S x S image, in its order: 1 to 3
    strokes, each a polyline of 9 to 28 vertices -- a random start, then steps of a clipped normal length at angles that
    alternate around 2 pi / 5 and its mirror, clipped to [0, S] -- and a width of 30 to 69 pixels."""
    mean_angle, angle_range = 2 * math.pi / 5, 2 * math.pi / 12
    radius = math.sqrt(2. * S * S) / 8
    strokes = []
    for _ in range(np_rng.randint(1, 4)):
        n_vertex = np_rng.randint(8, 28)
        lo = mean_angle - np_rng.uniform(0, angle_range)
        hi = mean_angle + np_rng.uniform(0, angle_range)
        angles = [np_rng.uniform(lo, hi) if i % 2 else 2 * math.pi - np_rng.uniform(lo, hi) for i in range(n_vertex)]
        vertices = [(int(np_rng.randint(0, S)), int(np_rng.randint(0, S)))]
        for a in angles:
            r = np.clip(np_rng.normal(loc=radius, scale=radius // 2), 0, 2 * radius)
            x = np.clip(vertices[-1][0] + r * math.cos(a), 0, S)
            y = np.clip(vertices[-1][1] + r * math.sin(a), 0, S)
            vertices.append((int(x), int(y)))
        strokes.append((vertices, int(np_rng.uniform(30, 70))))
    return strokes


def stroke_mask(S, strokes):
    """uint8 [S, S] mask, 255 under the strokes: each stroke drawn with PIL's ImageDraw as brush_stroke_mask draws it, a
    ``line`` of its width through the vertices, then a disc of diameter width // 2 * 2 at every vertex.  Pillow's fill
    rules are its own, so the mask is rasterised on the host."""
    from PIL import Image, ImageDraw            # only when masks are asked for
    img = Image.new('L', (S, S), 0)
    draw = ImageDraw.Draw(img)
    for vertices, width in strokes:
        draw.line(vertices, fill=255, width=width)
        h = width // 2
        for x, y in vertices:
            draw.ellipse((x - h, y - h, x + h, y + h), fill=255)
    return np.asarray(img, np.uint8).copy()


def _draw_jitter_pt(ranges, torch_rng):
    """color_jitter_pt's draws: torch.randperm(4), then one float32 uniform per op in permuted order whose range is set."""
    kw = {} if torch_rng is None else {'generator': torch_rng}
    out = []
    for op in torch.randperm(4, **kw).tolist():
        if ranges[op] is not None:
            out.append((JITTER_OPS[op], torch.tensor(1.0).uniform_(ranges[op][0], ranges[op][1], **kw).item()))
    return out


def sample_degradations(n, gt_size=512, in_size=512, kernel_list=('iso', 'aniso'), kernel_prob=(0.5, 0.5), blur_kernel_size=41,
                        blur_sigma=(1, 15), downsample_range=(4, 30), noise_range=(0, 20), jpeg_range=(30, 80), py_rng=random,
                        np_rng=np.random, use_corrupt=True, gen_inpaint_mask=False, color_jitter_prob=None,
                        color_jitter_shift=20, gray_prob=0.0, color_jitter_pt_prob=None, brightness=(0.5, 1.5),
                        contrast=(0.5, 1.5), saturation=(0, 1.5), hue=(-0.1, 0.1), torch_rng=None):
    """Draw the degradation parameters of ``n`` faces as FFHQBlindDataset does (defaults: CodeFormer_stage2.yml;
    ``COLORIZATION_OPTIONS`` and ``INPAINTING_OPTIONS`` give the other two tasks' settings).

    Returns a list of dicts with ``kernel_type``, ``sigma_x``, ``sigma_y``, ``rotation`` (0 for iso), ``kernel`` (float64
    [k, k]), ``scale``, ``size`` = int(gt_size // scale), ``noise_sigma`` and ``noise`` (float32 [size, size, 3], already
    multiplied by the sigma; both None without ``noise_range``) and ``quality`` = int(q) (None without ``jpeg_range``).
    Without corruption (``use_corrupt=False`` or ``gen_inpaint_mask=True``, as the dataset decides) all of these are None.
    Then the colour and mask keys:
      ``strokes``    [(vertices [(x, y), ...], width), ...] of the brush strokes, or None
      ``mask``       uint8 [gt_size, gt_size], 255 under the strokes (``stroke_mask``), or None
      ``jitter``     float32 [3], the colour shift in BGR order (``color_jitter_shift`` is in 0..255 units), or None
      ``gray``       bool, the cv2 BGR -> gray conversion
      ``jitter_pt``  [(op, factor), ...] of torchvision's adjust_brightness / contrast / saturation / hue, in the order
                     they apply, or None; ``brightness`` ... ``hue`` are their ranges (None leaves an op out)
    Per face the draws follow FFHQBlindDataset.__getitem__: corruption, strokes, the shift's probability and its three
    uniforms, the gray probability, the torch jitter's probability (np.random) and then torch.randperm(4) and its factors
    from ``torch_rng`` (None: torch's default CPU generator, as the dataset).  No horizontal flip is drawn: sample with
    ``use_hflip: false``.  ``py_rng`` / ``np_rng`` are the ``random`` and ``np.random`` modules or objects with their
    methods; with the colour and mask options at their defaults they are consumed exactly as without them."""
    if in_size > gt_size:
        raise ValueError(f'sample_degradations: in_size {in_size} exceeds gt_size {gt_size}')
    corrupt = use_corrupt and not gen_inpaint_mask
    if corrupt:
        if blur_kernel_size % 2 != 1:
            raise ValueError('sample_degradations: the blur kernel size must be odd')
        for kind in kernel_list:
            if kind not in ('iso', 'aniso'):
                raise NotImplementedError(f'sample_degradations: kernel type {kind!r} is not supported (iso, aniso)')
    elif in_size != gt_size:
        raise ValueError(f'sample_degradations: without corruption the dataset does not resize, so in_size ({in_size}) '
                         f'must equal gt_size ({gt_size})')
    jitter_ranges = (brightness, contrast, saturation, hue)
    out = []
    for _ in range(n):
        p = dict(kernel_type=None, sigma_x=None, sigma_y=None, rotation=None, kernel=None, scale=None, size=None,
                 noise_sigma=None, noise=None, quality=None)
        if corrupt:
            kind = py_rng.choices(list(kernel_list), list(kernel_prob))[0]
            sx, sy, theta, k = _draw_kernel(kind, blur_kernel_size, blur_sigma, np_rng)
            scale = np_rng.uniform(downsample_range[0], downsample_range[1])
            size = int(gt_size // scale)
            p.update(kernel_type=kind, sigma_x=sx, sigma_y=sy, rotation=theta, kernel=k, scale=scale, size=size)
            if noise_range is not None:
                p['noise_sigma'] = np_rng.uniform(noise_range[0] / 255., noise_range[1] / 255.)
                p['noise'] = np.float32(np_rng.randn(size, size, 3)) * p['noise_sigma']
            if jpeg_range is not None:
                p['quality'] = int(np_rng.uniform(jpeg_range[0], jpeg_range[1]))
        p.update(strokes=None, mask=None, jitter=None, gray=False, jitter_pt=None)
        if gen_inpaint_mask:
            p['strokes'] = _draw_strokes(gt_size, np_rng)
            p['mask'] = stroke_mask(gt_size, p['strokes'])
        if color_jitter_prob is not None and np_rng.uniform() < color_jitter_prob:
            shift = color_jitter_shift / 255.
            p['jitter'] = np_rng.uniform(-shift, shift, 3).astype(np.float32)
        if gray_prob and np_rng.uniform() < gray_prob:
            p['gray'] = True
        if color_jitter_pt_prob is not None and np_rng.uniform() < color_jitter_pt_prob:
            p['jitter_pt'] = _draw_jitter_pt(jitter_ranges, torch_rng)
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
    qualities.

    Faces whose parameters carry colour stages (``jitter``, ``gray``, ``jitter_pt``) or a ``mask`` also run the colour and
    mask stages, in the same launches for every op order (``COLORIZATION_OPTIONS``, ``INPAINTING_OPTIONS``); a face without
    them gives the bytes it gives without those keys.  Without corruption (``use_corrupt=False`` or masks) ``in_size`` must
    equal S and the faces of one call must agree on corruption.  Bad factors, jitter or mask shapes raise ``ValueError``;
    a mask together with colour stages raises ``NotImplementedError``."""
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
    if any(_has_color_stage(p) or p.get('mask') is not None or p['kernel'] is None for p in params):
        lq, _ = _run_color(x, params, in_size, debug=False)
    else:
        lq, _, _ = _run(x, params, in_size, debug=False)
    return lq, params


def _has_color_stage(p):
    return p.get('jitter') is not None or bool(p.get('gray')) or bool(p.get('jitter_pt'))


def _color_tables(params, S):
    """The per-face descriptors of cfb_degrade_faces_color: ops int32 [B, 6] (flags, n, op codes), factors float32 [B, 7]
    (shift BGR, factors) and the mask faces' indices."""
    B = len(params)
    ops = np.zeros((B, 6), np.int32)
    fac = np.zeros((B, 7), np.float32)
    masked = []
    for b, p in enumerate(params):
        if p.get('mask') is not None:
            if _has_color_stage(p):
                raise NotImplementedError('degrade_faces: masks with colour stages are not supported (the dataset runs them '
                                          'in float64 then, and its gray stage fails in cv2; no option set combines them)')
            if p['kernel'] is not None:
                raise ValueError('degrade_faces: a masked face is not corrupted (the dataset skips the chain with masks)')
            m = np.asarray(p['mask'])
            if m.shape != (S, S) or m.dtype != np.uint8:
                raise ValueError(f'degrade_faces: mask of face {b} must be uint8 [{S}, {S}], got {m.dtype} {m.shape}')
            ops[b, 0] |= 4
            masked.append(b)
        if p.get('jitter') is not None:
            j = np.asarray(p['jitter'], np.float32)
            if j.shape != (3,) or not np.isfinite(j).all():
                raise ValueError(f'degrade_faces: jitter of face {b} must be 3 finite values, got {p["jitter"]!r}')
            ops[b, 0] |= 1
            fac[b, :3] = j
        if p.get('gray'):
            ops[b, 0] |= 2
        seq = list(p.get('jitter_pt') or [])
        names = [op for op, _ in seq]
        if len(set(names)) != len(names) or any(op not in JITTER_OPS for op in names):
            raise ValueError(f'degrade_faces: jitter_pt of face {b} must name each of {JITTER_OPS} at most once, got {names}')
        ops[b, 1] = len(seq)
        for k, (op, f) in enumerate(seq):
            f32 = np.float32(f)
            if float(f32) != float(f):
                raise ValueError(f'degrade_faces: the {op} factor {f!r} of face {b} is not a float32 value')
            ok = -0.5 <= f <= 0.5 if op == 'hue' else f >= 0
            if not (math.isfinite(f) and ok):
                raise ValueError(f'degrade_faces: bad {op} factor {f!r} for face {b}' +
                                 (' (hue in [-0.5, 0.5])' if op == 'hue' else ' (>= 0)'))
            ops[b, 2 + k] = JITTER_OPS.index(op)
            fac[b, 3 + k] = f32
    return ops, fac, masked


def _run_color(x, params, in_size, debug):
    """The chain (for corrupted faces) and the colour and mask stages; returns (lq, contrast means or None)."""
    B, S = x.shape[0], x.shape[1]
    dev = x.device
    corrupt = {p['kernel'] is not None for p in params}
    if len(corrupt) > 1:
        raise ValueError('degrade_faces: corrupted and uncorrupted faces need separate calls')
    corrupt = corrupt.pop() if corrupt else True
    if not corrupt and in_size != S:
        raise ValueError(f'degrade_faces: without corruption the dataset does not resize, so in_size ({in_size}) must equal '
                         f'the face size ({S})')
    ops, fac, masked = _color_tables(params, S)
    lq = torch.empty((B, in_size, in_size, 3), dtype=torch.uint8, device=dev)
    means = torch.empty(max(B, 1), dtype=torch.float32, device=dev) if debug else None
    if B == 0:
        return lq, means
    lib = _lib.load()
    kern = noise = None
    sizes = qual = offs = None
    if corrupt:
        ks = {p['kernel'].shape[0] for p in params}
        if len(ks) > 1:
            raise ValueError('degrade_faces: every face needs the same blur kernel size')
        ks = ks.pop()
        sizes, qual, offs, fields = _chain_tables(params, S)
        kern = torch.from_numpy(np.stack([np.asarray(p['kernel'], np.float64) for p in params])).to(dev)
        noise = torch.from_numpy(np.concatenate(fields)).to(dev) if fields else None
    masks = None
    if masked:
        m = np.zeros((B, S, S), np.uint8)
        for b in masked:
            m[b] = params[b]['mask']
        masks = torch.from_numpy(m).to(dev)
    with torch.cuda.device(dev):
        ws = _workspace(lib.cfb_degrade_color_workspace_bytes(B, S, _host(sizes), _host(qual), ops.ctypes.data, in_size), dev,
                        'cfb_degrade_color_workspace_bytes')
        args = [_lib.ptr(x), B, S, _lib.ptr(kern), ks if corrupt else 0, _host(sizes), _host(qual), _lib.ptr(noise), _host(offs),
                ops.ctypes.data, fac.ctypes.data, _lib.ptr(masks), in_size, _lib.ptr(lq), _lib.ptr(ws), ws.numel()]
        if debug:
            _lib.check(lib.cfb_debug_degrade_faces_color(*args, _lib.ptr(means), _lib.stream(dev)),
                       'cfb_debug_degrade_faces_color')
        else:
            _lib.check(lib.cfb_degrade_faces_color(*args, _lib.stream(dev)), 'cfb_degrade_faces_color')
    return lq, means


def _host(a):
    return None if a is None else a.ctypes.data


def _chain_tables(params, S):
    """Small sizes, JPEG qualities (0 = none), noise offsets (-1 = none) and the noise fields of the corruption chain."""
    B = len(params)
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
    return sizes, qual, offs, fields


def _run(x, params, in_size, debug):
    B, S = x.shape[0], x.shape[1]
    dev = x.device
    ks = {p['kernel'].shape[0] for p in params}
    if len(ks) > 1:
        raise ValueError('degrade_faces: every face needs the same blur kernel size')
    ks = ks.pop() if ks else 1
    sizes, qual, offs, fields = _chain_tables(params, S)
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
