"""numpy / torch restatement of FFHQBlindDataset's colour and mask stages (basicsr/data/ffhq_blind_dataset.py:242-284) on the
float image the corruption chain leaves.  TEST INFRASTRUCTURE: written from the algorithms, checked against cv2 and
torchvision on the CPU; torchvision is not imported.

  gray_cv2          cv2.cvtColor(float32 BGR, COLOR_BGR2GRAY): fma(r, 0.299f, fma(b, 0.114f, g * 0.587f))
  rgb_to_gray       torchvision's rgb_to_grayscale on float32 CHW: (0.2989 r + 0.587 g) + 0.114 b, one torch op each
  adjust_*          torchvision's adjust_brightness / contrast / saturation / hue as torch op sequences (_blend, _rgb2hsv,
                    (h + f) % 1.0, _hsv2rgb); adjust_contrast takes the mean as an argument or takes torch's
  color_stages      shift, gray, BGR -> RGB, the ops in order, clip(round(x * 255)) -> uint8 BGR
  chain_float       the float32 image the chain leaves: its final INTER_LINEAR, or gt / 255 without corruption
  degrade_color     one face from uint8 GT and one entry of codeformer_b200.degradation.sample_degradations
"""
import numpy as np
import torch

from oracle import degradation_oracle as DO

F32 = np.float32


def gray_cv2(img):
    """float32 [H, W, 3] BGR -> float32 [H, W]."""
    b, g, r = img[..., 0], img[..., 1], img[..., 2]
    return DO.fma32(r, F32(0.299), DO.fma32(b, F32(0.114), (g * F32(0.587)).astype(F32)))


def rgb_to_gray(img):
    """float32 [3, H, W] RGB -> [1, H, W]."""
    r, g, b = img[0], img[1], img[2]
    return (0.2989 * r + 0.587 * g + 0.114 * b).unsqueeze(0)


def _blend(x, y, ratio):
    ratio = float(ratio)
    return (ratio * x + (1.0 - ratio) * y).clamp(0, 1.0)


def contrast_mean(img):
    """torch's CPU float32 mean of the gray, as adjust_contrast takes it."""
    return torch.mean(rgb_to_gray(img), dim=(-3, -2, -1), keepdim=True)


def adjust_brightness(img, f):
    return _blend(img, torch.zeros_like(img), f)


def adjust_contrast(img, f, mean=None):
    m = contrast_mean(img) if mean is None else torch.full((1, 1, 1), float(mean), dtype=torch.float32)
    return _blend(img, m, f)


def adjust_saturation(img, f):
    return _blend(img, rgb_to_gray(img), f)


def _rgb2hsv(img):
    r, g, b = img[0], img[1], img[2]
    maxc, minc = img.max(0).values, img.min(0).values
    same = maxc == minc
    span = maxc - minc
    one = torch.ones_like(maxc)
    s = span / torch.where(same, one, maxc)
    div = torch.where(same, one, span)
    rc, gc, bc = (maxc - r) / div, (maxc - g) / div, (maxc - b) / div
    h = (maxc == r) * (bc - gc) + ((maxc == g) & (maxc != r)) * (2.0 + rc - bc) + \
        ((maxc != g) & (maxc != r)) * (4.0 + gc - rc)
    return torch.fmod(h / 6.0 + 1.0, 1.0), s, maxc


def _hsv2rgb(h, s, v):
    i = torch.floor(h * 6.0)
    f = h * 6.0 - i
    i = i.to(torch.int32) % 6
    p = torch.clamp(v * (1.0 - s), 0.0, 1.0)
    q = torch.clamp(v * (1.0 - s * f), 0.0, 1.0)
    t = torch.clamp(v * (1.0 - s * (1.0 - f)), 0.0, 1.0)
    table = ((v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v), (v, p, q))     # (r, g, b) for i = 0 .. 5
    out = torch.zeros((3,) + h.shape, dtype=h.dtype)
    for k, rgb in enumerate(table):
        for c in range(3):
            out[c] = torch.where(i == k, rgb[c], out[c])
    return out


def adjust_hue(img, f):
    h, s, v = _rgb2hsv(img)
    return _hsv2rgb((h + f) % 1.0, s, v)


def apply_ops(img, ops, mean=None):
    """The (op, factor) list on float32 RGB [3, H, W]; ``mean`` replaces torch's contrast mean.  Returns (img, the mean
    the contrast op used or None)."""
    used = None
    for op, f in ops:
        if op == 'brightness':
            img = adjust_brightness(img, f)
        elif op == 'contrast':
            used = float(contrast_mean(img)) if mean is None else float(mean)
            img = adjust_contrast(img, f, used)
        elif op == 'saturation':
            img = adjust_saturation(img, f)
        elif op == 'hue':
            img = adjust_hue(img, f)
        else:
            raise ValueError(op)
    return img, used


def round_u8(x):
    """clip(round(x * 255)) of float32 values (torch rounds half to even)."""
    return DO.to_u8(np.asarray(x, F32) * F32(255.))


def color_stages(x, p, mean=None):
    """float32 [H, W, 3] BGR and one parameter dict -> (uint8 BGR, the contrast mean used or None)."""
    x = np.asarray(x, F32)
    if p.get('jitter') is not None:
        x = np.clip(x + np.asarray(p['jitter'], F32), 0, 1).astype(F32)
    if p.get('gray'):
        x = np.repeat(gray_cv2(x)[..., None], 3, 2)
    img = torch.from_numpy(np.ascontiguousarray(x[..., ::-1].transpose(2, 0, 1)))
    img, used = apply_ops(img, p.get('jitter_pt') or [], mean)
    return round_u8(img.numpy().transpose(1, 2, 0)[..., ::-1]), used


def chain_float(gt_u8, p, in_size):
    """The float32 image the colour stages start from: the chain's final INTER_LINEAR (the blur evaluated as the device
    evaluates it, oracle/degradation_oracle.py), or gt / 255 without corruption."""
    img = (gt_u8.astype(F32) / F32(255.)).astype(F32)
    if p['kernel'] is None:
        return img
    S, s = gt_u8.shape[0], p['size']
    y0, y1, _ = DO.linear_taps(s, S)
    rows = np.unique(np.concatenate([y0, y1]))
    full = np.zeros((S, S, 3), F32)
    full[np.ix_(rows, rows)] = DO.filter2d_f64(img, p['kernel'], rows, rows)
    return finish_chain(DO.resize_linear(full, s, s), p, in_size)


def finish_chain(x, p, in_size):
    """From the downsampled float image: noise and clip, the JPEG round trip, INTER_LINEAR to in_size."""
    if p['noise'] is not None:
        x = np.clip((x + p['noise']).astype(F32), 0, 1)
    if p['quality'] is not None:
        x = (DO.jpeg_roundtrip(DO.to_u8(x * F32(255.)), p['quality']).astype(F32) / F32(255.)).astype(F32)
    return DO.resize_linear(x, in_size, in_size)


def degrade_color(gt_u8, p, in_size, mean=None):
    """One face -> (lq uint8 BGR [in, in, 3], the contrast mean used or None)."""
    if p.get('mask') is not None:
        return np.where(np.asarray(p['mask'])[..., None] != 0, np.uint8(255), gt_u8), None
    return color_stages(chain_float(gt_u8, p, in_size), p, mean)
