"""CPU oracle for ``cv2.resize(..., interpolation=INTER_LANCZOS4)`` of uint16 images -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

cv2 resizes 16-bit images through float32 weights and float32 sums (imgproc/src/resize.cpp: HResizeLanczos4 with
VResizeLanczos4 / VResizeLanczos4Vec_32f16u), not through the 2048-scaled int16 taps of its uint8 path
(resize_lanczos4_oracle.py).  This numpy restatement of it is byte-equal to cv2 on the CPU:

  * per output coordinate d the source coordinate is ``f = (d + 0.5) * scale - 0.5`` rounded to float32 with
    ``scale = 1 / (dst / src)`` in double; ``s = floor(f)`` and the eight taps sit at ``s - 3 .. s + 4``, each clamped to the image;
  * the float32 weights of ``x = f - s`` (interpolateLanczos4): one sin / cos of ``-(x + 3) pi / 4`` with ``x + 3`` summed in
    float32, rotated by multiples of 45 degrees, each divided by its own ``y * y`` where ``y = -((x + 3) - i) pi / 4`` is formed
    in double from the float32 ``(x + 3) - i``; a tap whose ``|(x + 3) - i| < 1e-6`` is 1e30.  The float32 sum of the eight
    normalises them (``w *= 1 / sum``), so ``x = 0`` leaves the unit tap plus weights of about 1e-31;
  * the horizontal pass is ``((s0 w0 + s1 w1) + s2 w2) + ...`` in float32, every product and sum rounded (no fused
    multiply-add), and the vertical pass the same over the eight rows; then round half to even and saturate to uint16.

tests/test_oracle_lanczos_u16.py pins this restatement against cv2 and the tables of ``cfb_lanczos4_table_f32`` against
``tap_table``.
"""
import math

import numpy as np

S45 = 0.70710678118654752440084436210485
ROT = ((1, 0), (-S45, -S45), (0, 1), (S45, -S45), (-1, 0), (S45, S45), (0, -1), (-S45, S45))


def lanczos4_coeffs(x):
    """The eight float32 weights of one fractional offset ``x`` (a float32 in [0, 1))."""
    x = np.float32(x)
    x3 = np.float32(x + np.float32(3))
    y0 = -float(x3) * math.pi * 0.25
    s0, c0 = math.sin(y0), math.cos(y0)
    c = np.zeros(8, np.float32)
    total = np.float32(0)
    for i in range(8):
        t = np.float32(x3 - np.float32(i))
        if abs(t) >= np.float32(1e-6):
            y = -float(t) * math.pi * 0.25
            c[i] = np.float32((ROT[i][0] * s0 + ROT[i][1] * c0) / (y * y))
        else:
            c[i] = np.float32(1e30)
        total = np.float32(total + c[i])
    return c * (np.float32(1) / total)


def tap_table(src_len, dst_len):
    """-> (idx [dst_len] int32: floor of the source coordinate, coef [dst_len, 8] float32 weights)."""
    scale = 1.0 / (float(dst_len) / float(src_len))
    idx = np.zeros(dst_len, np.int32)
    coef = np.zeros((dst_len, 8), np.float32)
    for d in range(dst_len):
        f = np.float32((d + 0.5) * scale - 0.5)
        s = int(np.floor(f))
        idx[d] = s
        coef[d] = lanczos4_coeffs(np.float32(f - np.float32(s)))
    return idx, coef


def resize_lanczos4_u16(src, dsize):
    """cv2.resize(src, dsize, interpolation=cv2.INTER_LANCZOS4) for a uint16 [h, w, c] image, dsize = (w', h')."""
    src = np.asarray(src)
    assert src.dtype == np.uint16 and src.ndim == 3
    h, w = src.shape[:2]
    ow, oh = dsize
    if (ow, oh) == (w, h):
        return src.copy()
    xi, xt = tap_table(w, ow)
    yi, yt = tap_table(h, oh)
    s = src.astype(np.float32)
    rows = s[:, np.clip(xi - 3, 0, w - 1)] * xt[:, 0][None, :, None]
    for k in range(1, 8):
        rows = rows + s[:, np.clip(xi - 3 + k, 0, w - 1)] * xt[:, k][None, :, None]
    out = rows[np.clip(yi - 3, 0, h - 1)] * yt[:, 0][:, None, None]
    for k in range(1, 8):
        out = out + rows[np.clip(yi - 3 + k, 0, h - 1)] * yt[:, k][:, None, None]
    return np.clip(np.rint(out), 0, 65535).astype(np.uint16)
