"""CPU oracle for ``cv2.resize(..., interpolation=INTER_LANCZOS4)`` of uint8 images -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy restatement of cv2's fixed-point Lanczos-4 resize (imgproc/src/resize.cpp) for uint8 HWC images, enlarging or shrinking,
with independent factors per axis:

  * per output coordinate d the source coordinate is ``f = (d + 0.5) * scale - 0.5`` rounded to float32 with
    ``scale = 1 / (dst / src)`` in double; ``s = floor(f)`` and the eight taps sit at ``s - 3 .. s + 4``, each clamped to the image;
  * the float32 weights come from one sin / cos of ``-(frac + 3) pi / 4`` rotated by multiples of 45 degrees, each divided by
    its own ``y * y`` (y rounded to float32), normalised by their float32 sum; ``frac < FLT_EPSILON`` is the unit tap;
  * the weights are scaled by 2048 and saturated to int16 (no renormalisation), a horizontal pass sums into int32 and the
    vertical pass rounds with ``(v + 2^21) >> 22`` and saturates to uint8.

tests/test_oracle_lanczos_gray.py pins this restatement against cv2 on the CPU and the tables of ``cfb_lanczos4_table``
against ``tap_table``.
"""
import numpy as np

FLT_EPSILON = np.float32(1.1920929e-07)
S45 = 0.70710678118654752440084436210485
ROT = ((1, 0), (-S45, -S45), (0, 1), (S45, -S45), (-1, 0), (S45, S45), (0, -1), (-S45, S45))


def lanczos4_coeffs(frac):
    """The eight float32 weights of one fractional offset (a float32 in [0, 1))."""
    c = np.zeros(8, np.float32)
    if frac < FLT_EPSILON:
        c[3] = 1
        return c
    x = float(frac)
    y0 = -(x + 3) * np.pi * 0.25
    s0, c0 = np.sin(y0), np.cos(y0)
    total = np.float32(0)
    for i in range(8):
        y = float(np.float32(-(x + 3 - i) * np.pi * 0.25))
        c[i] = np.float32((ROT[i][0] * s0 + ROT[i][1] * c0) / (y * y))
        total = np.float32(total + c[i])
    return c * (np.float32(1) / total)


def tap_table(src_len, dst_len):
    """-> (idx [dst_len] int32: floor of the source coordinate, coef [dst_len, 8] int16: the weights * 2048)."""
    scale = 1.0 / (float(dst_len) / float(src_len))
    idx = np.zeros(dst_len, np.int32)
    coef = np.zeros((dst_len, 8), np.int16)
    for d in range(dst_len):
        f = np.float32((d + 0.5) * scale - 0.5)
        s = int(np.floor(f))
        idx[d] = s
        w = lanczos4_coeffs(np.float32(f - np.float32(s)))
        coef[d] = np.clip(np.rint(w * np.float32(2048)), -32768, 32767).astype(np.int16)
    return idx, coef


def resize_lanczos4_u8(src, dsize):
    """cv2.resize(src, dsize, interpolation=cv2.INTER_LANCZOS4) for a uint8 [h, w, c] image, dsize = (w', h')."""
    src = np.asarray(src)
    assert src.dtype == np.uint8 and src.ndim == 3
    h, w = src.shape[:2]
    ow, oh = dsize
    if (ow, oh) == (w, h):
        return src.copy()
    xi, xt = tap_table(w, ow)
    yi, yt = tap_table(h, oh)
    s = src.astype(np.int64)
    rows = np.zeros((h, ow, src.shape[2]), np.int64)
    for k in range(8):
        rows += s[:, np.clip(xi - 3 + k, 0, w - 1)] * xt[:, k].astype(np.int64)[None, :, None]
    out = np.zeros((oh, ow, src.shape[2]), np.int64)
    for k in range(8):
        out += rows[np.clip(yi - 3 + k, 0, h - 1)] * yt[:, k].astype(np.int64)[:, None, None]
    return np.clip((out + (1 << 21)) >> 22, 0, 255).astype(np.uint8)
