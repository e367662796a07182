"""CPU oracle for ``cv2.resize(..., interpolation=INTER_AREA)`` of uint8 images -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy restatement of the two shrinking paths of cv2's INTER_AREA (imgproc/src/resize.cpp) for uint8 HWC images:

  * ``resizeAreaFast`` when both inverse scales are integers (|scale - round(scale)| < DBL_EPSILON): integer window sums;
    an exact 2 x 2 halving rounds as ``(sum + 2) >> 2``, any other window as ``cvRound(float(sum) * (1.f / area))``.
  * the general path: ``computeResizeAreaTab`` weights in double (stored as float), every source row reduced to a float
    row buffer tap by tap (``buf += S * alpha``), the rows of one output row summed in float (``sum += beta * buf``) in
    table order, then ``saturate_cast<uchar>`` (round half to even, clamp).

``scale`` is ``1. / (dsize / ssize)`` in double, as cv::resize computes it from an explicit dsize.
tests/test_oracle_resize_area.py pins this restatement against cv2 on the CPU.
"""
import numpy as np

DBL_EPSILON = np.finfo(np.float64).eps


def inverse_scale(src_len, dst_len):
    """cv::resize's scale for an explicit dsize: 1 / (dst / src) in double."""
    return 1.0 / (float(dst_len) / float(src_len))


def is_area_fast(scale_x, scale_y):
    """The integer-factor test of cv::resize (iscale = saturate_cast<int>(scale), i.e. round half to even)."""
    ix, iy = int(np.rint(scale_x)), int(np.rint(scale_y))
    return abs(scale_x - ix) < DBL_EPSILON and abs(scale_y - iy) < DBL_EPSILON, ix, iy


def area_tab(ssize, dsize, scale):
    """computeResizeAreaTab: a list of (dst index, src index, float32 weight) in cv2's order."""
    tab = []
    for dx in range(dsize):
        fsx1 = dx * scale
        fsx2 = fsx1 + scale
        cell = min(scale, ssize - fsx1)
        sx1, sx2 = int(np.ceil(fsx1)), int(np.floor(fsx2))
        sx2 = min(sx2, ssize - 1)
        sx1 = min(sx1, sx2)
        if sx1 - fsx1 > 1e-3:
            tab.append((dx, sx1 - 1, np.float32((sx1 - fsx1) / cell)))
        for sx in range(sx1, sx2):
            tab.append((dx, sx, np.float32(1.0 / cell)))
        if fsx2 - sx2 > 1e-3:
            tab.append((dx, sx2, np.float32(min(min(fsx2 - sx2, 1.0), cell) / cell)))
    return tab


def tap_arrays(ssize, dsize, scale):
    """The table as [dsize, K] source indices and float32 weights (weight 0 pads the shorter rows: adding 0 * S is exact)."""
    tab = area_tab(ssize, dsize, scale)
    counts = np.zeros(dsize, np.int64)
    for d, _, _ in tab:
        counts[d] += 1
    K = int(counts.max()) if dsize else 0
    idx = np.zeros((dsize, K), np.int64)
    wt = np.zeros((dsize, K), np.float32)
    fill = np.zeros(dsize, np.int64)
    for d, s, a in tab:
        idx[d, fill[d]] = s
        wt[d, fill[d]] = a
        fill[d] += 1
    return idx, wt, counts


def _round_u8(v):
    return np.clip(np.rint(v), 0, 255).astype(np.uint8)


def resize_area_fast(src, sx, sy):
    h, w = src.shape[:2]
    oh, ow = h // sy, w // sx
    s = src[:oh * sy, :ow * sx].astype(np.int64).reshape(oh, sy, ow, sx, -1).sum(axis=(1, 3))
    if sx == 2 and sy == 2:
        return ((s + 2) >> 2).astype(np.uint8)
    scale = np.float32(1) / np.float32(sx * sy)
    return _round_u8(s.astype(np.float32) * scale)


def resize_area_general(src, dsize, scale_x, scale_y):
    h, w = src.shape[:2]
    ow, oh = dsize
    xi, xw, _ = tap_arrays(w, ow, scale_x)
    ytab = area_tab(h, oh, scale_y)
    S = src.astype(np.float32)
    buf = np.zeros((h, ow, src.shape[2]), np.float32)
    for t in range(xi.shape[1]):                         # buf[dx] = ((0 + S a0) + S a1) + ...
        buf = buf + S[:, xi[:, t]] * xw[:, t][None, :, None]
    out = np.zeros((oh, ow, src.shape[2]), np.float32)
    started = np.zeros(oh, bool)
    for dy, sy, beta in ytab:                             # sum = beta0 buf0; sum += beta_k buf_k
        term = np.float32(beta) * buf[sy]
        out[dy] = term if not started[dy] else out[dy] + term
        started[dy] = True
    return _round_u8(out)


def resize_area_u8(src, dsize):
    """cv2.resize(src, dsize, interpolation=cv2.INTER_AREA) for a uint8 [h, w, c] image with dsize = (w', h') <= (w, h)."""
    src = np.asarray(src)
    assert src.dtype == np.uint8 and src.ndim == 3
    h, w = src.shape[:2]
    ow, oh = dsize
    assert 0 < ow <= w and 0 < oh <= h, 'shrinking only'
    if (ow, oh) == (w, h):
        return src.copy()
    scale_x, scale_y = inverse_scale(w, ow), inverse_scale(h, oh)
    fast, ix, iy = is_area_fast(scale_x, scale_y)
    if fast:
        return resize_area_fast(src, ix, iy)
    return resize_area_general(src, dsize, scale_x, scale_y)


def detection_size(h, w, resize=640):
    """``get_face_landmarks_5(resize=...)``'s target: scale = resize / min(h, w) in double, (int(h scale), int(w scale))."""
    scale = resize / min(h, w)
    return int(h * scale), int(w * scale), scale
