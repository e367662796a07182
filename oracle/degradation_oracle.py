"""numpy restatement of FFHQBlindDataset's degradation chain (basicsr/data/ffhq_blind_dataset.py:210-240) and of the
cv2 / libjpeg-turbo arithmetic it runs on.  TEST INFRASTRUCTURE: written from the algorithms, checked against cv2 on the CPU.

  filter2d_f64     cv2.filter2D(img f32, -1, kernel f64), BORDER_REFLECT_101, correlation anchored at the centre, as the
                   float64 direct sum in a fixed order, rounded once to float32 (cv2 filters a 41 x 41 kernel by DFT instead)
  resize_linear    cv2.resize(img f32, (w, h), INTER_LINEAR): source coordinate fma(d + 0.5, src / dst, -0.5) in float64,
                   floor, t = the rest as float32, clamped taps; the horizontal lerp fma(b - a, t, a), then the vertical one
  to_u8            cv2's saturate_cast<uchar>(float): round half to even, then clamp
  jpeg_roundtrip   cv2.imdecode(cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, q]), 1): baseline 4:2:0, islow DCTs,
                   libjpeg's fixed-point colour conversion, h2v2 downsampling with alternating bias, fancy upsampling
                   (replication when the chroma plane is at most 2 samples wide)
  degrade          the whole chain from uint8 GT and the parameters of codeformer_b200.degradation.sample_degradations
"""
from fractions import Fraction

import numpy as np

# ---------------------------------------------------------------------------------------------------------------- blur


def filter2d_f64(img, kernel, rows=None, cols=None):
    """Correlation of float32 HWC ``img`` with the float64 ``kernel`` (odd square), BORDER_REFLECT_101, rounded once to
    float32; only at ``rows`` x ``cols`` (all pixels by default).  The float64 sum runs over kernel rows, then columns, each
    product rounded before it is added -- the order of the device's blur, so the two agree bit for bit."""
    h, w = img.shape[:2]
    k = kernel.shape[0]
    r = k // 2
    rows = np.arange(h) if rows is None else np.asarray(rows)
    cols = np.arange(w) if cols is None else np.asarray(cols)

    def reflect(i, n):
        if n == 1:
            return np.zeros_like(i)
        i = np.abs(i)
        p = 2 * (n - 1)
        i = i % p
        return np.where(i >= n, p - i, i)
    acc = np.zeros((len(rows), len(cols)) + img.shape[2:], np.float64)
    src = img.astype(np.float64)
    for dy in range(k):
        ry = reflect(rows + dy - r, h)
        sub = src[ry]
        for dx in range(k):
            acc += kernel[dy, dx] * sub[:, reflect(cols + dx - r, w)]
    return acc.astype(np.float32)

# -------------------------------------------------------------------------------------------------------------- resize


def linear_taps(dst, src):
    """INTER_LINEAR taps of one axis: (i0, i1, t float32)."""
    i0 = np.empty(dst, np.int64)
    t = np.empty(dst, np.float32)
    scale = src / dst
    for d in range(dst):
        f = float(Fraction(2 * d + 1, 2) * Fraction(scale) - Fraction(1, 2))      # fma in float64: one rounding
        fl = np.floor(f)
        i0[d] = int(fl)
        t[d] = np.float32(f - fl)
    i1 = np.clip(i0 + 1, 0, src - 1)
    return np.clip(i0, 0, src - 1), i1, t


def fma32(x, y, z):
    """Correctly rounded float32 fma(x, y, z): the float64 product is exact; the float64 sum is made round-to-odd from its
    exact error (TwoSum), so that the final rounding to float32 is the only one."""
    p = x.astype(np.float64) * y.astype(np.float64)
    c = np.broadcast_to(z, p.shape).astype(np.float64)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    even = (s.view(np.int64) & 1) == 0
    s = np.where((err != 0) & even, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def _lerp(a, b, t):
    """fma(b - a, t, a) in float32."""
    return fma32((b - a).astype(np.float32), t, a)


def resize_linear(img, w, h):
    """cv2.resize(float32 HWC img, (w, h), interpolation=cv2.INTER_LINEAR)."""
    sh, sw = img.shape[:2]
    x0, x1, tx = linear_taps(w, sw)
    y0, y1, ty = linear_taps(h, sh)
    row = _lerp(img[:, x0], img[:, x1], tx[None, :, None])
    return _lerp(row[y0], row[y1], ty[:, None, None])


def to_u8(x):
    """saturate_cast<uchar>(float32): round half to even, clamp to 0..255."""
    return np.clip(np.rint(np.asarray(x, np.float32)), 0, 255).astype(np.uint8)

# ---------------------------------------------------------------------------------------------------------------- JPEG


_STD_LUMA = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                      14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                      49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)
_STD_CHROMA = np.array([17, 18, 24, 47] + [99] * 4 + [18, 21, 26, 66] + [99] * 4 + [24, 26, 56] + [99] * 5 + [47, 66] +
                       [99] * 38, np.int64)


def quant_tables(q):
    """libjpeg's jpeg_set_quality(q, force_baseline=TRUE): the Annex K tables scaled and clamped to 1..255 (row-major)."""
    q = min(max(int(q), 1), 100)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return [np.clip((t * scale + 50) // 100, 1, 255) for t in (_STD_LUMA, _STD_CHROMA)]


def _fix(x):
    return int(x * 65536 + 0.5)


def _rgb_to_ycc(r, g, b):
    half, off = 1 << 15, 128 << 16
    y = (_fix(0.299) * r + _fix(0.587) * g + _fix(0.114) * b + half) >> 16
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + off + half - 1) >> 16
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + off + half - 1) >> 16
    return y, cb, cr


_C = dict(c298=2446, c390=3196, c541=4433, c765=6270, c899=7373, c1175=9633, c1501=12299, c1847=15137, c1961=16069,
          c2053=16819, c2562=20995, c3072=25172)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, pass1):
    """One pass of libjpeg's jfdctint (islow) over axis -1 of int64 ``d``."""
    c = _C
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o = [None] * 8
    sh = 13 - 2 if pass1 else 13 + 2
    if pass1:
        o[0], o[4] = (t10 + t11) << 2, (t10 - t11) << 2
    else:
        o[0], o[4] = _descale(t10 + t11, 2), _descale(t10 - t11, 2)
    z1 = (t12 + t13) * c['c541']
    o[2] = _descale(z1 + t13 * c['c765'], sh)
    o[6] = _descale(z1 - t12 * c['c1847'], sh)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * c['c1175']
    t4, t5, t6, t7 = t4 * c['c298'], t5 * c['c2053'], t6 * c['c3072'], t7 * c['c1501']
    z1, z2, z3, z4 = -z1 * c['c899'], -z2 * c['c2562'], -z3 * c['c1961'] + z5, -z4 * c['c390'] + z5
    o[7] = _descale(t4 + z1 + z3, sh)
    o[5] = _descale(t5 + z2 + z4, sh)
    o[3] = _descale(t6 + z2 + z3, sh)
    o[1] = _descale(t7 + z1 + z4, sh)
    return np.stack(o, -1)


def _idct_1d(d, pass1):
    """One pass of libjpeg's jidctint (islow) over axis -1 of int64 ``d`` (already dequantised)."""
    c = _C
    z2, z3 = d[..., 2], d[..., 6]
    z1 = (z2 + z3) * c['c541']
    t2 = z1 - z3 * c['c1847']
    t3 = z1 + z2 * c['c765']
    t0 = (d[..., 0] + d[..., 4]) << 13
    t1 = (d[..., 0] - d[..., 4]) << 13
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    t0, t1, t2, t3 = d[..., 7], d[..., 5], d[..., 3], d[..., 1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * c['c1175']
    t0, t1, t2, t3 = t0 * c['c298'], t1 * c['c2053'], t2 * c['c3072'], t3 * c['c1501']
    z1, z2, z3, z4 = -z1 * c['c899'], -z2 * c['c2562'], -z3 * c['c1961'] + z5, -z4 * c['c390'] + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    sh = 13 - 2 if pass1 else 13 + 2 + 3
    o = [t10 + t3, t11 + t2, t12 + t1, t13 + t0, t13 - t0, t12 - t1, t11 - t2, t10 - t3]
    return np.stack([_descale(v, sh) for v in o], -1)


def _quantize(x, qv):
    """libjpeg-turbo's quantisation by the reciprocal of divisor = 8 q: ((|x| + c) * r) >> s, sign restored."""
    d = qv * 8
    b = np.floor(np.log2(d)).astype(np.int64)
    r = 16 + b
    fq = (np.int64(1) << r) // d
    fr = (np.int64(1) << r) % d
    c = d // 2
    exact = fr == 0
    fq = np.where(exact, fq >> 1, fq)
    r = np.where(exact, r - 1, r)
    c = np.where(~exact & (fr <= d // 2), c + 1, c)
    fq = np.where(~exact & (fr > d // 2), fq + 1, fq)
    a = np.abs(x)
    v = ((a + c) * fq) >> r
    return np.where(x < 0, -v, v)


def _code_blocks(plane, qv):
    """Blocks [.., 8, 8] of centred samples -> decoded samples 0..255 (FDCT, quantise, dequantise, IDCT, range limit)."""
    f = _fdct_1d(plane, True)
    f = np.swapaxes(_fdct_1d(np.swapaxes(f, -1, -2), False), -1, -2)
    coef = _quantize(f, qv.reshape(8, 8)) * qv.reshape(8, 8)
    w = np.swapaxes(_idct_1d(np.swapaxes(coef, -1, -2), True), -1, -2)
    return np.clip(_idct_1d(w, False) + 128, 0, 255)


def _blocks(p):
    H, W = p.shape
    return p.reshape(H // 8, 8, W // 8, 8).swapaxes(1, 2)


def _unblocks(b):
    n, m = b.shape[:2]
    return b.swapaxes(1, 2).reshape(n * 8, m * 8)


def jpeg_roundtrip(img, q):
    """uint8 BGR HWC -> the uint8 BGR image cv2 decodes from cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, q])."""
    h, w = img.shape[:2]
    lq, cq = quant_tables(q)
    px = img.astype(np.int64)
    y, cb, cr = _rgb_to_ycc(px[..., 2], px[..., 1], px[..., 0])
    # luma: edge replication to whole 8 x 8 blocks
    yh, yw = -(-h // 8) * 8, -(-w // 8) * 8
    yp = np.pad(y, ((0, yh - h), (0, yw - w)), mode='edge')
    yd = _unblocks(_code_blocks(_blocks(yp - 128), lq))[:h, :w]
    # chroma: rows and columns clamped to the image, h2v2 average with bias 1, 2, 1, 2, ... along each row; rows of the
    # padded chroma plane beyond ceil(h / 2) repeat the last real one
    ch, cw = -(-h // 16) * 8, -(-w // 16) * 8
    rh, rw = -(-h // 2), -(-w // 2)
    ry = np.minimum(np.arange(2 * ch), h - 1)
    rx = np.minimum(np.arange(2 * cw), w - 1)
    bias = np.where(np.arange(cw) % 2 == 0, 1, 2)
    out = []
    for c in (cb, cr):
        full = c[ry][:, rx]
        ds = (full[0::2, 0::2] + full[0::2, 1::2] + full[1::2, 0::2] + full[1::2, 1::2] + bias[None]) >> 2
        ds[rh:] = ds[rh - 1]
        dec = _unblocks(_code_blocks(_blocks(ds - 128), cq))[:rh, :rw]
        if rw <= 2:             # libjpeg-turbo upsamples by replication unless the chroma plane is wider than 2 samples
            out.append(dec.repeat(2, 0).repeat(2, 1)[:h, :w])
            continue
        # fancy upsampling: column sums 3 * near + far row, then 3 * near + far column, biases 8 / 7
        up = np.minimum(np.arange(rh) + 1, rh - 1)
        dn = np.maximum(np.arange(rh) - 1, 0)
        cs = np.empty((2 * rh, rw), np.int64)
        cs[0::2] = 3 * dec + dec[dn]
        cs[1::2] = 3 * dec + dec[up]
        lf = np.maximum(np.arange(rw) - 1, 0)
        rt = np.minimum(np.arange(rw) + 1, rw - 1)
        o = np.empty((2 * rh, 2 * rw), np.int64)
        o[:, 0::2] = (3 * cs + cs[:, lf] + 8) >> 4
        o[:, 1::2] = (3 * cs + cs[:, rt] + 7) >> 4
        out.append(o[:h, :w])
    cbu, cru = out[0] - 128, out[1] - 128
    half = 1 << 15
    r = yd + ((_fix(1.402) * cru + half) >> 16)
    g = yd + ((-_fix(0.34414) * cbu + half - _fix(0.71414) * cru) >> 16)
    b = yd + ((_fix(1.772) * cbu + half) >> 16)
    return np.clip(np.stack([b, g, r], -1), 0, 255).astype(np.uint8)

# --------------------------------------------------------------------------------------------------------------- chain


def degrade(gt_u8, p, in_size):
    """One face: uint8 BGR [S, S, 3] and one entry of sample_degradations -> (lq uint8 [in, in, 3], stage-a float32 image,
    pre-JPEG uint8 image or None).  The blur is evaluated only where the resize reads it."""
    S = gt_u8.shape[0]
    s = p['size']
    img = (gt_u8.astype(np.float32) / np.float32(255.)).astype(np.float32)
    y0, y1, ty = linear_taps(s, S)
    rows = np.unique(np.concatenate([y0, y1]))
    blur = filter2d_f64(img, p['kernel'], rows, rows)
    full = np.zeros((S, S, 3), np.float32)
    full[np.ix_(rows, rows)] = blur
    x = resize_linear(full, s, s)
    stage_a = x
    if p['noise'] is not None:
        x = np.clip((x + p['noise']).astype(np.float32), 0, 1)
    pre = None
    if p['quality'] is not None:
        pre = to_u8(x * np.float32(255.))
        x = (jpeg_roundtrip(pre, p['quality']).astype(np.float32) / np.float32(255.)).astype(np.float32)
    x = resize_linear(x, in_size, in_size)
    return to_u8(x * np.float32(255.)), stage_a, pre
