"""CPU oracle for whole-image paste-back -- TEST INFRASTRUCTURE, NOT PRODUCT CODE (only tests/ and tools/ import it).

numpy restatement of ``FaceRestoreHelper.align_warp_face`` and ``paste_faces_to_input_image``
(/root/reference/facelib/utils/face_restoration_helper.py:319-349, 372-516) and of the cv2 primitives they call:
``warpAffine`` (bilinear u8 / f32 / f64, fixed-point coordinates), ``resize(INTER_LINEAR)`` (u8 and f64),
``erode`` with a rectangular kernel, ``getGaussianKernel`` and ``GaussianBlur`` (separable, BORDER_REFLECT_101) and
``invertAffineTransform``.  The float64 resize and the blurs are cv2's fused multiply-adds, so they call the C restatement in
oracle/c/oracle_kernels.c (built by oracle/build_c.py).  ``paste_faces`` returns the canvas BEFORE the final ``astype(uint8)`` so the tests can compare
continuously.  tests/test_oracle_pasteback.py pins every primitive against cv2 and the whole step against
tests/golden/pasteback.npz, written from the UNMODIFIED reference by oracle/gen_golden_pasteback.py.
"""
import ctypes
import functools

import numpy as np

BORDER_CONSTANT, BORDER_REFLECT, BORDER_REFLECT101 = 0, 2, 4


@functools.lru_cache(None)
def _clib():
    """The C restatements (oracle/build_c.py): numpy has no fused multiply-add, and cv2's filters use it."""
    from oracle import build_c
    return build_c.load()


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)
MASK_COLORMAP = np.array([0, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 0, 255, 0, 0, 0], np.uint8)


def invert_affine(M):
    """cv2.invertAffineTransform in double."""
    M = np.asarray(M, np.float64)
    D = M[0, 0] * M[1, 1] - M[0, 1] * M[1, 0]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22, A12, A21 = M[1, 1] * D, M[0, 0] * D, -M[0, 1] * D, -M[1, 0] * D
    b1 = -A11 * M[0, 2] - A12 * M[1, 2]
    b2 = -A21 * M[0, 2] - A22 * M[1, 2]
    return np.array([[A11, A12, b1], [A21, A22, b2]], np.float64)


def border_index(p, n, mode):
    """cv2.borderInterpolate for REFLECT / REFLECT_101; CONSTANT gives -1 outside [0, n)."""
    p = np.asarray(p, np.int64)
    if mode == BORDER_CONSTANT:
        return np.where((p >= 0) & (p < n), p, -1)
    if mode == BORDER_REFLECT101:
        if n == 1:
            return np.zeros_like(p)
        per = 2 * (n - 1)
        q = np.mod(p, per)
        return np.where(q >= n, per - q, q)
    per = 2 * n
    q = np.mod(p, per)
    return np.where(q >= n, per - 1 - q, q)


def warp_coords(M, dsize):
    """Fixed-point source coordinates of cv2.warpAffine (no WARP_INVERSE_MAP): integer part and 1/32 fraction.  cv2 stores
    the integer part as int16 (saturate_cast<short>), which a near-singular matrix reaches; the fraction keeps its bits."""
    dw, dh = dsize
    A = invert_affine(M)
    x = np.arange(dw, dtype=np.float64)
    y = np.arange(dh, dtype=np.float64)
    adelta = np.rint(A[0, 0] * x * 1024).astype(np.int64)
    bdelta = np.rint(A[1, 0] * x * 1024).astype(np.int64)
    X0 = np.rint((A[0, 1] * y + A[0, 2]) * 1024).astype(np.int64) + 16
    Y0 = np.rint((A[1, 1] * y + A[1, 2]) * 1024).astype(np.int64) + 16
    X = (X0[:, None] + adelta[None, :]) >> 5
    Y = (Y0[:, None] + bdelta[None, :]) >> 5
    return np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767), X & 31, Y & 31


def _gather(src, ys, xs, mode, cval):
    """src[ys, xs] with the border rule; src is [h, w] or [h, w, c]."""
    h, w = src.shape[:2]
    yi, xi = border_index(ys, h, mode), border_index(xs, w, mode)
    ok = (yi >= 0) & (xi >= 0)
    v = src[np.maximum(yi, 0), np.maximum(xi, 0)]
    if mode == BORDER_CONSTANT:
        cv = np.asarray(cval, dtype=src.dtype).reshape((1,) * ok.ndim + (-1,)) if src.ndim == 3 else src.dtype.type(cval)
        v = np.where(ok[..., None] if src.ndim == 3 else ok, v, cv)
    return v


def warp_linear_u8(src, M, dsize, mode=BORDER_CONSTANT, cval=(0, 0, 0)):
    """cv2.warpAffine(src u8 HWC, M, dsize, INTER_LINEAR, mode, cval): weights (32-fy)(32-fx)*32 ..., (sum + 2^14) >> 15."""
    ix, iy, fx, fy = warp_coords(M, dsize)
    fx, fy = fx[..., None], fy[..., None]
    w = [(32 - fy) * (32 - fx) * 32, (32 - fy) * fx * 32, fy * (32 - fx) * 32, fy * fx * 32]
    acc = np.zeros(ix.shape + (src.shape[2],), np.int64)
    for k, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        acc += _gather(src, iy + dy, ix + dx, mode, cval).astype(np.int64) * w[k]
    return np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def warp_linear_float(src, M, dsize):
    """cv2.warpAffine(src f32 / f64 2-D, M, dsize) with BORDER_CONSTANT 0: ((v0 w0 + v1 w1) + v2 w2) + v3 w3 in src's dtype,
    with the exact float32 weights (1-b)(1-a), (1-b)a, b(1-a), ba at a, b = i/32.  flags=3 (the parse mask) is INTER_AREA,
    which warpAffine runs as INTER_LINEAR."""
    ix, iy, fx, fy = warp_coords(M, dsize)
    a, b = fx.astype(np.float32) / np.float32(32), fy.astype(np.float32) / np.float32(32)
    one = np.float32(1)
    w = [(one - b) * (one - a), (one - b) * a, b * (one - a), b * a]
    acc = None
    for k, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        t = _gather(src, iy + dy, ix + dx, BORDER_CONSTANT, 0) * w[k].astype(src.dtype)
        acc = t if acc is None else (acc + t).astype(src.dtype)
    return acc


def _linear_taps(dst, src, dtype):
    scale = 1.0 / (dst / src)
    f = ((np.arange(dst) + 0.5) * scale - 0.5).astype(np.float32)
    i = np.floor(f).astype(np.int64)
    return i, (f - i.astype(np.float32)).astype(np.float32)


def resize_linear_u8(src, dsize):
    """cv2.resize(src u8 HWC, dsize, INTER_LINEAR): 11-bit weights, horizontal clamped, vertical not; an exact halving
    is INTER_AREA's 2x2 mean (cv2 switches to it)."""
    dw, dh = dsize
    h, w = src.shape[:2]
    if (dw, dh) == (w, h):
        return src.copy()
    if w == 2 * dw and h == 2 * dh:
        s = src.astype(np.int32)
        return ((s[0::2, 0::2] + s[0::2, 1::2] + s[1::2, 0::2] + s[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    sx, fx = _linear_taps(dw, w, np.float32)
    lo, hi = sx < 0, sx >= w - 1
    fx = np.where(lo | hi, np.float32(0), fx)
    sx = np.where(lo, 0, np.where(hi, w - 1, sx))
    a0 = np.rint((np.float32(1) - fx) * np.float32(2048)).astype(np.int64)
    a1 = np.rint(fx * np.float32(2048)).astype(np.int64)
    s = src.astype(np.int64)
    row = s[:, sx] * a0[None, :, None] + s[:, np.minimum(sx + 1, w - 1)] * a1[None, :, None]
    sy, fy = _linear_taps(dh, h, np.float32)
    b0 = np.rint((np.float32(1) - fy) * np.float32(2048)).astype(np.int64)
    b1 = np.rint(fy * np.float32(2048)).astype(np.int64)
    r0 = row[np.clip(sy, 0, h - 1)] >> 4
    r1 = row[np.clip(sy + 1, 0, h - 1)] >> 4
    out = (((b0[:, None, None] * r0) >> 16) + ((b1[:, None, None] * r1) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


def resize_linear_f64(src, dsize):
    """cv2.resize(src f64 2-D, dsize, INTER_LINEAR), both sides >= 2: double coordinates and lerp FMAs (resize_linear_f64_ref
    in oracle/c/oracle_kernels.c)."""
    dw, dh = dsize
    h, w = src.shape
    if (dw, dh) == (w, h):
        return src.copy()
    src = np.ascontiguousarray(src, np.float64)
    out = np.empty((dh, dw), np.float64)
    _clib().resize_linear_f64_ref(_ptr(src), h, w, _ptr(out), dh, dw)
    return out


def erode_rect(src, k):
    """cv2.erode(src 2-D, np.ones((k, k))): anchor k // 2, pixels outside the image never erode; k == 0 erodes 3x3."""
    if k == 0:
        k = 3
    a = k // 2
    h, w = src.shape
    big = np.inf
    pad = np.full((h, w + k - 1), big, src.dtype)
    pad[:, a:a + w] = src
    r = pad[:, 0:w].copy()
    for j in range(1, k):
        r = np.minimum(r, pad[:, j:j + w])
    pad = np.full((h + k - 1, w), big, src.dtype)
    pad[a:a + h] = r
    out = pad[0:h].copy()
    for i in range(1, k):
        out = np.minimum(out, pad[i:i + h])
    return out


_SMALL_GAUSS = {1: [1.0], 3: [0.25, 0.5, 0.25], 5: [0.0625, 0.25, 0.375, 0.25, 0.0625],
                7: [0.03125, 0.109375, 0.21875, 0.28125, 0.21875, 0.109375, 0.03125],
                9: [0.015625, 0.05078125, 0.1171875, 0.19921875, 0.234375, 0.19921875, 0.1171875, 0.05078125, 0.015625]}


# cv2.getGaussianKernel(101, 11, CV_64F), taps 0 .. 50 (the rest mirror them): cv2 exponentiates in its software double,
# whose last bit numpy's exp does not always reproduce.  The parse mask's blur uses it; csrc/pasteback.cu holds the same table.
PARSE_KERNEL_HALF = [float.fromhex(v) for v in (
    '0x1.3d9320997c25bp-20', '0x1.de17a7bf38417p-20', '0x1.64e8ed67fb58cp-19', '0x1.08402ac73792fp-18',
    '0x1.8412e6ca94be9p-18', '0x1.1a9d258b611acp-17', '0x1.983ce6e2d8b48p-17', '0x1.246cb61c4022cp-16',
    '0x1.9f7c2e4f210b2p-16', '0x1.24bcaeb80f233p-15', '0x1.991c4ec5d6f8ep-15', '0x1.1b85423e811abp-14',
    '0x1.85bc1908d022ep-14', '0x1.09aa455fcb2a8p-13', '0x1.673421a12de51p-13', '0x1.e1add23bf2656p-13',
    '0x1.404c85f10d7b6p-12', '0x1.a677dc2924522p-12', '0x1.1452178d2dfc5p-11', '0x1.667cb15ebc175p-11',
    '0x1.cd4230959cfabp-11', '0x1.264dd24853bf3p-10', '0x1.7477bd22f281bp-10', '0x1.d382d89d4adafp-10',
    '0x1.22fd1739f5a24p-9', '0x1.6740df70cfe47p-9', '0x1.b7e1e31cfeb7cp-9', '0x1.0b165029af448p-8',
    '0x1.41ab7619e5c97p-8', '0x1.8037efebc0c46p-8', '0x1.c727155fbb708p-8', '0x1.0b5f5ae5abc27p-7',
    '0x1.378ad7eba8e32p-7', '0x1.680578de9fdf6p-7', '0x1.9c9eb782d6717p-7', '0x1.d502d0b5254c3p-7',
    '0x1.085c4a7f64ae8p-6', '0x1.27904729ecf7bp-6', '0x1.47bada6c7b599p-6', '0x1.6867edea4945bp-6',
    '0x1.8913f51fae714p-6', '0x1.a92eec6952cc7p-6', '0x1.c82029c32f07fp-6', '0x1.e54ae009f9925p-6',
    '0x1.0009941ac006fp-5', '0x1.0bf1ac50126f9p-5', '0x1.1618b501c3bf9p-5', '0x1.1e421299af7d2p-5',
    '0x1.243bea305ece7p-5', '0x1.27e11b8751b9cp-5', '0x1.291ac05d51e68p-5',
)]


def gaussian_kernel(n, sigma, dtype):
    """cv2.getGaussianKernel(n, sigma, CV_32F / CV_64F); the float64 kernel is exact for the parse mask's (101, 11) and within an
    ulp otherwise."""
    if sigma <= 0 and n in _SMALL_GAUSS:
        return np.array(_SMALL_GAUSS[n], dtype)
    if (n, sigma) == (101, 11) and np.dtype(dtype) == np.float64:
        return np.array(PARSE_KERNEL_HALF + PARSE_KERNEL_HALF[-2::-1], np.float64)
    sig = sigma if sigma > 0 else n * 0.15 + 0.35
    scale2 = -0.125 / (sig * sig)
    n2 = (n - 1) // 2
    vals = [np.exp(float((x * x)) * scale2) for x in range(1 - n, 1 - n + 2 * n2, 2)]
    s = 0.0
    for v in vals:
        s += v
    s = s * 2 + 1.0
    mul = 1.0 / s
    half = [v * mul for v in vals]
    k = np.array(half + [mul] + half[::-1], np.float64)
    return k.astype(dtype)


def blur_reflect101(src, kern):
    """cv2.GaussianBlur(src, (n, n), ...) = sepFilter2D(src, kern, kern, BORDER_REFLECT_101) in src's dtype (float32 or
    float64), both sides >= 2: cv2 4.13's x86-64 AVX2 arithmetic, restated in C with its fused multiply-adds
    (gauss_blur_f32_ref / gauss_blur_f64_ref in oracle/c/oracle_kernels.c)."""
    src = np.ascontiguousarray(src)
    kern = np.ascontiguousarray(kern, src.dtype)
    fn = {np.dtype(np.float32): 'gauss_blur_f32_ref', np.dtype(np.float64): 'gauss_blur_f64_ref'}[src.dtype]
    out, tmp = np.empty_like(src), np.empty_like(src)
    getattr(_clib(), fn)(_ptr(src), _ptr(out), _ptr(tmp), src.shape[0], src.shape[1], _ptr(kern), len(kern))
    return out


def parse_soft_mask(parse_u8):
    """The parse mask of paste_faces_to_input_image:472-480 (before the resize): two (101,101)/11 blurs in float64, the
    10-pixel border zeroed, /255."""
    pm = parse_u8.astype(np.float64)
    k = gaussian_kernel(101, 11, np.float64)
    pm = blur_reflect101(blur_reflect101(pm, k), k)
    pm[:10, :] = 0
    pm[-10:, :] = 0
    pm[:, :10] = 0
    pm[:, -10:] = 0
    return pm / 255.


def face_roi(inverse_affine, face_size, h_up, w_up, pad=2):
    """(x0, y0, x1, y1) of the canvas pixels a face can touch: the face square grown by 2 source pixels (beyond the
    bilinear footprint), mapped by the inverse affine, grown by `pad` canvas pixels, clipped.  Outside it every warp is 0."""
    A = np.asarray(inverse_affine, np.float64)
    c = np.array([[-2, -2, 1], [face_size + 2, -2, 1], [-2, face_size + 2, 1], [face_size + 2, face_size + 2, 1]], np.float64)
    p = c @ A.T
    x0 = max(int(np.floor(p[:, 0].min())) - pad, 0)
    y0 = max(int(np.floor(p[:, 1].min())) - pad, 0)
    x1 = min(int(np.ceil(p[:, 0].max())) + pad + 1, w_up)
    y1 = min(int(np.ceil(p[:, 1].max())) + pad + 1, h_up)
    return x0, y0, max(x1, x0), max(y1, y0)


def paste_faces(input_img, restored_faces, inverse_affines, upscale, parse_masks=None, upsample_img=None, face_size=512,
                face_upsampler=None, return_info=False):
    """paste_faces_to_input_image:372-499 up to (not including) the astype(uint8).  parse_masks: per face the uint8
    0/255 MASK_COLORMAP image of the parsing network's argmax (the network itself is the caller's), or None for
    use_parse=False.  inverse_affines are adjusted in place as the reference does.  Returns the float canvas
    (float64 with parse masks, float32 without) and, with return_info, per face dict(w_edge, soft, roi)."""
    h, w = input_img.shape[:2]
    h_up, w_up = int(h * upscale), int(w * upscale)
    canvas = resize_linear_u8(input_img, (w_up, h_up)) if upsample_img is None else upsample_img
    info = []
    for i, (face, inv) in enumerate(zip(restored_faces, inverse_affines)):
        if face_upsampler is not None:
            face = face_upsampler(face)
            inv /= upscale
            inv[:, 2] *= upscale
            fs = face_size * upscale
        else:
            inv[:, 2] += 0.5 * upscale if upscale > 1 else 0
            fs = face_size
        inv_restored = warp_linear_u8(face, inv, (w_up, h_up))
        inv_mask = warp_linear_float(np.ones((fs, fs), np.float32), inv, (w_up, h_up))
        erosion = erode_rect(inv_mask, int(2 * upscale))
        pasted = erosion[:, :, None] * inv_restored
        area = np.sum(erosion, dtype=np.float64)
        w_edge = int(area ** 0.5) // 20
        center = erode_rect(erosion, w_edge * 2)
        soft = blur_reflect101(center, gaussian_kernel(2 * w_edge + 1, 0, np.float32))
        m = soft[:, :, None]
        if parse_masks is not None:
            pm = resize_linear_f64(parse_soft_mask(parse_masks[i]), (fs, fs))
            pm = warp_linear_float(pm, inv, (w_up, h_up))[:, :, None]
            m = np.where(pm < m, pm, m.astype(np.float64))
        canvas = m * pasted + (1 - m) * canvas
        info.append(dict(w_edge=w_edge, soft=m[:, :, 0], roi=face_roi(inv, fs, h_up, w_up), area=area))
    return (canvas, info) if return_info else canvas


def to_u8(canvas):
    """astype(np.uint8) of a float canvas as numpy does it on x86: truncate, then keep the low byte."""
    return np.trunc(canvas).astype(np.int64).astype(np.uint8)


# ---- synthetic whole-image inputs (tests/golden/pasteback.npz stores only their parameters) ----------------------
def synthetic_background(h, w, seed):
    """A smooth BGR background from integer triangle waves: every platform reproduces it bit for bit."""
    y, x = np.mgrid[0:h, 0:w].astype(np.int64)
    img = np.empty((h, w, 3), np.int64)
    for c in range(3):
        p = 61 + 17 * c + seed
        v = ((3 + 2 * c + seed % 5) * x + (5 + c + seed % 3) * y) % (2 * p)
        v2 = ((c + 2) * x + (seed % 4 + 1) * y) % 94
        img[..., c] = 40 + np.abs(v - p) * 160 // p + np.abs(v2 - 47)
    return np.clip(img, 0, 255).astype(np.uint8)


def synthetic_input(faces_bgr, placements, h, w, seed):
    """faces_bgr[i] warped by T (face -> image, bilinear) over synthetic_background where the warped square covers > 1/2."""
    img = synthetic_background(h, w, seed)
    ones = np.ones(faces_bgr.shape[1:3], np.float32)
    for i, T in placements:
        warped = warp_linear_u8(faces_bgr[i], T, (w, h))
        m = warp_linear_float(ones, T, (w, h)) > 0.5
        img[m] = warped[m]
    return img


def synthetic_upsample(img, up):
    """A stand-in for a background upsampler's output: nearest x`up` plus a fixed integer ripple."""
    r = np.repeat(np.repeat(img, up, axis=0), up, axis=1).astype(np.int16)
    y, x = np.mgrid[0:r.shape[0], 0:r.shape[1]]
    return np.clip(r + (((x * 7 + y * 13) % 17) - 8)[..., None], 0, 255).astype(np.uint8)


def sample_index(size, n=5000):
    """Spread-out flat indices of the canvas samples the golden keeps."""
    return (np.arange(n, dtype=np.int64) * 2654435761) % size


def golden_case(g, faces_bgr, case, up):
    """Rebuild a case of tests/golden/pasteback.npz: (input image, upsample_img or None, background, reference uint8 result)."""
    h, w, seed = (int(v) for v in g[f'{case}_input'])
    img = synthetic_input(faces_bgr, list(zip(g[f'{case}_faces'], g[f'{case}_T'])), h, w, seed)
    upsample = synthetic_upsample(img, up) if case == 'P3' else None
    bg = resize_linear_u8(img, (w * up, h * up)) if upsample is None else upsample
    return img, upsample, bg, bg + g[f'{case}_delta']
