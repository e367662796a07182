"""The numpy paste-back oracle (oracle/pasteback_oracle.py) against cv2 and against the reference golden.  CPU only.

The golden comparisons need no cv2.  The blur and float64 resize comparisons hold the oracle to cv2 4.13 bit for bit as
built for x86-64 with its AVX2 dispatch (the PyPI wheels): which outputs take cv2's fused multiply-adds depends on its SIMD
blocks, so another build of cv2 fails them, with a message that says so."""
import hashlib
import os
import platform
import re

import numpy as np
import pytest

from oracle import pasteback_oracle as O

try:
    import cv2
except ImportError:
    cv2 = None
needs_cv2 = pytest.mark.skipif(cv2 is None, reason='needs cv2')
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
PASTEBACK_CU = os.path.join(os.path.dirname(__file__), '..', 'codeformer_b200', 'csrc', 'pasteback.cu')


def require_x86_avx2_cv2():
    """The restated filter arithmetic is cv2's x86-64 AVX2 code path: fail clearly on another cv2 build."""
    # 11 is cv::CPU_AVX2, which the Python bindings do not export
    probe = np.random.default_rng(0).random((9, 13)).astype(np.float32)
    same = np.array_equal(O.blur_reflect101(probe, O.gaussian_kernel(7, 0, np.float32)), cv2.GaussianBlur(probe, (7, 7), 0))
    if not (platform.machine().lower() in ('x86_64', 'amd64') and cv2.checkHardwareSupport(11) and same):
        pytest.fail(f'cv2 {cv2.__version__} on {platform.machine()} does not run the x86-64 AVX2 filter arithmetic that '
                    'oracle/c/oracle_kernels.c restates (cv2 4.13 wheels on an AVX2 CPU); its blur differs in the last bit')


def similarity(rng, w, h):
    a, s = rng.uniform(-0.35, 0.35), rng.uniform(0.4, 3.0)
    c, si = np.cos(a) * s, np.sin(a) * s
    return np.array([[c, -si, rng.uniform(-w / 2, w / 2)], [si, c, rng.uniform(-h / 2, h / 2)]])


@needs_cv2
@pytest.mark.parametrize('mode', [O.BORDER_CONSTANT, O.BORDER_REFLECT101, O.BORDER_REFLECT])
def test_warp_u8(mode):
    rng = np.random.default_rng(mode)
    src = rng.integers(0, 256, (131, 117, 3), dtype=np.uint8)
    for _ in range(8):
        M = similarity(rng, 117, 131)
        ref = cv2.warpAffine(src, M, (150, 140), borderMode=mode, borderValue=(135, 133, 132))
        assert np.array_equal(O.warp_linear_u8(src, M, (150, 140), mode, (135, 133, 132)), ref)


@needs_cv2
@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_warp_float(dtype):
    """f32 bilinear (the ones mask) and the parse mask's f64 warp (flags=3, INTER_AREA -> INTER_LINEAR)."""
    rng = np.random.default_rng(1)
    for src in (np.ones((96, 96), dtype), rng.random((90, 100)).astype(dtype)):
        for _ in range(6):
            M = similarity(rng, src.shape[1], src.shape[0])
            ref = cv2.warpAffine(src, M, (160, 150), flags=3 if dtype == np.float64 else cv2.INTER_LINEAR)
            assert np.array_equal(O.warp_linear_float(src, M, (160, 150)), ref)


@needs_cv2
@pytest.mark.parametrize('scale', [1, 2, 3, 4, 0.5])
def test_resize_u8(scale):
    rng = np.random.default_rng(2)
    for w, h in ((57, 41), (64, 48)):
        src = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        size = (int(w * scale), int(h * scale))
        assert np.array_equal(O.resize_linear_u8(src, size), cv2.resize(src, size, interpolation=cv2.INTER_LINEAR))


@needs_cv2
def test_resize_f64():
    """The parse mask's resize (512 -> 1024 for a face upsampler, other factors too) and random size pairs with sides >= 2,
    bit for bit.  (cv2 treats 1-pixel sides apart; the paste-back never resizes one.)"""
    require_x86_avx2_cv2()
    rng = np.random.default_rng(3)
    src = rng.random((64, 64))
    assert np.array_equal(O.resize_linear_f64(src, (128, 128)), cv2.resize(src, (128, 128)))
    pm = O.parse_soft_mask((rng.random((512, 512)) < 0.5).astype(np.uint8) * np.uint8(255))
    for S in (768, 1024, 1536, 2048):
        assert np.array_equal(O.resize_linear_f64(pm, (S, S)), cv2.resize(pm, (S, S))), S
    for _ in range(300):
        h, w, oh, ow = (int(v) for v in rng.integers(2, 90, 4))
        src = rng.random((h, w)) * rng.choice([1., 255., 1e-3])
        assert np.array_equal(O.resize_linear_f64(src, (ow, oh)), cv2.resize(src, (ow, oh))), (h, w, oh, ow)


@needs_cv2
@pytest.mark.parametrize('k', [0, 2, 3, 4, 6, 11])
def test_erode(k):
    src = np.random.default_rng(k).random((70, 53)).astype(np.float32)
    assert np.array_equal(O.erode_rect(src, k), cv2.erode(src, np.ones((k, k), np.uint8)))


@needs_cv2
def test_gaussian_kernels():
    for k in range(1, 402, 2):
        assert np.array_equal(O.gaussian_kernel(k, 0, np.float32), cv2.getGaussianKernel(k, 0, cv2.CV_32F)[:, 0]), k
    # the parse mask's kernel is cv2's own table (cv2 exponentiates in software double)
    assert np.array_equal(O.gaussian_kernel(101, 11, np.float64), cv2.getGaussianKernel(101, 11, cv2.CV_64F)[:, 0])


def test_device_parse_kernel_is_the_oracle_table():
    """csrc/pasteback.cu's kParseKernelHalf holds the same 51 float64 values as the oracle's PARSE_KERNEL_HALF."""
    src = open(PASTEBACK_CU).read()
    body = src[src.index('kParseKernelHalf[kParseK / 2 + 1] = {'):]
    body = body[body.index('{') + 1:body.index('};')]
    vals = [float.fromhex(v) for v in re.findall(r'0x[0-9a-f.]+p[-+]?\d+', body)]
    assert vals == O.PARSE_KERNEL_HALF and len(vals) == 51


def _blur_inputs(rng, h, w):
    box = np.zeros((h, w), np.float32)
    box[h // 4:h - h // 4, w // 5:w - w // 3] = 1
    ramp = (np.add.outer(np.arange(h), 2 * np.arange(w)) / (h + 2 * w)).astype(np.float32)
    return {'box': box, 'ramp': ramp, 'random': rng.random((h, w)).astype(np.float32)}


@needs_cv2
def test_blur_f32_matches_cv2():
    """GaussianBlur(m, (n, n), 0) for every soft-mask kernel (n = 2 w_edge + 1 for w_edge 0 .. 60), with widths and heights
    over every residue mod 16 (widths under 8 too), on a box, a ramp and noise: bit for bit."""
    require_x86_avx2_cv2()
    rng = np.random.default_rng(5)
    for n in range(1, 122, 2):
        for res in range(16):
            h = 2 + (res + 5 * n) % 16 + 16 * int(rng.integers(0, 4))
            w = 2 + res + 16 * int(rng.integers(0, 4)) if res < 14 else res - 12
            for kind, m in _blur_inputs(rng, h, w).items():
                out = O.blur_reflect101(m, O.gaussian_kernel(n, 0, np.float32))
                ref = cv2.GaussianBlur(m, (n, n), 0)
                assert np.array_equal(out, ref), f'n={n} {h}x{w} {kind}: {int((out != ref).sum())} values differ'


@needs_cv2
def test_blur_f64_matches_cv2():
    """The parse mask's GaussianBlur(pm, (101, 101), 11) in float64, twice, on 0/255 masks and noise over widths and heights
    of every residue mod 16, and at the mask's own 512 x 512: bit for bit."""
    require_x86_avx2_cv2()
    rng = np.random.default_rng(6)
    k = O.gaussian_kernel(101, 11, np.float64)
    for res in range(16):
        h, w = 2 + (res * 7) % 16 + 16 * int(rng.integers(0, 8)), 2 + res + 16 * int(rng.integers(0, 8))
        for m in ((rng.random((h, w)) < 0.5) * 255., rng.random((h, w)) * 255.):
            assert np.array_equal(O.blur_reflect101(m, k), cv2.GaussianBlur(m, (101, 101), 11)), (h, w)
    box = np.zeros((512, 512))
    box[60:450, 100:400] = 255
    for m in (box, (rng.random((512, 512)) < 0.7) * 255.):
        ref = cv2.GaussianBlur(cv2.GaussianBlur(m, (101, 101), 11), (101, 101), 11)
        assert np.array_equal(O.blur_reflect101(O.blur_reflect101(m, k), k), ref)


@needs_cv2
def test_invert_affine():
    rng = np.random.default_rng(6)
    for _ in range(10):
        M = similarity(rng, 300, 300)
        assert np.array_equal(O.invert_affine(M), cv2.invertAffineTransform(M))


@pytest.fixture(scope='module')
def oracle_runs():
    g = np.load(os.path.join(GOLD, 'pasteback.npz'))
    faces = np.ascontiguousarray(np.load(os.path.join(GOLD, 'faces.npz'))['faces'][..., ::-1])
    runs = {}
    for case, up in (('P1', 2), ('P2', 1), ('P3', 2)):
        img, upsample, _, ref = O.golden_case(g, faces, case, up)
        restored = [faces[i] for i in g[f'{case}_faces']]
        n = len(restored)
        masks = None
        if f'{case}_parse' in g:
            masks = np.unpackbits(g[f'{case}_parse'])[:n * 512 * 512].reshape(n, 512, 512) * np.uint8(255)
        ups = (lambda f: np.repeat(np.repeat(f, 2, 0), 2, 1)) if case == 'P3' else None
        canvas, info = O.paste_faces(img, restored, [m.copy() for m in g[f'{case}_inv']], up, masks, upsample,
                                     face_upsampler=ups, return_info=True)
        runs[case] = (canvas, info, ref, img)
    return g, runs


@pytest.mark.parametrize('case', ['P1', 'P2', 'P3'])
def test_oracle_matches_reference(oracle_runs, case):
    """Equal to the reference's uint8 result, byte for byte."""
    g, runs = oracle_runs
    canvas, info, ref, _ = runs[case]
    out = O.to_u8(canvas)
    assert np.array_equal(out, ref), f'{int((out != ref).sum())} values differ'
    np.testing.assert_allclose(canvas.reshape(-1)[O.sample_index(canvas.size)], g[f'{case}_sample_val'], rtol=0, atol=1e-4)
    assert [i['w_edge'] for i in info] == list(g[f'{case}_w_edge'])
    if case == 'P2':
        assert info[1]['w_edge'] == 0


@pytest.mark.parametrize('case', ['P1', 'P2', 'P3'])
def test_roi_contains_soft_mask(oracle_runs, case):
    """Restricting every per-face step to its ROI is exact: the final soft mask is 0 outside it."""
    _, runs = oracle_runs
    for i in runs[case][1]:
        x0, y0, x1, y1 = i['roi']
        outside = np.ones(i['soft'].shape, bool)
        outside[y0:y1, x0:x1] = False
        assert not i['soft'][outside].any()
        assert x1 > x0 and y1 > y0


@pytest.mark.parametrize('mode', ['constant', 'reflect101', 'reflect'])
def test_oracle_crops_match_reference(oracle_runs, mode):
    """The oracle's crop of the border-clipped face hashes to the reference's, in every border mode."""
    g, runs = oracle_runs
    img = runs['P1'][3]
    code = {'constant': O.BORDER_CONSTANT, 'reflect101': O.BORDER_REFLECT101, 'reflect': O.BORDER_REFLECT}[mode]
    crop = O.warp_linear_u8(img, g['crop_affine'], (512, 512), code, (135, 133, 132))
    assert hashlib.sha256(crop.tobytes()).hexdigest() == str(g[f'crop_{mode}_sha256'])


@needs_cv2
def test_synthetic_input_matches_cv2():
    """The rebuilt golden inputs are what cv2 composes (integer background, cv2-exact warps)."""
    g = np.load(os.path.join(GOLD, 'pasteback.npz'))
    faces = np.ascontiguousarray(np.load(os.path.join(GOLD, 'faces.npz'))['faces'][..., ::-1])
    h, w, seed = (int(v) for v in g['P1_input'])
    img = O.synthetic_input(faces, list(zip(g['P1_faces'], g['P1_T'])), h, w, seed)
    ref = O.synthetic_background(h, w, seed)
    for i, T in zip(g['P1_faces'], g['P1_T']):
        m = cv2.warpAffine(np.ones((512, 512), np.float32), T, (w, h)) > 0.5
        ref[m] = cv2.warpAffine(faces[i], T, (w, h))[m]
    assert np.array_equal(img, ref)
