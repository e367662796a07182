"""The numpy paste-back oracle (oracle/pasteback_oracle.py) against cv2 and against the reference golden.  CPU only."""
import hashlib
import os

import numpy as np
import pytest

from oracle import pasteback_oracle as O

cv2 = pytest.importorskip('cv2')
GOLD = os.path.join(os.path.dirname(__file__), 'golden')


def similarity(rng, w, h):
    a, s = rng.uniform(-0.35, 0.35), rng.uniform(0.4, 3.0)
    c, si = np.cos(a) * s, np.sin(a) * s
    return np.array([[c, -si, rng.uniform(-w / 2, w / 2)], [si, c, rng.uniform(-h / 2, h / 2)]])


@pytest.mark.parametrize('mode', [cv2.BORDER_CONSTANT, cv2.BORDER_REFLECT101, cv2.BORDER_REFLECT])
def test_warp_u8(mode):
    rng = np.random.default_rng(mode)
    src = rng.integers(0, 256, (131, 117, 3), dtype=np.uint8)
    for _ in range(8):
        M = similarity(rng, 117, 131)
        ref = cv2.warpAffine(src, M, (150, 140), borderMode=mode, borderValue=(135, 133, 132))
        assert np.array_equal(O.warp_linear_u8(src, M, (150, 140), mode, (135, 133, 132)), ref)


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_warp_float(dtype):
    """f32 bilinear (the ones mask) and the parse mask's f64 warp (flags=3, INTER_AREA -> INTER_LINEAR)."""
    rng = np.random.default_rng(1)
    for src in (np.ones((96, 96), dtype), rng.random((90, 100)).astype(dtype)):
        for _ in range(6):
            M = similarity(rng, src.shape[1], src.shape[0])
            ref = cv2.warpAffine(src, M, (160, 150), flags=3 if dtype == np.float64 else cv2.INTER_LINEAR)
            assert np.array_equal(O.warp_linear_float(src, M, (160, 150)), ref)


@pytest.mark.parametrize('scale', [1, 2, 3, 4, 0.5])
def test_resize_u8(scale):
    rng = np.random.default_rng(2)
    for w, h in ((57, 41), (64, 48)):
        src = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        size = (int(w * scale), int(h * scale))
        assert np.array_equal(O.resize_linear_u8(src, size), cv2.resize(src, size, interpolation=cv2.INTER_LINEAR))


def test_resize_f64():
    """512 -> 1024 of the parse mask: cv2 rounds some sums differently in the last bit."""
    rng = np.random.default_rng(3)
    src = rng.random((64, 64))
    np.testing.assert_allclose(O.resize_linear_f64(src, (128, 128)), cv2.resize(src, (128, 128)), rtol=0, atol=1e-15)


@pytest.mark.parametrize('k', [0, 2, 3, 4, 6, 11])
def test_erode(k):
    src = np.random.default_rng(k).random((70, 53)).astype(np.float32)
    assert np.array_equal(O.erode_rect(src, k), cv2.erode(src, np.ones((k, k), np.uint8)))


def test_gaussian_kernels():
    for k in range(1, 402, 2):
        assert np.array_equal(O.gaussian_kernel(k, 0, np.float32), cv2.getGaussianKernel(k, 0, cv2.CV_32F)[:, 0]), k
    a, b = O.gaussian_kernel(101, 11, np.float64), cv2.getGaussianKernel(101, 11, cv2.CV_64F)[:, 0]
    np.testing.assert_allclose(a, b, rtol=0, atol=2e-17)      # cv2 exponentiates in software double


def test_blur_close_to_cv2():
    """The separable blur sums taps in order; cv2 rounds some sums differently in the last bits."""
    rng = np.random.default_rng(5)
    m = rng.random((80, 90)).astype(np.float32)
    for k in (1, 3, 5, 11, 31):
        np.testing.assert_allclose(O.blur_reflect101(m, O.gaussian_kernel(k, 0, np.float32)), cv2.GaussianBlur(m, (k, k), 0),
                                   rtol=0, atol=1e-6)


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
    """Equal to the reference's uint8 result except where the pre-cast value is within 1e-3 of an integer (cv2's
    float32 blur rounds in the last bit there); within 1 there."""
    g, runs = oracle_runs
    canvas, info, ref, _ = runs[case]
    ambig = np.unpackbits(g[f'{case}_ambig'])[:ref.size].reshape(ref.shape).astype(bool)
    d = O.to_u8(canvas).astype(np.int16) - ref
    assert not d[~ambig].any() and np.abs(d).max() <= 1
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
