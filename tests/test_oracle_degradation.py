"""not gpu: the degradation sampler against the UNMODIFIED reference (basicsr/data/gaussian_kernels.py and the draw order of
FFHQBlindDataset.__getitem__; skips without the reference tree), and the numpy restatement of the chain's cv2 / libjpeg-turbo
arithmetic (oracle/degradation_oracle.py) against cv2."""
import importlib.util
import math
import os
import random

import cv2
import numpy as np
import pytest

from codeformer_b200 import degradation as DG
from oracle import degradation_oracle as DO
from oracle import ref_shim

RANGES = {'stage2': DG.STAGE2_RANGES, 'stage3': DG.STAGE3_RANGES}


def _reference_kernels():
    if not ref_shim.available():
        pytest.skip('reference tree not available')
    path = os.path.join(ref_shim.REF_ROOT, 'basicsr', 'data', 'gaussian_kernels.py')
    spec = importlib.util.spec_from_file_location('_ref_gaussian_kernels', path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _reference_draw(gk, r, gt_size=512):
    """The draws of ffhq_blind_dataset.py:210-236 for one face, in its order, with the reference's kernel sampler."""
    kernel = gk.random_mixed_kernels(['iso', 'aniso'], [0.5, 0.5], 41, r['blur_sigma'], r['blur_sigma'], [-math.pi, math.pi],
                                     noise_range=None)
    scale = np.random.uniform(r['downsample_range'][0], r['downsample_range'][1])
    size = int(gt_size // scale)
    noise_sigma = np.random.uniform(r['noise_range'][0] / 255., r['noise_range'][1] / 255.)
    noise = np.float32(np.random.randn(size, size, 3)) * noise_sigma
    q = int(np.random.uniform(r['jpeg_range'][0], r['jpeg_range'][1]))
    return kernel, scale, size, noise, q


def kernel_bar(p):
    """1e-15 plus the float64 rounding of the exponent: each kernel value k carries an error of about eps * k * M, where
    M = |p| x^2 + 2 |r x y| + |q| y^2 sums the magnitudes of the quadratic form's terms.  The terms cancel along the ridge
    of a narrow rotated kernel (sigma 0.1 against 10 in the stage-3 ranges), so there M / 2 far exceeds the exponent and
    neither the reference's kernel nor any other float64 evaluation is within 1e-15 of the exact one (up to 1.2e-14 for
    both, measured against a 200-bit evaluation); for the stage-2 ranges the bar stays at about 1e-15."""
    c, s_ = math.cos(p['rotation']), math.sin(p['rotation'])
    ix, iy = p['sigma_x'] ** -2., p['sigma_y'] ** -2.
    a, r, q = c * c * ix + s_ * s_ * iy, c * s_ * (ix - iy), s_ * s_ * ix + c * c * iy
    off = np.arange(41.) - 20
    x, y = off[None, :], off[:, None]
    m = abs(a) * x * x + 2 * abs(r * x * y) + abs(q) * y * y
    return 1e-15 + 8 * np.finfo(np.float64).eps * (p['kernel'] * m).max()


@pytest.mark.parametrize('stage', ['stage2', 'stage3'])
def test_sampler_matches_reference_draws(stage):
    gk = _reference_kernels()
    r = RANGES[stage]
    for seed in range(200):
        random.seed(seed)
        np.random.seed(seed)
        kernel, scale, size, noise, q = _reference_draw(gk, r)
        ref_state = (random.getstate(), np.random.get_state()[1].copy())
        random.seed(seed)
        np.random.seed(seed)
        p = DG.sample_degradations(1, **r)[0]
        assert (random.getstate(), ) == (ref_state[0], )
        assert np.array_equal(np.random.get_state()[1], ref_state[1]), 'the sampler consumed np.random differently'
        assert p['scale'] == scale and p['size'] == size and p['quality'] == q
        assert p['noise'].dtype == noise.dtype == np.float32 and np.array_equal(p['noise'], noise)
        err = np.abs(p['kernel'] - kernel).max()
        assert err <= kernel_bar(p), (seed, err, kernel_bar(p))
        # the sigmas and the rotation: replay the kernel's uniforms
        random.seed(seed)
        np.random.seed(seed)
        kind = random.choices(['iso', 'aniso'], [0.5, 0.5])[0]
        assert kind == p['kernel_type']
        u = [np.random.uniform(*r['blur_sigma'])]
        if kind == 'aniso':
            u += [np.random.uniform(*r['blur_sigma']), np.random.uniform(-math.pi, math.pi)]
            assert (p['sigma_x'], p['sigma_y'], p['rotation']) == tuple(u)
        else:
            assert p['sigma_x'] == p['sigma_y'] == u[0] and p['rotation'] == 0


def test_sampler_options_and_errors():
    rs = np.random.RandomState(3)
    p = DG.sample_degradations(4, noise_range=None, jpeg_range=None, py_rng=random.Random(1), np_rng=rs)
    assert all(x['noise'] is None and x['quality'] is None for x in p)
    rs2 = np.random.RandomState(3)
    p2 = DG.sample_degradations(4, noise_range=None, jpeg_range=None, py_rng=random.Random(1), np_rng=rs2)
    assert all(np.array_equal(a['kernel'], b['kernel']) and a['size'] == b['size'] for a, b in zip(p, p2))
    p = DG.sample_degradations(3, gt_size=256, in_size=128, **DG.STAGE3_RANGES)
    assert all(1 <= x['size'] <= 256 and x['noise'].shape == (x['size'], x['size'], 3) for x in p)
    with pytest.raises(NotImplementedError):
        DG.sample_degradations(1, kernel_list=('generalized',), kernel_prob=(1,))
    with pytest.raises(ValueError):
        DG.sample_degradations(1, gt_size=256, in_size=512)

# -------------------------------------------------------------------------------------------------------------- JPEG


def cv2_jpeg(img, q):
    ok, enc = cv2.imencode('.jpg', img, [int(cv2.IMWRITE_JPEG_QUALITY), int(q)])
    assert ok
    return cv2.imdecode(enc, 1)


def jpeg_contents(h, w, seed=0):
    """Random, smooth, black / white checker and gray content of one size."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    smooth = np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), (xx + yy) * 127 // max(h + w - 2, 1)], -1)
    bw = np.where(((yy // 3 + xx // 2) % 2 == 0)[..., None], 255, 0).repeat(3, 2)
    gray = rng.integers(0, 256, (h, w, 1)).repeat(3, 2)
    return {'random': rng.integers(0, 256, (h, w, 3)).astype(np.uint8), 'smooth': smooth.astype(np.uint8),
            'bw': bw.astype(np.uint8), 'gray': gray.astype(np.uint8)}


# 2 x 300 ... 4 x 4 and 5 x 3: chroma planes of at most 2 samples across, which libjpeg-turbo upsamples by replication
JPEG_SIZES = [(1, 1), (7, 9), (16, 16), (17, 23), (33, 65), (128, 128), (512, 512), (2, 300), (4, 4), (5, 3), (9, 4), (40, 2),
              (64, 2), (300, 2)]
JPEG_QUALITIES = [1, 30, 55, 79, 100]


def test_jpeg_every_quality():
    img = np.random.default_rng(7).integers(0, 256, (40, 56, 3)).astype(np.uint8)
    img[:, :28] = cv2.GaussianBlur(img[:, :28], (7, 7), 2)
    for q in range(1, 101):
        assert np.array_equal(DO.jpeg_roundtrip(img, q), cv2_jpeg(img, q)), q


@pytest.mark.parametrize('size', JPEG_SIZES, ids=lambda s: f'{s[0]}x{s[1]}')
def test_jpeg_sizes_and_content(size):
    for name, img in jpeg_contents(*size).items():
        for q in JPEG_QUALITIES:
            got, want = DO.jpeg_roundtrip(img, q), cv2_jpeg(img, q)
            assert np.array_equal(got, want), (name, q, int((got != want).sum()))

# ------------------------------------------------------------------------------------------------ resize, blur, uint8


SMALL_SIZES = [17, 18, 19, 21, 23, 26, 30, 34, 39, 42, 51, 64, 73, 85, 102, 113, 128, 170, 204, 256, 300, 341, 400, 455, 511]


@pytest.mark.parametrize('gt', [256, 512])
def test_resize_linear_matches_cv2(gt):
    rng = np.random.default_rng(gt)
    big = rng.random((gt, gt, 3), dtype=np.float32)
    for s in [x for x in SMALL_SIZES if x <= gt] + [gt]:
        small = rng.random((s, s, 3), dtype=np.float32)
        assert np.array_equal(DO.resize_linear(big, s, s), cv2.resize(big, (s, s), interpolation=cv2.INTER_LINEAR)), s
        for out in {512, gt, 128}:
            want = cv2.resize(small, (out, out), interpolation=cv2.INTER_LINEAR)
            assert np.array_equal(DO.resize_linear(small, out, out), want), (s, out)


@pytest.mark.parametrize('kind', ['iso', 'aniso'])
@pytest.mark.parametrize('sigma', [1, 15])
def test_filter2d_within_one_ulp_of_cv2(kind, sigma):
    rng = np.random.default_rng(sigma)
    img = (rng.integers(0, 256, (70, 90, 3)).astype(np.float32) / np.float32(255.)).astype(np.float32)
    img = cv2.GaussianBlur(img, (5, 5), 1) if kind == 'iso' else img
    if kind == 'iso':
        k = DG._gaussian_kernel(41, sigma ** -2., 0., sigma ** -2.)
    else:
        k = DG._gaussian_kernel(41, sigma ** -2., 0.5 * sigma ** -2., 2 * sigma ** -2.)
    got = DO.filter2d_f64(img, k)
    want = cv2.filter2D(img, -1, k, borderType=cv2.BORDER_REFLECT_101)
    ulp = np.spacing(np.maximum(np.abs(got), np.abs(want)).astype(np.float32))
    assert (np.abs(got.astype(np.float64) - want) <= ulp).all()
    rows = np.array([0, 3, 40, 69])
    assert np.array_equal(DO.filter2d_f64(img, k, rows, rows[:3]), got[np.ix_(rows, rows[:3])])


def test_to_u8_rounds_half_to_even_like_cv2():
    v = np.array([0.5, 1.5, 2.5, 3.5, 254.5, 255.5, -0.5, -3., 300., 127.49999, 127.5, 128.5], np.float32)
    want = cv2.imdecode(cv2.imencode('.png', v.reshape(1, -1))[1], cv2.IMREAD_UNCHANGED)[0]
    assert np.array_equal(DO.to_u8(v), want)
    assert list(DO.to_u8(v)[:4]) == [0, 2, 2, 4]

# ------------------------------------------------------------------------------------------------------ whole chain


def host_chain(gt_u8, p, in_size):
    """ffhq_blind_dataset.py:210-240 written out with cv2, from the same parameters."""
    img = gt_u8.astype(np.float32) / 255.
    img = cv2.filter2D(img, -1, p['kernel'])
    s = p['size']
    img = cv2.resize(img, (s, s), interpolation=cv2.INTER_LINEAR)
    if p['noise'] is not None:
        img = np.clip(img + p['noise'], 0, 1)
    if p['quality'] is not None:
        _, enc = cv2.imencode('.jpg', img * 255., [int(cv2.IMWRITE_JPEG_QUALITY), p['quality']])
        img = np.float32(cv2.imdecode(enc, 1)) / 255.
    img = cv2.resize(img, (in_size, in_size), interpolation=cv2.INTER_LINEAR)
    return np.clip((img * 255.).round(), 0, 255).astype(np.uint8)


def test_oracle_chain_close_to_host_chain():
    rng = np.random.default_rng(5)
    gt = cv2.GaussianBlur(rng.integers(0, 256, (128, 128, 3)).astype(np.uint8), (9, 9), 3)
    params = DG.sample_degradations(3, gt_size=128, in_size=128, py_rng=random.Random(2), np_rng=np.random.RandomState(2),
                                    blur_sigma=(1, 4), downsample_range=(2, 6), noise_range=(0, 10), jpeg_range=(30, 80))
    for p in params:
        lq, _, _ = DO.degrade(gt, p, 128)
        want = host_chain(gt, p, 128)
        assert (lq == want).mean() > 0.97
        assert np.abs(lq.astype(int) - want).max() <= 40
