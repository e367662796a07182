"""not gpu: the PSNR / SSIM restatement (oracle/metrics_oracle.py) against the UNMODIFIED reference functions
(basicsr/metrics/psnr_ssim.py; skips without the reference tree), and its deliberate deviations."""
import numpy as np
import pytest

from oracle import metrics_oracle as MO
from oracle import ref_shim


def _reference():
    if not ref_shim.available():
        pytest.skip('reference tree not available')
    ref_shim.load()                       # seeds the basicsr namespaces; the metrics modules import as they are
    from basicsr.metrics.metric_util import to_y_channel
    from basicsr.metrics.psnr_ssim import calculate_psnr, calculate_ssim
    return calculate_psnr, calculate_ssim, to_y_channel


def pair(dtype, h, w, c=3, seed=0):
    """A seeded image and a perturbed copy, in the value range of ``dtype`` (floats in [0, 255])."""
    rng = np.random.default_rng(seed)
    shape = (h, w, c) if c else (h, w)
    if dtype == np.uint8:
        a = rng.integers(0, 256, shape)
        return a.astype(np.uint8), np.clip(a + rng.integers(-24, 25, shape), 0, 255).astype(np.uint8)
    if dtype == np.uint16:
        a = rng.integers(0, 65536, shape)
        return a.astype(np.uint16), np.clip(a + rng.integers(-3000, 3001, shape), 0, 65535).astype(np.uint16)
    a = rng.random(shape) * 255
    return a.astype(dtype), (a + rng.standard_normal(shape) * 6).astype(dtype)


DTYPES = [np.uint8, np.uint16, np.float32, np.float64]


@pytest.mark.parametrize('dtype', DTYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize('y', [False, True], ids=['rgb', 'y'])
@pytest.mark.parametrize('crop', [0, 4])
@pytest.mark.parametrize('order', ['HWC', 'CHW', '2d'])
def test_oracle_matches_reference(dtype, y, crop, order):
    ref_psnr, ref_ssim, _ = _reference()
    a, b = pair(dtype, 48, 61, c=0 if order == '2d' else 3, seed=crop + 7 * y)
    io = 'HWC'
    if order == 'CHW':
        a, b, io = a.transpose(2, 0, 1), b.transpose(2, 0, 1), 'CHW'
    assert MO.ssim(a, b, crop, io, y) == ref_ssim(a, b, crop, io, y)
    p, r = MO.psnr(a, b, crop, io, y), ref_psnr(a, b, crop, io, y)
    if y:          # the reference averages the float32 squares in float32
        assert abs(p - float(r)) < 1e-4
    else:
        assert p == r


@pytest.mark.parametrize('dtype', DTYPES, ids=lambda d: np.dtype(d).name)
def test_oracle_512_faces(dtype):
    ref_psnr, ref_ssim, _ = _reference()
    a, b = pair(dtype, 512, 512, seed=3)
    for y in (False, True):
        assert MO.ssim(a, b, 0, 'HWC', y) == ref_ssim(a, b, 0, 'HWC', y)
        p, r = MO.psnr(a, b, 0, 'HWC', y), ref_psnr(a, b, 0, 'HWC', y)
        assert (abs(p - float(r)) < 1e-4) if y else p == r


def test_y_channel_matches_reference():
    _, _, to_y = _reference()
    for seed in range(4):
        a = pair(np.uint8, 512, 512, seed=seed)[0].astype(np.float64)
        assert np.array_equal(MO.y_channel(a), to_y(a))
    f = pair(np.float64, 128, 96, seed=9)[0]
    assert np.array_equal(MO.y_channel(f), to_y(f))
    g = pair(np.float32, 40, 30, c=1, seed=2)[0].astype(np.float64)     # one channel: rounded through float32 only
    assert np.array_equal(MO.y_channel(g), to_y(g))


@pytest.mark.parametrize('dtype', DTYPES, ids=lambda d: np.dtype(d).name)
def test_identical_images(dtype):
    a = pair(dtype, 40, 33, seed=1)[0]
    for y in (False, True):
        assert MO.psnr(a, a.copy(), 2, 'HWC', y) == float('inf')
        assert MO.ssim(a, a.copy(), 2, 'HWC', y) == 1.0


def test_mixed_dtypes_equal_the_common_float64():
    a, b = pair(np.uint8, 30, 40, seed=4)
    for y in (False, True):
        assert MO.psnr(a, b.astype(np.float64), 1, 'HWC', y) == MO.psnr(a.astype(np.float64), b.astype(np.float64), 1, 'HWC', y)
        assert MO.ssim(a, b.astype(np.float32), 1, 'HWC', y) == MO.ssim(a, b, 1, 'HWC', y)


def test_deviations_raise():
    a, b = pair(np.uint8, 20, 24, seed=5)
    with pytest.raises(AssertionError):
        MO.psnr(a, b[:-1], 0)
    with pytest.raises(ValueError, match='input_order'):
        MO.psnr(a, b, 0, 'WHC')
    with pytest.raises(ValueError, match='crop_border'):
        MO.psnr(a, b, -1)
    with pytest.raises(ValueError):
        MO.psnr(a, b, 10)                 # no pixel left
    assert np.isfinite(MO.psnr(a, b, 9))
    with pytest.raises(ValueError):
        MO.ssim(a, b, 5)                  # 10 x 14 after the crop
    assert np.isfinite(MO.ssim(a, b, 4))
    with pytest.raises(NotImplementedError):
        MO.psnr(a.astype(np.int32), b.astype(np.int32), 0)
    with pytest.raises(NotImplementedError):
        MO.ssim(a.astype(np.float16), b.astype(np.float16), 0)


def test_nan_gives_nan():
    a, b = pair(np.float32, 24, 24, seed=6)
    a[3, 4, 1] = np.nan
    assert np.isnan(MO.psnr(a, b, 0)) and np.isnan(MO.ssim(a, b, 0))
