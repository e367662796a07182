"""CPU: the numpy INTER_LANCZOS4 restatement for uint16 images (oracle/resize_lanczos4_u16_oracle.py) against cv2.resize on
CV_16U, and the float tap tables the C host code builds (cfb_lanczos4_table_f32) against the restatement."""
import ctypes

import numpy as np
import pytest

from oracle import resize_lanczos4_u16_oracle as L

cv2 = pytest.importorskip('cv2')

# (h, w, out_h, out_w): x0.5 / x1.5 / x2 on odd sizes, one and three rows or columns, mixed factors
CASES = [
    (41, 53, 82, 106),           # x2
    (41, 53, 20, 26),            # x0.5
    (41, 53, 61, 79),            # x1.5
    (99, 77, 198, 154),
    (99, 77, 148, 115),
    (1, 37, 2, 74),              # one row
    (37, 1, 55, 1),              # one column
    (1, 1, 2, 2),
    (3, 29, 6, 58),              # three rows
    (29, 3, 14, 1),              # three columns
    (3, 3, 4, 4),
    (517, 389, 1000, 300),       # up on one axis, down on the other
    (33, 31, 33, 30),            # one axis unchanged: unit taps with their ~1e-31 neighbours
    (24, 36, 24, 36),            # same size: a copy
]


def case_id(c):
    return '{}x{}-{}x{}'.format(*c)


@pytest.mark.parametrize('case', CASES, ids=case_id)
@pytest.mark.parametrize('hi', [255, 65535], ids=['below256', 'full'])
def test_lanczos4_u16_oracle_matches_cv2(case, hi):
    h, w, oh, ow = case
    src = np.random.default_rng(h * 7919 + w + hi).integers(0, hi + 1, (h, w, 3), dtype=np.uint16)
    ref = cv2.resize(src, (ow, oh), interpolation=cv2.INTER_LANCZOS4)
    out = L.resize_lanczos4_u16(src, (ow, oh))
    assert out.dtype == ref.dtype == np.uint16 and np.array_equal(out, ref)


def test_lanczos4_u16_oracle_saturated_images():
    """Black / white checks and constant 65535: the overshoot of the negative lobes meets the clamp at both ends."""
    for h, w, oh, ow in [(40, 50, 80, 100), (80, 100, 40, 50), (41, 53, 61, 79)]:
        yy, xx = np.mgrid[:h, :w]
        check = (((yy // 3 + xx // 3) % 2) * 65535).astype(np.uint16)[:, :, None].repeat(3, axis=2)
        for src in (check, np.full((h, w, 3), 65535, np.uint16)):
            assert np.array_equal(L.resize_lanczos4_u16(src, (ow, oh)), cv2.resize(src, (ow, oh), interpolation=cv2.INTER_LANCZOS4))


@pytest.mark.parametrize('axis', [(1080, 2160), (1920, 2880), (2160, 1080), (3840, 5760), (1024, 1536)], ids=lambda a: f'{a[0]}-{a[1]}')
def test_lanczos4_u16_oracle_matches_cv2_on_frame_axes(axis):
    """One axis at the sizes of real frames (the other stays 8 pixels), both orientations."""
    n_in, n_out = axis
    src = np.random.default_rng(n_in + n_out).integers(0, 65536, (8, n_in, 3), dtype=np.uint16)
    assert np.array_equal(L.resize_lanczos4_u16(src, (n_out, 8)), cv2.resize(src, (n_out, 8), interpolation=cv2.INTER_LANCZOS4))
    src = np.ascontiguousarray(src.transpose(1, 0, 2))
    assert np.array_equal(L.resize_lanczos4_u16(src, (8, n_out)), cv2.resize(src, (8, n_out), interpolation=cv2.INTER_LANCZOS4))


def test_c_float_tap_tables_match_oracle():
    """cfb_lanczos4_table_f32 (the host code behind cfb_resize_lanczos4_u16) builds the oracle's tables; no device needed."""
    from codeformer_b200 import _lib
    lib = _lib.load()
    axes = {(c[0], c[2]) for c in CASES} | {(c[1], c[3]) for c in CASES} | {(1080, 2160), (2160, 1080), (1920, 2880)}
    for n_in, n_out in sorted(axes):
        idx = np.zeros(n_out, np.int32)
        coef = np.zeros((n_out, 8), np.float32)
        lib.cfb_lanczos4_table_f32(n_in, n_out, idx.ctypes.data_as(ctypes.c_void_p), coef.ctypes.data_as(ctypes.c_void_p))
        ref_idx, ref_coef = L.tap_table(n_in, n_out)
        assert np.array_equal(idx, ref_idx), (n_in, n_out)
        assert np.array_equal(coef.view(np.uint32), ref_coef.view(np.uint32)), (n_in, n_out)
