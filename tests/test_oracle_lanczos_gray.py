"""CPU: the numpy INTER_LANCZOS4 restatement (oracle/resize_lanczos4_oracle.py) against cv2.resize, the tap tables the C
host code builds (cfb_lanczos4_table) against the restatement, and the gray branch (oracle/gray_oracle.py) against the
reference's own adain_npy / bgr2gray and paste_faces_to_input_image with is_gray=True."""
import ctypes

import numpy as np
import pytest

from oracle import gray_oracle as G
from oracle import pasteback_oracle as O
from oracle import ref_shim
from oracle import resize_lanczos4_oracle as L

cv2 = pytest.importorskip('cv2')

# (h, w, out_h, out_w)
CASES = [
    (40, 50, 80, 100),           # 2x up
    (80, 100, 40, 50),           # 0.5x down
    (60, 90, 90, 135),           # 1.5x
    (60, 90, 80, 120),           # 4/3x
    (90, 120, 30, 40),           # 1/3x
    (517, 389, 1000, 300),       # non-uniform: up on one axis, down on the other
    (41, 53, 61, 79),
    (5, 6, 11, 9),               # fewer than 8 pixels on both axes
    (3, 100, 7, 40),
    (1, 1, 4, 5),
    (33, 31, 33, 30),            # one axis unchanged
    (24, 36, 24, 36),            # same size: a copy
]
# axis lengths of the frame sizes restore_images meets: x2plus output of a 1080p frame to x0.5 / x1.5 / x2, small inputs to x4
AXES = [(2160, 1080), (3840, 1920), (2160, 3240), (3840, 5760), (2160, 4320), (1080, 2160), (300, 512), (512, 2048), (719, 1917)]


def case_id(c):
    return '{}x{}-{}x{}'.format(*c)


@pytest.mark.parametrize('case', CASES, ids=case_id)
def test_lanczos4_oracle_matches_cv2(case):
    h, w, oh, ow = case
    src = np.random.default_rng(h * 7919 + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    ref = cv2.resize(src, (ow, oh), interpolation=cv2.INTER_LANCZOS4)
    assert np.array_equal(L.resize_lanczos4_u8(src, (ow, oh)), ref)


def test_lanczos4_oracle_saturated_images():
    """Black / white checks and constant 255: the overshoot of the negative lobes meets the clamp."""
    for h, w, oh, ow in [(40, 50, 80, 100), (80, 100, 40, 50), (41, 53, 61, 79)]:
        yy, xx = np.mgrid[:h, :w]
        check = (((yy // 3 + xx // 3) % 2) * 255).astype(np.uint8)[:, :, None].repeat(3, axis=2)
        for src in (check, np.full((h, w, 3), 255, np.uint8)):
            assert np.array_equal(L.resize_lanczos4_u8(src, (ow, oh)), cv2.resize(src, (ow, oh), interpolation=cv2.INTER_LANCZOS4))


@pytest.mark.parametrize('axis', AXES, ids=lambda a: f'{a[0]}-{a[1]}')
def test_lanczos4_oracle_matches_cv2_on_frame_axes(axis):
    """One axis at the sizes of real frames (the other stays 8 pixels), both orientations."""
    n_in, n_out = axis
    rng = np.random.default_rng(n_in + n_out)
    src = rng.integers(0, 256, (8, n_in, 3), dtype=np.uint8)
    assert np.array_equal(L.resize_lanczos4_u8(src, (n_out, 8)), cv2.resize(src, (n_out, 8), interpolation=cv2.INTER_LANCZOS4))
    src = np.ascontiguousarray(src.transpose(1, 0, 2))
    assert np.array_equal(L.resize_lanczos4_u8(src, (8, n_out)), cv2.resize(src, (8, n_out), interpolation=cv2.INTER_LANCZOS4))


def test_c_tap_tables_match_oracle():
    """cfb_lanczos4_table (the host code behind cfb_resize_lanczos4_u8) builds the oracle's tables; no device needed."""
    from codeformer_b200 import _lib
    lib = _lib.load()
    axes = {(c[0], c[2]) for c in CASES} | {(c[1], c[3]) for c in CASES} | set(AXES)
    for n_in, n_out in sorted(axes):
        idx = np.zeros(n_out, np.int32)
        coef = np.zeros((n_out, 8), np.int16)
        lib.cfb_lanczos4_table(n_in, n_out, idx.ctypes.data_as(ctypes.c_void_p), coef.ctypes.data_as(ctypes.c_void_p))
        ref_idx, ref_coef = L.tap_table(n_in, n_out)
        assert np.array_equal(idx, ref_idx), (n_in, n_out)
        assert np.array_equal(coef, ref_coef), (n_in, n_out)


# ---- the gray branch ---------------------------------------------------------------------------------------------------
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason='reference tree not present')


def _gray_faces(n, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:512, :512]
    out = []
    for i in range(n):
        base = (np.sin(xx / (17.0 + i)) * np.cos(yy / (23.0 + 2 * i)) * 90 + 128)[:, :, None]
        out.append(np.clip(base + rng.normal(0, 6, (512, 512, 3)), 0, 255).astype(np.uint8))
    return out


@needs_ref
def test_gray_adain_matches_reference():
    from oracle.gen_golden_pasteback import load_helper_class
    _, mod = load_helper_class()
    restored, cropped = _gray_faces(2, 1), _gray_faces(2, 2)
    for r, c in zip(restored, cropped):
        ref = mod.adain_npy(mod.bgr2gray(r), c)
        out = G.gray_adain(r, c)
        assert out.dtype == np.float64 and out.shape == (512, 512, 3)
        np.testing.assert_allclose(out, ref, rtol=1e-12, atol=0)


@needs_ref
@pytest.mark.parametrize('upscale', [1, 2])
def test_f64_paste_matches_reference(upscale):
    """A synthetic gray image with two faces through the reference's paste with is_gray=True, use_parse=False (cv2 on the
    host), against the float64 paste oracle, byte for byte."""
    from oracle.gen_golden_pasteback import load_helper_class, make_helper
    cls, mod = load_helper_class()
    h, w = 300, 420
    bg = cv2.cvtColor(cv2.cvtColor(O.synthetic_background(h, w, 3), cv2.COLOR_BGR2GRAY), cv2.COLOR_GRAY2BGR)
    restored, cropped = _gray_faces(2, 5), _gray_faces(2, 6)
    aff = [np.array([[2.1, 0.3, -120.], [-0.3, 2.1, -60.]]), np.array([[2.6, -0.4, -600.], [0.4, 2.6, -330.]])]
    helper = make_helper(cls, bg, [], upscale, False, None)
    helper.is_gray = True
    for r, c in zip(restored, cropped):
        helper.add_restored_face(r, c)
    assert all(f.dtype == np.float64 for f in helper.restored_faces)
    helper.inverse_affine_matrices = [cv2.invertAffineTransform(a) * upscale for a in aff]
    invs = [m.copy() for m in helper.inverse_affine_matrices]
    ref = helper.paste_faces_to_input_image()
    faces = [G.gray_adain(r, c) for r, c in zip(restored, cropped)]
    for a, b in zip(faces, helper.restored_faces):
        assert np.array_equal(a, b)                # the same numpy expressions: the paste below sees identical faces
    out = G.final_cast(G.paste_faces_f64(bg, faces, invs, upscale))
    assert out.dtype == ref.dtype == np.uint8 and np.array_equal(out, ref)
    assert (ref != cv2.resize(bg, (w * upscale, h * upscale), interpolation=cv2.INTER_LINEAR)).mean() > 0.05


@needs_ref
def test_bright_face_gives_uint16_as_the_reference():
    from oracle.gen_golden_pasteback import load_helper_class, make_helper
    cls, _ = load_helper_class()
    bg = np.full((300, 420, 3), 200, np.uint8)
    face = np.full((512, 512, 3), 300.0)           # what the colour transfer can produce for a bright crop
    helper = make_helper(cls, bg, [], 1, False, None)
    helper.is_gray = True
    helper.restored_faces = [face]
    aff = np.array([[2.1, 0.3, -120.], [-0.3, 2.1, -60.]])
    helper.inverse_affine_matrices = [cv2.invertAffineTransform(aff)]
    invs = [m.copy() for m in helper.inverse_affine_matrices]
    ref = helper.paste_faces_to_input_image()
    out = G.final_cast(G.paste_faces_f64(bg, [face], invs, 1))
    assert ref.dtype == np.uint16 and out.dtype == np.uint16 and np.array_equal(out, ref)
