"""The CPU twin of tests/test_gpu_paste_sweep.py: the oracle (oracle/pasteback_oracle.py, oracle/gray_oracle.py) against
the reference's paste written out with cv2, on the same seeded scenes (tests/paste_scenes.py), byte for byte and on the
float canvas before the cast; and the oracle's warp and resize against cv2 over general matrices and sizes."""
import numpy as np
import pytest

from oracle import pasteback_oracle as O
from tests import paste_scenes as PS

cv2 = pytest.importorskip('cv2')
BORDERS = (O.BORDER_CONSTANT, O.BORDER_REFLECT101, O.BORDER_REFLECT)


@pytest.mark.parametrize('i', range(PS.N_SCENES))
def test_oracle_paste_matches_cv2(i):
    sc = PS.scene(i)
    out, canvas, info = PS.oracle_paste(sc)
    ref, ref_canvas = PS.cv2_paste(cv2, sc)
    assert out.dtype == ref.dtype and np.array_equal(out, ref), f'{int((out != ref).sum())} values differ'
    assert np.array_equal(canvas, ref_canvas), f'{int((canvas != ref_canvas).sum())} canvas values differ'
    if info is not None:            # the first face's w_edge is about the scene's target (0 .. 50)
        assert abs(info[0]['w_edge'] - PS.W_EDGES[i]) <= 1


@pytest.mark.parametrize('kind', ['shear', 'flip', 'scale', 'singular'])
def test_oracle_warp_general_affines(kind):
    """u8 warps of general matrices from sources of 1 x 1 up, in every border mode; the near-singular matrices map the
    output beyond int16 source coordinates, where cv2 saturates them."""
    rng = np.random.default_rng(len(kind))
    saturated = 0
    for t in range(24):
        sh, sw = (int(v) for v in rng.integers(1, 90, 2)) if t % 4 else (1 + t % 3, 1 + t % 2)
        oh, ow = (int(v) for v in rng.integers(1, 120, 2))
        src = rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8)
        M = PS.general_affine(rng, kind, sw, sh, ow, oh)
        ix, iy = O.warp_coords(M, (ow, oh))[:2]
        saturated += int((np.abs(ix) >= 32767).any() or (np.abs(iy) >= 32767).any())
        for mode in BORDERS:
            cval = tuple(int(v) for v in rng.integers(0, 256, 3))
            ref = cv2.warpAffine(src, M, (ow, oh), borderMode=mode, borderValue=cval)
            assert np.array_equal(O.warp_linear_u8(src, M, (ow, oh), mode, cval), ref), (t, mode)
    assert kind != 'singular' or saturated > 0


def test_oracle_resize_u8_random_sizes():
    rng = np.random.default_rng(11)
    for _ in range(200):
        h, w, oh, ow = (int(v) for v in rng.integers(1, 70, 4))
        src = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        assert np.array_equal(O.resize_linear_u8(src, (ow, oh)), cv2.resize(src, (ow, oh), interpolation=cv2.INTER_LINEAR)), (h, w, oh, ow)
