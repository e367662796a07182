"""The numpy INTER_AREA restatement (oracle/resize_area_oracle.py) against cv2.resize on the CPU."""
import numpy as np
import pytest

from oracle import resize_area_oracle as O

cv2 = pytest.importorskip('cv2')

# (h, w, out_h, out_w): integer factors, the detection sizes of get_face_landmarks_5(resize=640), odd sizes, 1-pixel edges
CASES = [
    (64, 96, 32, 48),            # 2x: (sum + 2) >> 2
    (90, 123, 30, 41),           # 3x: cvRound(sum * (1.f / 9))
    (60, 90, 30, 30),            # 2x by 3x
    (48, 20, 12, 20),            # 4x by 1x
    (1080, 1440, 640, 853),      # 1080 -> 640
    (853, 1280, 640, 960),       # 853 -> 640
    (1080, 1920, 640, 1137),     # a 1080p frame
    (1920, 1080, 1137, 640),     # portrait
    (1280, 1920, 640, 960),      # 2x at detection size
    (1920, 2880, 640, 960),      # 3x at detection size
    (101, 77, 37, 29),
    (641, 643, 640, 641),
    (7, 1, 3, 1),
    (1, 9, 1, 4),
    (5, 5, 1, 1),
    (13, 2, 4, 1),
    (33, 31, 33, 30),            # one axis unchanged
]


def case_id(c):
    return '{}x{}-{}x{}'.format(*c)


@pytest.mark.parametrize('case', CASES, ids=case_id)
def test_resize_area_matches_cv2(case):
    h, w, oh, ow = case
    rng = np.random.default_rng(h * 7919 + w)
    src = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    ref = cv2.resize(src, (ow, oh), interpolation=cv2.INTER_AREA)
    assert np.array_equal(O.resize_area_u8(src, (ow, oh)), ref)


def test_resize_area_smooth_and_saturated_images():
    """Ramps and constant 0 / 255 images: many pre-cast values near a .5 boundary and at the clamp."""
    for h, w, oh, ow in [(1080, 1920, 640, 1137), (90, 123, 30, 41), (101, 77, 37, 29)]:
        yy, xx = np.mgrid[:h, :w]
        ramp = np.stack([(xx * 255 // max(w - 1, 1)), (yy * 255 // max(h - 1, 1)), (xx + yy) % 256], -1).astype(np.uint8)
        for src in (ramp, np.zeros((h, w, 3), np.uint8), np.full((h, w, 3), 255, np.uint8)):
            ref = cv2.resize(src, (ow, oh), interpolation=cv2.INTER_AREA)
            assert np.array_equal(O.resize_area_u8(src, (ow, oh)), ref)


def test_both_paths_are_covered():
    fast = [c for c in CASES if O.is_area_fast(O.inverse_scale(c[1], c[3]), O.inverse_scale(c[0], c[2]))[0]]
    assert 0 < len(fast) < len(CASES)


@pytest.mark.parametrize('hw', [(1080, 1920), (853, 1280), (1920, 1080), (2160, 3840), (641, 700)])
def test_detection_size(hw):
    """The helper's target size: scale = 640 / min(h, w) in double, int() of both products."""
    h, w = hw
    oh, ow, scale = O.detection_size(h, w)
    assert scale < 1 and min(oh, ow) in (639, 640)
    assert (oh, ow) == (int(h * (640 / min(h, w))), int(w * (640 / min(h, w))))
