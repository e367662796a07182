"""gpu: the paste-back, the crop warp and the INTER_LINEAR resize on the device over seeded scenes and random geometry.
Each result is held to the CPU oracle (oracle/pasteback_oracle.py, oracle/gray_oracle.py) bit for bit, and, where cv2 is
installed, to cv2 itself: the paste to the reference's chain written out with cv2 (tests/paste_scenes.py), byte for byte.
The scenes are those of tests/test_paste_sweep_cpu.py, which holds the oracle to the same cv2 chain."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from codeformer_b200 import pasteback as PB
from oracle import pasteback_oracle as O
from tests import paste_scenes as PS

pytestmark = pytest.mark.gpu
DEV = 'cuda'
BORDERS = {'constant': O.BORDER_CONSTANT, 'reflect101': O.BORDER_REFLECT101, 'reflect': O.BORDER_REFLECT}


def _cuda(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def device_paste(sc):
    """paste_faces on the scene, as a caller passes it: matrices as get_inverse_affine leaves them."""
    return PB.paste_faces(_cuda(sc.img), _cuda(sc.faces), sc.invs, sc.upscale, upsample_img=_cuda(sc.upsample),
                          masks=_cuda(sc.masks)).cpu().numpy()


@pytest.mark.parametrize('i', range(PS.N_SCENES))
def test_paste_matches_oracle(i):
    """The image, and for uint8 faces the float canvas before the cast (the debug canvas) and w_edge, equal the oracle's."""
    sc = PS.scene(i)
    ref, canvas, info = PS.oracle_paste(sc)
    out = device_paste(sc)
    assert out.dtype == ref.dtype and np.array_equal(out, ref), f'{int((out != ref).sum())} values differ'
    if not sc.f64:
        S = sc.faces.shape[1]
        _, w_edge, dbg = PB._paste(_cuda(sc.img), _cuda(sc.faces), PS.adjusted(sc), sc.upscale, S, _cuda(sc.masks),
                                   _cuda(sc.upsample), debug=True)
        assert list(w_edge) == [d['w_edge'] for d in info]
        dbg, want = dbg.cpu().numpy(), canvas.astype(np.float32)
        assert np.array_equal(dbg, want), f'{int((dbg != want).sum())} canvas values differ'


@pytest.mark.parametrize('i', range(PS.N_SCENES))
def test_paste_matches_cv2(i):
    cv2 = pytest.importorskip('cv2')
    sc = PS.scene(i)
    out = device_paste(sc)
    ref = PS.cv2_paste(cv2, sc)[0]
    assert out.dtype == ref.dtype and np.array_equal(out, ref), f'{int((out != ref).sum())} values differ'


@pytest.mark.parametrize('i', [2, 3, 8, 14, 20, 22, 28])
def test_paste_multi_matches_oracle(i):
    """paste_faces_multi over the scene's image and its mirror image, the faces dealt to them in turn: each image equals
    the oracle's paste of its own faces."""
    sc = PS.scene(i)
    imgs = np.stack([sc.img, sc.img[::-1, ::-1]])
    ups = None if sc.upsample is None else np.stack([sc.upsample, sc.upsample[::-1, ::-1]])
    img_index = [j % 2 for j in range(len(sc.faces))]
    out = PB.paste_faces_multi(_cuda(imgs), _cuda(sc.faces), sc.invs, img_index, sc.upscale, upsample_imgs=_cuda(ups),
                               masks=_cuda(sc.masks)).cpu().numpy()
    for k in range(2):
        sel = [j for j in range(len(sc.faces)) if img_index[j] == k]
        sub = SimpleNamespace(**{**vars(sc), 'img': imgs[k], 'faces': sc.faces[sel], 'invs': [sc.invs[j] for j in sel],
                                 'masks': None if sc.masks is None else sc.masks[sel], 'upsample': None if ups is None else ups[k]})
        ref = PS.oracle_paste(sub)[0]
        assert np.array_equal(out[k], ref), f'image {k}: {int((out[k] != ref).sum())} values differ'


def _warp_cases(kind, seed):
    rng = np.random.default_rng(seed)
    for t in range(10):
        sh, sw = (int(v) for v in rng.integers(1, 90, 2)) if t % 4 else (1 + t % 3, 1 + t % 2)
        S = (1, 7, 96, 257, 512)[t % 5]
        src = rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8)
        yield t, src, [PS.general_affine(rng, kind, sw, sh, S, S) for _ in range(3)], S, tuple(int(v) for v in rng.integers(0, 256, 3))


@pytest.mark.parametrize('mode', list(BORDERS))
@pytest.mark.parametrize('kind', ['shear', 'flip', 'scale', 'singular'])
def test_warp_faces_general_affines(kind, mode):
    """warp_faces and warp_faces_multi equal the oracle (and cv2.warpAffine) for general matrices, sources of 1 x 1 up,
    output sizes other than 512 and any border value; the near-singular matrices need cv2's int16 source coordinates."""
    try:
        import cv2
    except ImportError:
        cv2 = None
    for t, src, Ms, S, cval in _warp_cases(kind, len(kind) * 7 + len(mode)):
        out = PB.warp_faces(_cuda(src), Ms, S, mode, cval).cpu().numpy()
        multi = PB.warp_faces_multi(_cuda(np.stack([src[::-1].copy(), src])), Ms, [1, 1, 1], S, mode, cval).cpu().numpy()
        for j, M in enumerate(Ms):
            ref = O.warp_linear_u8(src, M, (S, S), BORDERS[mode], cval)
            assert np.array_equal(out[j], ref) and np.array_equal(multi[j], ref), (t, j)
            if cv2 is not None:
                assert np.array_equal(ref, cv2.warpAffine(src, M, (S, S), borderMode=BORDERS[mode], borderValue=cval)), (t, j)


def test_resize_linear_random_sizes():
    """resize_linear (single and batched) equals the oracle and cv2 over random size pairs: enlarging, shrinking, exact
    halvings and 1-pixel sides."""
    try:
        import cv2
    except ImportError:
        cv2 = None
    rng = np.random.default_rng(12)
    pairs = [tuple(int(v) for v in rng.integers(1, 80, 4)) for _ in range(60)] + [(40, 60, 20, 30), (1, 9, 1, 4), (64, 2, 32, 1)]
    for h, w, oh, ow in pairs:
        src = rng.integers(0, 256, (2, h, w, 3), dtype=np.uint8)
        out = PB.resize_linear(_cuda(src), (ow, oh)).cpu().numpy()
        for k in range(2):
            ref = O.resize_linear_u8(src[k], (ow, oh))
            assert np.array_equal(out[k], ref), (h, w, oh, ow)
            if cv2 is not None:
                assert np.array_equal(ref, cv2.resize(src[k], (ow, oh), interpolation=cv2.INTER_LINEAR)), (h, w, oh, ow)


def test_resize_linear_factor_matches_cv2():
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(13)
    for f in (1, 1.25, 1.5, 2, 2.5, 3, 3.7, 4):
        h, w = (int(v) for v in rng.integers(1, 90, 2))
        src = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        out = PB.resize_linear_factor(_cuda(src), f).cpu().numpy()
        ref = cv2.resize(src, (0, 0), fx=f, fy=f, interpolation=cv2.INTER_LINEAR)
        assert out.shape == ref.shape and np.array_equal(out, ref), (h, w, f)


def test_async_status_clear():
    from codeformer_b200 import _lib
    torch.cuda.synchronize()
    assert _lib.load().cfb_check_async_status() == 0
