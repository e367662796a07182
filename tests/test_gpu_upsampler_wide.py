"""gpu: RealESRGANer on the device for uint16, float32 and float64 images (cfb_rrdb_forward_tiles, RealESRGANer.enhance_batch),
INTER_LANCZOS4 on uint16 images (cfb_resize_lanczos4_u16) against cv2, and restore_images upsampling the float64 faces of gray
photos in one batch.  The reference throughout is ``_enhance_host``: the reference's enhance with cv2 on the host."""
import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import wholeimage as WI
from tests.test_gpu_upsampler_batch import HostChain, _imgs, _net, _spy

cv2 = pytest.importorskip('cv2')
pytestmark = pytest.mark.gpu
DEV = 'cuda'
F32_ABOVE_256 = float(np.nextafter(np.float32(256), np.float32(300)))       # the first float32 above 256


def wide_images(kind, n, h, w, seed):
    """n images of one kind whose per-image max_range alternates: image 0 is 16-bit to enhance, image 1 is 8-bit (a float
    image with one element at 256, or for float64 just above 256 but 256 in float32), image 2 is 16-bit by one element just
    above 256; the float images carry negative values."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        if kind == 'uint16':
            img = rng.integers(0, (65536, 256, 257)[i % 3], (h, w, 3)).astype(np.uint16)
            if i % 3 == 2:
                img[h // 2, w // 3, 1] = 257
        else:
            dt = np.float32 if kind == 'float32' else np.float64
            hi = (40000.0, 255.0, 255.0)[i % 3]
            img = rng.uniform(-30.0, hi, (h, w, 3)).astype(dt)
            if i % 3 == 1:
                img[h // 3, w // 2, 0] = 256.0 + (1e-9 if dt == np.float64 else 0.0)      # not above 256 in float32
            if i % 3 == 2:
                img[h // 2, w // 3, 2] = F32_ABOVE_256
        out.append(img)
    return np.stack(out)


def _check_equal(got, ref, what):
    got = got.cpu().numpy()
    assert got.dtype == ref.dtype and got.shape == ref.shape, f'{what}: {got.dtype} {got.shape} vs {ref.dtype} {ref.shape}'
    d = got != ref
    assert not d.any(), f'{what}: {int(d.sum())} elements differ'


@pytest.mark.parametrize('precision', ['fp32', 'fp16'])
@pytest.mark.parametrize('pre_pad', [0, 10])
@pytest.mark.parametrize('tile', [0, 24])
@pytest.mark.parametrize('scale', [2, 4])
def test_enhance_batch_wide_equals_enhance_host(scale, tile, pre_pad, precision):
    net = _net(scale, precision=precision)
    er = cb.RealESRGANer(scale=scale, model=net, tile=tile, tile_pad=6, pre_pad=pre_pad, device=DEV)
    H, W = 37, 45                                         # odd: mod pad at x2; tile 24 / pad 6 leaves ragged edge tiles
    for kind in ('uint16', 'float32', 'float64'):
        imgs = wide_images(kind, 3, H, W, scale * 100 + tile + pre_pad)
        refs = [er._enhance_host(im)[0] for im in imgs]
        assert [r.dtype for r in refs] == [np.uint16, np.uint8, np.uint16]
        x = torch.from_numpy(imgs).to(DEV)
        for mt in (1, None):
            res = er.enhance_batch(x, max_tiles=mt)
            assert isinstance(res, list) and len(res) == 3
            for i, (r, ref) in enumerate(zip(res, refs)):
                assert r.is_cuda
                _check_equal(r, ref, f'{kind} image {i}, max_tiles {mt}')
        # batch 1 and enhance() give the same bytes
        _check_equal(er.enhance_batch(x[1:2])[0], refs[1], f'{kind} alone')
        e, mode = er.enhance(imgs[2])
        assert mode == 'RGB' and e.dtype == refs[2].dtype and np.array_equal(e, refs[2])
    r = np.concatenate([x.ravel() for x in refs if x.dtype == np.uint16])
    assert (r == 0).any() and (r == 65535).any(), 'clamp exercised at both ends'
    torch.cuda.synchronize()
    cb.check_async_status()


@pytest.mark.parametrize('outscale', [3, 1.5, 2.5])
def test_enhance_batch_wide_outscale_lanczos(outscale):
    net = _net(2)
    er = cb.RealESRGANer(scale=2, model=net, tile=0, pre_pad=10, device=DEV)
    for kind in ('uint16', 'float64'):
        imgs = wide_images(kind, 3, 31, 27, 7)
        refs = [er._enhance_host(im, outscale=outscale)[0] for im in imgs]
        res = er.enhance_batch(torch.from_numpy(imgs).to(DEV), outscale=outscale, lanczos=True)
        for i, (r, ref) in enumerate(zip(res, refs)):
            assert ref.shape == (int(31 * outscale), int(27 * outscale), 3)
            _check_equal(r, ref, f'{kind} image {i} at x{outscale}')
        e, _ = er.enhance(imgs[0], outscale=outscale)
        assert e.dtype == np.uint16 and np.array_equal(e, refs[0])
    with pytest.raises(NotImplementedError, match='lanczos=True'):
        er.enhance_batch(torch.from_numpy(imgs).to(DEV), outscale=3)


def test_enhance_routes_wide_images_to_the_device(monkeypatch):
    er = cb.RealESRGANer(scale=2, model=_net(2), tile=0, pre_pad=0, device=DEV)
    calls = []
    orig = er._enhance_host
    monkeypatch.setattr(er, '_enhance_host', lambda *a, **k: calls.append(a[0].dtype) or orig(*a, **k))
    for kind in ('uint16', 'float32', 'float64'):
        er.enhance(wide_images(kind, 1, 20, 24, 3)[0])
        er.enhance(wide_images(kind, 1, 20, 24, 3)[0], outscale=3)
    assert calls == []
    er.enhance(np.zeros((20, 24), np.uint16))                 # 2-D gray and BGRA stay on the host
    er.enhance(np.zeros((20, 24, 4), np.float32))
    assert calls == [np.uint16, np.float32]
    with pytest.raises(NotImplementedError):                # and enhance_batch still refuses them
        er.enhance_batch(torch.zeros(1, 20, 24, 4, dtype=torch.float32, device=DEV))
    with pytest.raises(NotImplementedError):
        er.enhance_batch(torch.empty(1, 20, 24, dtype=torch.uint16, device=DEV))


def test_forward_tiles_u8_kind_equals_the_u8_entry_point():
    """cfb_rrdb_forward_tiles with uint8 images: a uint8 canvas equals cfb_rrdb_forward_u8_tiles, a uint16 canvas holds the
    same values; max_range is 255 for every image."""
    net = _net(2)
    er = cb.RealESRGANer(scale=2, model=net, tile=24, tile_pad=6, pre_pad=10, device=DEV)
    imgs = torch.from_numpy(_imgs(2, 37, 45, 4)).to(DEV)
    ref = er.enhance_batch(imgs)
    lib = cb._lib.load()
    groups = er.tile_groups(2, 37, 45, None, lambda n, th, tw: lib.cfb_rrdb_workspace_bytes(net._handle(), n, th, tw))
    mr = torch.zeros(2, dtype=torch.int32, device=DEV)
    for dt in (torch.uint8, torch.uint16):
        out = torch.empty((2, 74, 90, 3), dtype=dt, device=DEV)     # every canvas pixel is written
        for th, tw, rows in groups:
            net.forward_tiles(imgs, er.pre_pad, rows, th, tw, out, mr)
        assert mr.tolist() == [255, 255]
        assert torch.equal(out.view(torch.int16).to(torch.uint8) if dt == torch.uint16 else out, ref)


def test_non_finite_float_input():
    """NaN: no fault, a clean status word, and the dtype numpy's maximum picks (a NaN maximum is not above 256: uint8).
    An infinity reaches the network's fp16 operand planes, whose range guard reports it as it does for RRDBNet.forward; the
    status word is clean again after that report and the next call is exact."""
    er = cb.RealESRGANer(scale=2, model=_net(2), tile=0, pre_pad=10, device=DEV)
    imgs = wide_images('float32', 3, 24, 20, 9)
    imgs[0, 3, 4, 0] = np.nan                            # with values up to 40000: NaN still makes it 8-bit
    imgs[2, 9, 9, 0] = np.nan                            # with one value above 256
    res = er.enhance_batch(torch.from_numpy(imgs).to(DEV))
    torch.cuda.synchronize()
    cb.check_async_status()
    assert [r.dtype for r in res] == [torch.uint8] * 3 and [r.shape for r in res] == [(48, 40, 3)] * 3
    _check_equal(res[1], er._enhance_host(imgs[1])[0], 'finite image beside NaN images')
    for v in (np.inf, -np.inf):
        bad = imgs[1:2].copy()
        bad[0, 5, 6, 1] = v
        try:
            r = er.enhance_batch(torch.from_numpy(bad).to(DEV))
            torch.cuda.synchronize()
            cb.check_async_status()
            assert r[0].dtype == (torch.uint16 if v > 0 else torch.uint8)
        except RuntimeError as e:
            assert 'fp16 operand overflow' in str(e), str(e)
        torch.cuda.synchronize()
        cb.check_async_status()
        _check_equal(er.enhance_batch(torch.from_numpy(imgs[1:2]).to(DEV))[0], er._enhance_host(imgs[1])[0], 'after an infinity')


# ---- INTER_LANCZOS4 on uint16 ----------------------------------------------------------------------------------------
LZ_CASES = [(41, 53, 82, 106), (41, 53, 20, 26), (41, 53, 61, 79), (1, 37, 2, 74), (37, 1, 55, 1), (3, 29, 6, 58),
            (29, 3, 14, 1), (517, 389, 1000, 300), (33, 31, 33, 30), (24, 36, 24, 36), (1080, 1920, 540, 960)]


@pytest.mark.parametrize('case', LZ_CASES, ids=lambda c: '{}x{}-{}x{}'.format(*c))
def test_resize_lanczos4_u16_equals_cv2(case):
    h, w, oh, ow = case
    rng = np.random.default_rng(h + w)
    imgs = rng.integers(0, 65536, (2, h, w, 3)).astype(np.uint16)
    imgs[1, ::3] = 65535                                    # saturated rows: the negative lobes meet the clamp
    out = cb.resize_lanczos4(torch.from_numpy(imgs).to(DEV), (ow, oh))
    assert out.dtype == torch.uint16 and out.shape == (2, oh, ow, 3)
    for i in range(2):
        ref = cv2.resize(imgs[i], (ow, oh), interpolation=cv2.INTER_LANCZOS4)
        _check_equal(out[i], ref, f'image {i}')
        _check_equal(cb.resize_lanczos4(torch.from_numpy(imgs[i]).to(DEV), (ow, oh)), ref, f'image {i} alone')


# ---- restore_images: the float64 faces of gray photos ------------------------------------------------------------------
from tests.test_gpu_wholeimage import nets, whole_images  # noqa: E402,F401  (the module fixture)
from tests.test_gpu_lanczos_gray import _to_gray, gray_reference_loop  # noqa: E402


def test_restore_images_gray_faces_in_one_batch(nets, monkeypatch):
    up = cb.RealESRGANer(scale=2, model=_net(2, seed=12), tile=400, tile_pad=40, pre_pad=0, device=DEV)
    host = HostChain(up)
    # dark gray frames: the colour transfer keeps their faces below 256
    imgs = [(_to_gray(whole_images()[-1]) * 0.5).astype(np.uint8), whole_images()[-1],
            (_to_gray(whole_images()[-2]) * 0.6).astype(np.uint8)]
    refs = [gray_reference_loop(im, nets.net, nets.det, nets.parser, face_upsampler=host) for im in imgs]
    assert [g for _, _, g in refs] == [True, False, True]
    gray_with_faces = sum(1 for _, f, g in refs if g and len(f))
    assert gray_with_faces >= 1 and sum(len(f) for _, f, g in refs if g) >= 2, 'the gray images need faces'
    calls = _spy(up)
    batches = []
    orig = up.enhance_batch
    monkeypatch.setattr(up, 'enhance_batch', lambda x, **k: batches.append(x.dtype) or orig(x, **k))
    for max_batch in (1, 4):
        res = cb.restore_images(imgs, nets.net, nets.det, parser=nets.parser, face_upsampler=up, max_batch=max_batch)
        for i, ((ref, _, _), out) in enumerate(zip(refs, res)):
            assert out.dtype == ref.dtype and np.array_equal(out, ref), f'image {i}, max_batch {max_batch}: ' \
                                                                          f'{int((out != ref).sum())} bytes differ'
    assert not calls, 'enhance is not called per face'
    # one enhance_batch of float64 faces per chunk with gray faces: per gray image at max_batch 1, once at max_batch 4
    assert batches.count(torch.float64) == gray_with_faces + 1
    # a gray face the colour transfer pushed above 256 is 16-bit to enhance: still not pasted
    adain = WI.gray_adain_faces
    monkeypatch.setattr(WI, 'gray_adain_faces', lambda r, c: adain(r, c) * 0.2 + 270.0)
    k = next(i for i, (_, f, g) in enumerate(refs) if g and len(f))
    with pytest.raises(NotImplementedError, match='16-bit'):
        cb.restore_images(imgs[k:k + 1], nets.net, nets.det, parser=nets.parser, face_upsampler=up)
    torch.cuda.synchronize()
    cb.check_async_status()
