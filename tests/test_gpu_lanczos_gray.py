"""gpu: whole-image mode for gray images and any output scale.  INTER_LANCZOS4 on the device against cv2.resize, byte for
byte; RealESRGANer with outscale != scale against cv2 on its own output; the gray branch of add_restored_face against numpy;
the paste of float64 faces against the reference's blend written out with cv2 on the host; restore_images on gray, mixed and
small images and other scales against the per-image loop with this package's drop-ins."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import pasteback as PB
from oracle import gray_oracle as G
from oracle import pasteback_oracle as O
from tests.test_gpu_pasteback import gold                       # noqa: F401  (fixture)
from tests.test_gpu_upsampler_batch import _imgs, _net
from tests.test_gpu_wholeimage import _affines, nets, whole_images   # noqa: F401  (nets: fixture)
from tests.test_oracle_lanczos_gray import CASES, _gray_faces, case_id

cv2 = pytest.importorskip('cv2')
pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _lanczos(img, size):
    return cv2.resize(img, size, interpolation=cv2.INTER_LANCZOS4)


# ---- INTER_LANCZOS4 ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', CASES + [(1080, 1920, 2160, 3840), (2160, 3840, 1080, 1920), (2160, 3840, 3240, 5760)], ids=case_id)
def test_resize_lanczos4_bit_exact(case):
    h, w, oh, ow = case
    imgs = np.random.default_rng(h + w).integers(0, 256, (2, h, w, 3), dtype=np.uint8)
    out = cb.resize_lanczos4(torch.from_numpy(imgs).to(DEV), (ow, oh))
    assert out.shape == (2, oh, ow, 3)
    for i in range(2):
        assert np.array_equal(out[i].cpu().numpy(), _lanczos(imgs[i], (ow, oh))), f'image {i}'
        assert torch.equal(cb.resize_lanczos4(torch.from_numpy(imgs[i]).to(DEV), (ow, oh)), out[i])


def test_resize_lanczos4_saturates_like_cv2():
    yy, xx = np.mgrid[:90, :130]
    check = (((yy // 3 + xx // 3) % 2) * 255).astype(np.uint8)[:, :, None].repeat(3, axis=2)
    for size in [(260, 180), (65, 45), (200, 61)]:
        assert np.array_equal(cb.resize_lanczos4(torch.from_numpy(check).to(DEV), size).cpu().numpy(), _lanczos(check, size))


@pytest.mark.parametrize('outscale', [1, 1.5, 3, 4])
def test_enhance_batch_outscale(outscale):
    er = cb.RealESRGANer(scale=2, model=_net(2), tile=0, pre_pad=10, device=DEV)
    imgs = _imgs(3, 37, 52, 4)
    x = torch.from_numpy(imgs).to(DEV)
    native = er.enhance_batch(x).cpu().numpy()
    out = er.enhance_batch(x, outscale=outscale, lanczos=True).cpu().numpy()
    size = (int(52 * outscale), int(37 * outscale))
    assert out.shape == (3, size[1], size[0], 3)
    for i in range(3):
        assert np.array_equal(out[i], _lanczos(native[i], size)), f'image {i}'
    # enhance() takes the device path and returns what its host branch returns
    dev_out, mode = er.enhance(imgs[0], outscale=outscale)
    host_out, _ = er._enhance_host(imgs[0], outscale)
    assert mode == 'RGB' and np.array_equal(dev_out, out[0]) and np.array_equal(dev_out, host_out)


# ---- the gray branch of add_restored_face --------------------------------------------------------------------------
def _adain_np(restored, cropped, wide=False):
    """adain_npy(bgr2gray(restored), cropped) of facelib/utils/misc.py, written out.  ``wide``: the statistics summed in
    extended precision (numpy's own float64 sums over 262144 rows, one row after another, carry an error of a few 1e-12)."""
    gray = 0.2989 * restored[:, :, 2] + 0.5870 * restored[:, :, 1] + 0.1140 * restored[:, :, 0]
    content = gray[:, :, None].repeat(3, axis=2)

    def mean_std(f):
        flat = f.reshape(-1, 3).astype(np.longdouble if wide else np.float64)
        return flat.mean(axis=0).astype(np.float64), np.sqrt(flat.var(axis=0) + 1e-5).astype(np.float64)
    smean, sstd = mean_std(cropped)
    cmean, cstd = mean_std(content)
    return (content - cmean) / cstd * sstd + smean, np.stack([cmean, cstd, smean, sstd])


def test_gray_adain_faces():
    restored, cropped = np.stack(_gray_faces(32, 1)), np.stack(_gray_faces(32, 2))
    restored[3] = 77                                            # a constant face: std = sqrt(1e-5)
    cropped[4] = (250 + np.random.default_rng(0).integers(-1, 2, (512, 512, 3))).astype(np.uint8)     # mean 250 +- 1
    restored[5] = cropped[4]
    r, c = torch.from_numpy(restored).to(DEV), torch.from_numpy(cropped).to(DEV)
    out, stats = cb.gray_adain_faces(r, c, with_stats=True)
    assert out.dtype == torch.float64 and out.shape == (32, 512, 512, 3) and stats.shape == (32, 4, 3)
    out_h, stats_h = out.cpu().numpy(), stats.cpu().numpy()
    for i in range(32):
        ref, ref_stats = _adain_np(restored[i], cropped[i], wide=True)
        np.testing.assert_allclose(stats_h[i], ref_stats, rtol=1e-13, atol=0, err_msg=f'face {i}')
        assert np.abs(out_h[i] - ref).max() < 1e-9, f'face {i}'     # the constant face scales the mean's rounding by 1.4e4
        ref, ref_stats = _adain_np(restored[i], cropped[i])                      # numpy as the reference runs it
        np.testing.assert_allclose(stats_h[i], ref_stats, rtol=1e-10, atol=0, err_msg=f'face {i}')
        # on the constant face numpy's own mean (off by 4e-11) is scaled by sstd / sqrt(1e-5) = 1.4e4
        assert np.abs(out_h[i] - ref).max() < (1e-8 if i != 3 else 1e-5), f'face {i}'
    assert abs(stats_h[3, 1, 0] - np.sqrt(1e-5)) < 1e-15 and np.isfinite(out_h).all()
    assert torch.equal(cb.gray_adain_faces(r, c), out)                               # the same on every run
    for i in (0, 3, 17, 31):                                                          # and for a face alone
        assert torch.equal(cb.gray_adain_faces(r[i:i + 1], c[i:i + 1])[0], out[i])


# ---- the paste of float64 faces ------------------------------------------------------------------------------------
def host_paste(img, faces, invs, upscale, masks=None, upsample_img=None):
    """paste_faces_to_input_image:372-499 for faces of any dtype, with cv2 on the host; ``masks`` stands for the parsing
    network's MASK_COLORMAP image (0/255) of each face.  ``invs`` are the matrices after the reference's offset."""
    h, w = img.shape[:2]
    h_up, w_up = int(h * upscale), int(w * upscale)
    if upsample_img is None:
        canvas = cv2.resize(img, (w_up, h_up), interpolation=cv2.INTER_LINEAR)
    else:
        canvas = _lanczos(upsample_img, (w_up, h_up))
    for i, (face, inv) in enumerate(zip(faces, invs)):
        fs = face.shape[:2]
        inv_restored = cv2.warpAffine(face, inv, (w_up, h_up))
        inv_mask = cv2.warpAffine(np.ones(fs, np.float32), inv, (w_up, h_up))
        erosion = cv2.erode(inv_mask, np.ones((int(2 * upscale), int(2 * upscale)), np.uint8))
        pasted = erosion[:, :, None] * inv_restored
        w_edge = int(np.sum(erosion) ** 0.5) // 20
        center = cv2.erode(erosion, np.ones((w_edge * 2, w_edge * 2), np.uint8))
        soft = cv2.GaussianBlur(center, (w_edge * 2 + 1, w_edge * 2 + 1), 0)[:, :, None]
        if masks is not None:
            pm = cv2.GaussianBlur(cv2.GaussianBlur(masks[i].astype(np.float64), (101, 101), 11), (101, 101), 11)
            pm[:10, :] = 0
            pm[-10:, :] = 0
            pm[:, :10] = 0
            pm[:, -10:] = 0
            pm = cv2.warpAffine(cv2.resize(pm / 255., fs), inv, (w_up, h_up), flags=3)[:, :, None]
            fuse = (pm < soft).astype('int')
            soft = pm * fuse + soft * (1 - fuse)
        canvas = soft * pasted + (1 - soft) * canvas
    return canvas.astype(np.uint16) if np.max(canvas) > 256 else canvas.astype(np.uint8)


def _paste_inputs(upscale, seed=3):
    rng = np.random.default_rng(seed)
    h, w = 280, 360
    img = cv2.cvtColor(cv2.cvtColor(O.synthetic_background(h, w, seed), cv2.COLOR_BGR2GRAY), cv2.COLOR_GRAY2BGR)
    aff = _affines(rng, 3, h, w)
    invs = PB.adjust_inverse_affines([cv2.invertAffineTransform(a) * upscale for a in aff], upscale, False)
    restored, cropped = np.stack(_gray_faces(3, seed)), np.stack(_gray_faces(3, seed + 1))
    masks = (rng.random((3, 512, 512)) < 0.7).astype(np.uint8) * 255
    return img, invs, restored, cropped, masks


@pytest.mark.parametrize('other_bg', [False, True])
@pytest.mark.parametrize('upscale,use_parse', [(1, False), (2, False), (2, True), (1, True)])
def test_f64_paste_matches_cv2(upscale, use_parse, other_bg):
    img, invs, restored, cropped, masks = _paste_inputs(upscale)
    bg = O.synthetic_background(150, 190, 8) if other_bg else None     # another size: INTER_LANCZOS4 to the output size
    faces = cb.gray_adain_faces(torch.from_numpy(restored).to(DEV), torch.from_numpy(cropped).to(DEV))
    dmasks = torch.from_numpy(masks).to(DEV) if use_parse else None
    out, _ = PB._paste(torch.from_numpy(img).to(DEV), faces, invs, upscale, 512, dmasks,
                       None if bg is None else torch.from_numpy(bg).to(DEV))
    out = out.cpu().numpy()
    host_faces = list(faces.cpu().numpy())
    # the same float64 faces through the numpy restatement (taps of the soft mask's blur summed in order, as on the device):
    # the warp and the blend agree exactly
    if not use_parse:
        same = G.final_cast(G.paste_faces_f64(img, host_faces, [m - [[0, 0, 0.5 * upscale if upscale > 1 else 0]] * 2 for m in invs],
                                              upscale, None, None if bg is None else _lanczos(bg, (360 * upscale, 280 * upscale))))
        assert out.dtype == same.dtype == np.uint8 and np.array_equal(out, same), f'{int((out != same).sum())} bytes differ'
    # the same faces through cv2 on the host: cv2's float32 GaussianBlur rounds the soft mask's last bit differently (as for
    # uint8 faces), so a truncation boundary may move by one level on a few pixels
    same = host_paste(img, host_faces, invs, upscale, masks if use_parse else None, bg)
    d = np.abs(out.astype(np.int16) - same)
    print('pixels off by one level against cv2, same faces:', int((d != 0).sum()), 'of', d.size)
    assert out.dtype == same.dtype == np.uint8 and d.max() <= 1 and (d != 0).mean() <= 1e-4
    # numpy's faces differ from the device's in their last bits as well
    ref = host_paste(img, [_adain_np(r, c)[0] for r, c in zip(restored, cropped)], invs, upscale, masks if use_parse else None, bg)
    d = np.abs(out.astype(np.int16) - ref)
    print('pixels off by one level against cv2, numpy faces:', int((d != 0).sum()), 'of', d.size)
    assert d.max() <= 1 and (d != 0).mean() <= 1e-4
    assert (out != host_paste(img, [], [], upscale, None, bg)).mean() > 0.05      # the faces are there


def test_f64_paste_multi_and_drop_in():
    """paste_faces_multi with float64 faces equals paste_faces per image; the drop-ins (add_restored_face, then
    paste_faces_to_input_image with a differently-sized upsample_img) equal the device-level call."""
    img, invs, restored, cropped, _ = _paste_inputs(2)
    raw = [m.copy() for m in invs]
    for m in raw:
        m[:, 2] -= 1.0                       # undo the offset: the public functions add it themselves
    imgs = torch.from_numpy(np.stack([img, img[::-1].copy()])).to(DEV)
    faces = cb.gray_adain_faces(torch.from_numpy(restored).to(DEV), torch.from_numpy(cropped).to(DEV))
    multi = cb.paste_faces_multi(imgs, faces, raw, [1, 0, 1], 2)
    assert torch.equal(multi[0], cb.paste_faces(imgs[0], faces[1:2], raw[1:2], 2))
    assert torch.equal(multi[1], cb.paste_faces(imgs[1], faces[[0, 2]], [raw[0], raw[2]], 2))
    helper = SimpleNamespace(input_img=img, upscale_factor=2, face_size=(512, 512), restored_faces=[], is_gray=True,
                             inverse_affine_matrices=[m.copy() for m in raw], use_parse=False, face_parse=None)
    for r, c in zip(restored, cropped):
        cb.add_restored_face(helper, r, c)
    assert all(f.dtype == np.float64 and np.array_equal(f, g) for f, g in zip(helper.restored_faces, faces.cpu().numpy()))
    bg = O.synthetic_background(150, 190, 8)
    out = cb.paste_faces_to_input_image(helper, upsample_img=bg, lanczos=True)
    dev = cb.paste_faces(imgs[0], faces, raw, 2, upsample_img=torch.from_numpy(bg).to(DEV)).cpu().numpy()
    assert out.dtype == np.uint8 and np.array_equal(out, dev)
    colour, face = SimpleNamespace(restored_faces=[], is_gray=False), restored[0]
    cb.add_restored_face(colour, face, cropped[0])
    assert colour.restored_faces[0] is face


def test_bright_gray_face_returns_uint16():
    """A face the colour transfer pushed above 256: the reference returns astype(np.uint16) for that image only."""
    img, invs, restored, cropped, _ = _paste_inputs(1)
    faces = cb.gray_adain_faces(torch.from_numpy(restored).to(DEV), torch.from_numpy(cropped).to(DEV))
    faces[1] = faces[1] * 0.2 + 270.0
    out, _ = PB._paste(torch.from_numpy(img).to(DEV), faces, invs, 1, 512, None, None)
    ref = G.final_cast(G.paste_faces_f64(img, list(faces.cpu().numpy()), [m.copy() for m in invs], 1))
    assert ref.dtype == np.uint16 and out.dtype == torch.uint16 and np.array_equal(out.cpu().numpy(), ref)
    cv = host_paste(img, list(faces.cpu().numpy()), invs, 1)
    assert cv.dtype == np.uint16 and np.abs(out.cpu().numpy().astype(np.int32) - cv).max() <= 1
    imgs = torch.from_numpy(np.stack([img, img])).to(DEV)
    wide = {}
    multi = cb.paste_faces_multi(imgs, faces, [m.copy() for m in invs], [0, 1, 0], 1, wide=wide)
    assert sorted(wide) == [1] and multi.dtype == torch.uint8
    assert torch.equal(wide[1], PB._paste(imgs[1], faces[1:2], invs[1:2], 1, 512, None, None)[0])
    assert torch.equal(multi[0], PB._paste(imgs[0], faces[[0, 2]], [invs[0], invs[2]], 1, 512, None, None)[0])


def test_float_face_above_256_is_16_bit_to_enhance():
    """RealESRGANer.enhance reads a float face above 256 as 16-bit and returns uint16 (realesrgan_utils.py:193-199); the host
    route of gray faces through a face upsampler inherits that, and restore_images refuses to paste such a face."""
    er = cb.RealESRGANer(scale=2, model=_net(2), tile=0, pre_pad=0, device=DEV)
    face = np.full((32, 32, 3), 300.0)
    assert er.enhance(face, outscale=2)[0].dtype == np.uint16
    assert er.enhance(np.full((32, 32, 3), 200.0), outscale=2)[0].dtype == np.uint8


# ---- restore_images ---------------------------------------------------------------------------------------------------
def gray_reference_loop(img, net, det, parser, upscale=2, bg_upsampler=None, face_upsampler=None):
    """inference_codeformer.py:178-229 for one image, gray or not, with this package's per-image drop-ins and host cv2 for
    read_image and the detector's resize (tests/test_gpu_wholeimage.py's reference_loop with the gray branch)."""
    from codeformer_b200.wholeimage import FACE_TEMPLATE, is_gray
    helper = SimpleNamespace(upscale_factor=upscale, face_size=(512, 512), face_template=FACE_TEMPLATE, pad_blur=False,
                             all_landmarks_5=[], det_faces=[], affine_matrices=[], cropped_faces=[], restored_faces=[],
                             inverse_affine_matrices=[], use_parse=parser is not None, face_parse=parser, is_gray=is_gray(img))
    helper.input_img = img
    if min(img.shape[:2]) < 512:
        f = 512.0 / min(img.shape[:2])
        helper.input_img = cv2.resize(img, (0, 0), fx=f, fy=f, interpolation=cv2.INTER_LINEAR)
    h, w_ = helper.input_img.shape[0:2]
    scale = 640 / min(h, w_)
    input_img = cv2.resize(helper.input_img, (int(w_ * scale), int(h * scale)),
                           interpolation=cv2.INTER_AREA if scale < 1 else cv2.INTER_LINEAR)
    with torch.no_grad():
        bboxes = det.detect_faces(input_img)
    if bboxes is not None and bboxes.shape[0] > 0:
        for bbox in bboxes / scale:
            if np.linalg.norm([bbox[6] - bbox[8], bbox[7] - bbox[9]]) < 5:
                continue
            helper.all_landmarks_5.append(np.array([[bbox[i], bbox[i + 1]] for i in range(5, 15, 2)]))
    PB.align_warp_face(helper)
    with torch.no_grad():
        restored = net.restore_faces(helper.cropped_faces, w=0.5, adain=True) if helper.cropped_faces else []
    for r, c in zip(restored, helper.cropped_faces):
        PB.add_restored_face(helper, r, c)
    bg_img = bg_upsampler.enhance(img, outscale=upscale)[0] if bg_upsampler is not None else None
    for a in helper.affine_matrices:
        helper.inverse_affine_matrices.append(cv2.invertAffineTransform(a) * upscale)
    out = PB.paste_faces_to_input_image(helper, upsample_img=bg_img, face_upsampler=face_upsampler, lanczos=True)
    return out, helper.restored_faces, helper.is_gray


def _to_gray(img):
    return cv2.cvtColor(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), cv2.COLOR_GRAY2BGR)


def test_restore_images_gray_and_colour_mixed(nets):
    base = whole_images()
    imgs = [_to_gray(base[1]), base[2], _to_gray(base[-1]), base[-2], _to_gray(base[0])]     # base[1] / base[2]: one size
    refs = [gray_reference_loop(im, nets.net, nets.det, nets.parser) for im in imgs]
    assert [g for _, _, g in refs] == [True, False, True, False, True]
    assert sum(len(f) for _, f, g in refs if g) >= 2, 'the gray images need faces'
    res, _, faces = cb.restore_images(imgs, nets.net, nets.det, parser=nets.parser, max_batch=4, return_faces=True)
    for i, ((ref, rf, g), out) in enumerate(zip(refs, res)):
        assert out.dtype == ref.dtype and np.array_equal(out, ref), f'image {i}: {int((out != ref).sum())} bytes differ'
        assert faces[i].shape[0] == len(rf) and (not len(rf) or faces[i].dtype == (np.float64 if g else np.uint8))
        for a, b in zip(faces[i], rf):
            assert np.array_equal(a, b)
    # the colour images are what a call without the gray ones gives
    alone = cb.restore_images([imgs[1], imgs[3]], nets.net, nets.det, parser=nets.parser)
    assert np.array_equal(alone[0], res[1]) and np.array_equal(alone[1], res[3])
    # no parse masks: the float64 canvas with the float32 first product
    ref = gray_reference_loop(imgs[2], nets.net, nets.det, None, upscale=1)[0]
    assert np.array_equal(cb.restore_images([imgs[2]], nets.net, nets.det, upscale=1)[0], ref)
    cb.check_async_status()


@pytest.mark.parametrize('upscale', [1, 3, 4])
def test_restore_images_other_scales_with_x2_upsampler(nets, upscale):
    """An x2 background upsampler with --upscale 1 / 3 / 4, on a frame and on a 300 x 400 image that read_image enlarges (the
    background then needs the second INTER_LANCZOS4 of paste_faces_to_input_image), gray and colour.  At another scale the
    upsampler is called once per image through enhance, whose network and resize run on the device."""
    bg = cb.RealESRGANer(scale=2, model=_net(2), tile=0, pre_pad=0, device=DEV)
    img = np.ascontiguousarray(whole_images()[-1][:200, :240])
    assert np.array_equal(bg.enhance(img, outscale=upscale)[0], bg._enhance_host(img, upscale)[0])
    small = cv2.resize(whole_images()[0], (400, 300), interpolation=cv2.INTER_AREA)
    imgs = [O.synthetic_background(512, 600, 7), small, _to_gray(small)]
    res = cb.restore_images(imgs, nets.net, nets.det, parser=nets.parser, upscale=upscale, bg_upsampler=bg)
    for i, (im, out) in enumerate(zip(imgs, res)):
        ref = gray_reference_loop(im, nets.net, nets.det, nets.parser, upscale=upscale, bg_upsampler=bg)[0]
        assert out.shape == ref.shape and np.array_equal(out, ref), f'image {i}'
    assert res[1].shape[:2] == (int(512 * upscale), int(683 * upscale))      # read_image: 300 x 400 -> 512 x 683


def test_restore_images_gray_with_face_upsampler(nets):
    """The float64 faces of a gray image go to the face upsampler on the host and come back uint8, as in the reference."""
    up = cb.RealESRGANer(scale=2, model=_net(2), tile=0, pre_pad=0, device=DEV)
    # a dark frame: the colour transfer keeps its faces below 256 (above it a float face is 16-bit to enhance)
    imgs = [(_to_gray(whole_images()[-1]) * 0.5).astype(np.uint8), whole_images()[-1]]
    res = cb.restore_images(imgs, nets.net, nets.det, parser=nets.parser, bg_upsampler=up, face_upsampler=up)
    for i, (im, out) in enumerate(zip(imgs, res)):
        ref = gray_reference_loop(im, nets.net, nets.det, nets.parser, bg_upsampler=up, face_upsampler=up)[0]
        assert np.array_equal(out, ref), f'image {i}'


# ---- what still raises, and what no longer does ----------------------------------------------------------------------------
def test_lanczos_is_opt_in_where_a_size_was_refused(gold):      # noqa: F811
    """enhance_batch and the paste drop-in keep refusing another size unless ``lanczos=True`` asks for the reference's resize;
    draw_box, pad_blur, alpha and 16-bit inputs still raise."""
    er = cb.RealESRGANer(scale=2, model=_net(2), tile=0, pre_pad=10, device=DEV)
    x = torch.from_numpy(_imgs(1, 20, 24, 1)).to(DEV)
    with pytest.raises(NotImplementedError, match='lanczos=True'):
        er.enhance_batch(x, outscale=3)
    assert er.enhance_batch(x, outscale=3, lanczos=True).shape == (1, 60, 72, 3)
    assert torch.equal(er.enhance_batch(x, outscale=2, lanczos=True), er.enhance_batch(x))
    with pytest.raises(ValueError):
        er.enhance_batch(x, outscale=0, lanczos=True)
    g, faces = gold
    img = O.golden_case(g, faces, 'P2', 1)[0]

    def helper(**kw):
        return SimpleNamespace(**{**dict(input_img=img, upscale_factor=1, face_size=(512, 512), restored_faces=[faces[3]],
                                         inverse_affine_matrices=[g['P2_inv'][0].copy()], use_parse=False, face_parse=None), **kw})
    small = np.random.default_rng(1).integers(0, 256, (10, 10, 3), dtype=np.uint8)
    with pytest.raises(NotImplementedError, match='lanczos=True'):
        cb.paste_faces_to_input_image(helper(), upsample_img=small)
    out = cb.paste_faces_to_input_image(helper(), upsample_img=small, lanczos=True)
    ref = host_paste(img, [faces[3]], [g['P2_inv'][0].copy()], 1, None, small)
    assert out.shape == ref.shape and np.abs(out.astype(np.int16) - ref).max() <= 1
    dev = cb.paste_faces(torch.from_numpy(img).to(DEV), torch.from_numpy(faces[3:4].copy()).to(DEV), g['P2_inv'][:1], 1,
                         upsample_img=torch.from_numpy(small).to(DEV))
    assert np.array_equal(dev.cpu().numpy(), out)
    with pytest.raises(NotImplementedError):
        cb.paste_faces_to_input_image(helper(), draw_box=True)
    with pytest.raises(NotImplementedError):
        PB.align_warp_face(helper(pad_blur=True))
    with pytest.raises(NotImplementedError):
        cb.paste_faces_to_input_image(helper(input_img=np.zeros((8, 8, 4), np.uint8)))
    with pytest.raises(NotImplementedError):
        cb.paste_faces_to_input_image(helper(input_img=img.astype(np.uint16)))
