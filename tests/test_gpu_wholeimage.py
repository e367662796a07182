"""gpu: whole-image mode over batches (codeformer_b200.wholeimage.restore_images) and the kernels under it: INTER_AREA
against cv2, the cross-image crop warp and paste-back against their per-image counterparts, and restore_images against a
literal per-image run of the reference loop body with host cv2.resize and the package's existing drop-ins."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import pasteback as PB
from oracle import pasteback_oracle as O
from tests.test_oracle_resize_area import CASES, case_id

cv2 = pytest.importorskip('cv2')
pytestmark = pytest.mark.gpu
DEV = 'cuda'
WHOLE = os.path.join(os.path.dirname(__file__), 'golden', 'whole_imgs')


def _rand(h, w, seed, n=None):
    return np.random.default_rng(seed).integers(0, 256, ((n,) if n else ()) + (h, w, 3), dtype=np.uint8)


# ---- kernels ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', CASES, ids=case_id)
def test_resize_area_bit_exact(case):
    h, w, oh, ow = case
    imgs = _rand(h, w, h + w, n=3)
    out = cb.resize_area(torch.from_numpy(imgs).to(DEV), (ow, oh)).cpu().numpy()
    for i in range(3):
        assert np.array_equal(out[i], cv2.resize(imgs[i], (ow, oh), interpolation=cv2.INTER_AREA)), f'image {i}'
    one = cb.resize_area(torch.from_numpy(imgs[1]).to(DEV), (ow, oh)).cpu().numpy()
    assert np.array_equal(one, out[1])


def test_resize_linear_factor_bit_exact():
    """read_image's enlargement: cv2.resize(img, (0, 0), fx=f, fy=f, INTER_LINEAR), taps from f itself."""
    for h, w in [(310, 491), (189, 248), (225, 225), (123, 77), (511, 700)]:
        f = 512.0 / min(h, w)
        imgs = _rand(h, w, h, n=2)
        out = PB.resize_linear_factor(torch.from_numpy(imgs).to(DEV), f).cpu().numpy()
        for i in range(2):
            assert np.array_equal(out[i], cv2.resize(imgs[i], (0, 0), fx=f, fy=f, interpolation=cv2.INTER_LINEAR))


def _affines(rng, n, h, w):
    out = []
    for _ in range(n):
        a, s = rng.uniform(-0.3, 0.3), rng.uniform(1.5, 4.0)     # image -> 512 crop: faces of 128..340 pixels
        c, si = np.cos(a) * s, np.sin(a) * s
        cx, cy = rng.uniform(0, w), rng.uniform(0, h)
        M = np.array([[c, -si, 0.], [si, c, 0.]])
        M[:, 2] = np.array([256., 256.]) - M[:, :2] @ np.array([cx, cy])
        out.append(M)
    return out


@pytest.mark.parametrize('mode', ['constant', 'reflect101'])
def test_warp_multi_equals_per_image(mode):
    rng = np.random.default_rng(5)
    imgs = torch.from_numpy(np.stack([O.synthetic_background(300, 420, s) for s in range(3)])).to(DEV)
    counts = [2, 0, 3]
    owner = [k for k, c in enumerate(counts) for _ in range(c)]
    aff = _affines(rng, len(owner), 300, 420)
    multi = PB.warp_faces_multi(imgs, aff, owner, 512, mode)
    for k in range(3):
        sel = [i for i, o in enumerate(owner) if o == k]
        if sel:
            assert torch.equal(multi[sel], cb.warp_faces(imgs[k], [aff[i] for i in sel], 512, mode))
    assert PB.warp_faces_multi(imgs, [], [], 512).shape == (0, 512, 512, 3)


@pytest.mark.parametrize('upscale,use_parse', [(1, False), (2, False), (2, True), (1, True)])
def test_paste_multi_equals_per_image(upscale, use_parse):
    rng = np.random.default_rng(upscale * 2 + use_parse)
    h, w = 280, 360
    imgs = torch.from_numpy(np.stack([O.synthetic_background(h, w, s) for s in range(4)])).to(DEV)
    counts = [1, 0, 3, 2]                      # image 1 has no face
    owner = [k for k, c in enumerate(counts) for _ in range(c)]
    aff = _affines(rng, len(owner), h, w)
    inv = [cv2.invertAffineTransform(a) * upscale for a in aff]
    faces = torch.from_numpy(_rand(512, 512, 9, n=len(owner))).to(DEV)
    masks = None
    if use_parse:
        masks = torch.from_numpy((rng.random((len(owner), 512, 512)) < 0.7).astype(np.uint8) * 255).to(DEV)
    multi = cb.paste_faces_multi(imgs, faces, inv, owner, upscale, masks=masks)
    assert multi.shape == (4, h * upscale, w * upscale, 3)
    for k in range(4):
        sel = [i for i, o in enumerate(owner) if o == k]
        one = cb.paste_faces(imgs[k], faces[sel], [inv[i] for i in sel], upscale,
                             masks=None if masks is None else masks[sel] if sel else None)
        assert torch.equal(multi[k], one), f'image {k}'
    # chunking the images differently does not change any byte
    a = cb.paste_faces_multi(imgs[:2], faces[:1], inv[:1], [0], upscale, masks=None if masks is None else masks[:1])
    assert torch.equal(a, multi[:2])


# ---- end to end ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def nets():
    from codeformer_b200 import spec as S
    from codeformer_b200.detection import random_retinaface_state_dict
    from codeformer_b200.parsing import parsenet_spec, random_parsenet_state_dict
    net = cb.ARCH_REGISTRY.get('CodeFormer')(dim_embd=512, codebook_size=1024, n_head=8, n_layers=9,
                                             connect_list=['32', '64', '128', '256']).to(DEV)
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    det = cb.RetinaFace().to(DEV)
    det.load_state_dict(random_retinaface_state_dict(1, class_gain=8.0, class_bias=2.0), strict=True)
    parser = cb.init_parsing_model(device='cpu')
    parser.load_state_dict(random_parsenet_state_dict(parsenet_spec(512, 512, 32, 64, 19, 10, (32, 256)), 41), strict=False)
    return SimpleNamespace(net=net.eval(), det=det.eval(), parser=parser.to(DEV).eval())


def whole_images():
    """The reference's small inputs (all enlarged by read_image), one of them twice (mirrored) so that a size group has
    two images, and two synthetic frames that the detector's resize shrinks with INTER_AREA."""
    imgs = [cv2.imread(os.path.join(WHOLE, f'{n}.jpg'), cv2.IMREAD_COLOR) for n in ('00', '01', '03', '04', '05')]
    imgs.insert(2, np.ascontiguousarray(imgs[1][:, ::-1]))
    imgs += [O.synthetic_background(720, 960, 3), O.synthetic_background(720, 960, 4)]
    return imgs


def reference_loop(img, net, det, parser, w=0.5, upscale=2, only_center_face=False, bg_upsampler=None):
    """inference_codeformer.py:178-229 for one image with FaceRestoreHelper(upscale, face_size=512, crop_ratio=(1, 1),
    use_parse=parser is not None): host cv2.resize for read_image and get_face_landmarks_5(resize=640), the package's
    detect_faces / align_warp_face / restore_faces / paste_faces_to_input_image."""
    from codeformer_b200.wholeimage import FACE_TEMPLATE, get_center_face, is_gray
    helper = SimpleNamespace(upscale_factor=upscale, face_size=(512, 512), face_template=FACE_TEMPLATE, pad_blur=False,
                             all_landmarks_5=[], det_faces=[], affine_matrices=[], cropped_faces=[], restored_faces=[],
                             inverse_affine_matrices=[], use_parse=parser is not None, face_parse=parser)
    # read_image
    helper.input_img = img
    assert not is_gray(img)
    if min(img.shape[:2]) < 512:
        f = 512.0 / min(img.shape[:2])
        helper.input_img = cv2.resize(img, (0, 0), fx=f, fy=f, interpolation=cv2.INTER_LINEAR)
    # get_face_landmarks_5(only_center_face, resize=640, eye_dist_threshold=5)
    h, w_ = helper.input_img.shape[0:2]
    scale = 640 / min(h, w_)
    h, w_ = int(h * scale), int(w_ * scale)
    interp = cv2.INTER_AREA if scale < 1 else cv2.INTER_LINEAR
    input_img = cv2.resize(helper.input_img, (w_, h), interpolation=interp)
    with torch.no_grad():
        bboxes = det.detect_faces(input_img)
    if bboxes is not None and bboxes.shape[0] > 0:
        bboxes = bboxes / scale
        for bbox in bboxes:
            eye_dist = np.linalg.norm([bbox[6] - bbox[8], bbox[7] - bbox[9]])
            if eye_dist < 5:
                continue
            helper.all_landmarks_5.append(np.array([[bbox[i], bbox[i + 1]] for i in range(5, 15, 2)]))
            helper.det_faces.append(bbox[0:5])
        if helper.det_faces and only_center_face:
            hh, ww, _ = helper.input_img.shape
            helper.det_faces, idx = get_center_face(helper.det_faces, hh, ww)
            helper.all_landmarks_5 = [helper.all_landmarks_5[idx]]
    PB.align_warp_face(helper)
    with torch.no_grad():
        helper.restored_faces = net.restore_faces(helper.cropped_faces, w=w, adain=True) if helper.cropped_faces else []
    bg_img = bg_upsampler.enhance(img, outscale=upscale)[0] if bg_upsampler is not None else None
    for a in helper.affine_matrices:
        inv = cv2.invertAffineTransform(a)
        inv *= upscale
        helper.inverse_affine_matrices.append(inv)
    return PB.paste_faces_to_input_image(helper, upsample_img=bg_img), len(helper.cropped_faces)


def test_restore_images_equals_reference_loop(nets):
    imgs = whole_images()
    refs = [reference_loop(im, nets.net, nets.det, nets.parser) for im in imgs]
    counts = [n for _, n in refs]
    print('faces per image', counts)
    assert sum(counts) >= 3
    outs = {}
    for mb in (1, 4, 32):
        res, crops, faces = cb.restore_images(imgs, nets.net, nets.det, parser=nets.parser, max_batch=mb, return_faces=True)
        for i, ((ref, n), out) in enumerate(zip(refs, res)):
            assert isinstance(out, np.ndarray) and out.shape == ref.shape
            assert np.array_equal(out, ref), f'image {i} (max_batch {mb}): {int((out != ref).sum())} bytes differ'
            assert crops[i].shape[0] == n and faces[i].shape[0] == n
        outs[mb] = faces
    for a, b in zip(outs[1], outs[32]):
        assert np.array_equal(a, b)
    # CUDA inputs give CUDA outputs with the same bytes
    dev_out = cb.restore_images([torch.from_numpy(im).to(DEV) for im in imgs[-2:]], nets.net, nets.det, parser=nets.parser)
    for (ref, _), out in zip(refs[-2:], dev_out):
        assert out.is_cuda and np.array_equal(out.cpu().numpy(), ref)
    cb.check_async_status()


def test_only_center_face_upscale1(nets):
    imgs = whole_images()[4:]
    refs = [reference_loop(im, nets.net, nets.det, None, upscale=1, only_center_face=True)[0] for im in imgs]
    res = cb.restore_images(imgs, nets.net, nets.det, upscale=1, only_center_face=True, max_batch=4)
    for i, (ref, out) in enumerate(zip(refs, res)):
        assert np.array_equal(out, ref), f'image {i}'


def test_yolov5l_detector(nets):
    from codeformer_b200.yolov5face import random_yolov5l_state_dict
    det = cb.init_detection_model('YOLOv5l', device=DEV)
    det.detector.load_state_dict(random_yolov5l_state_dict(2, obj_bias=(1.25, -4.0, -4.0)), strict=True)
    imgs = whole_images()[-2:]          # 0 and 3 faces with these weights
    refs = [reference_loop(im, nets.net, det, nets.parser) for im in imgs]
    assert sum(n for _, n in refs) > 0
    res = cb.restore_images(imgs, nets.net, det, parser=nets.parser, max_batch=4)
    for i, ((ref, _), out) in enumerate(zip(refs, res)):
        assert np.array_equal(out, ref), f'image {i}'


def test_background_upsampler(nets):
    from codeformer_b200 import spec as S
    rrdb = cb.RRDBNet(3, 3, scale=2, num_block=1)
    rrdb.load_state_dict(S.random_state_dict(S.rrdbnet_spec(3, 3, 2, 64, 1, 32), 11))
    bg = cb.RealESRGANer(scale=2, model=rrdb, tile=0, pre_pad=0, device=DEV)
    img = O.synthetic_background(512, 600, 7)
    ref, _ = reference_loop(img, nets.net, nets.det, nets.parser, bg_upsampler=bg)
    out = cb.restore_images([img], nets.net, nets.det, parser=nets.parser, bg_upsampler=bg)[0]
    assert np.array_equal(out, ref)


def test_errors_and_fallback(nets):
    img = whole_images()[-1]
    with pytest.raises(RuntimeError):
        cb.restore_images([torch.from_numpy(img)], nets.net, nets.det)
    with pytest.raises(NotImplementedError):
        cb.restore_images([img.astype(np.uint16)], nets.net, nets.det)
    with pytest.raises(NotImplementedError):
        cb.restore_images([np.zeros((600, 600, 4), np.uint8)], nets.net, nets.det)
    with pytest.raises(NotImplementedError):
        cb.restore_images([img[:, :, 0]], nets.net, nets.det)
    with pytest.raises(RuntimeError):
        cb.resize_area(torch.from_numpy(img), (10, 10))
    with pytest.raises(NotImplementedError):
        cb.resize_area(torch.from_numpy(img).to(DEV), (2000, 10))
    # a CodeFormer failure gives the input faces back, as the reference's per-face fallback does
    orig = nets.net.forward_u8

    def boom(*a, **k):
        raise RuntimeError('injected failure')
    nets.net.forward_u8 = boom
    try:
        out, crops, faces = cb.restore_images([img], nets.net, nets.det, max_batch=2, return_faces=True)
    finally:
        nets.net.forward_u8 = orig
    assert crops[0].shape[0] > 0 and np.array_equal(crops[0], faces[0])
    assert cb.restore_images.last_errors and 'injected failure' in cb.restore_images.last_errors[0][1]
    torch.cuda.synchronize()
    cb.check_async_status()
    # the unbuilt detectors and options still raise
    with pytest.raises(NotImplementedError):
        cb.RetinaFace(network_name='mobile0.25')
    with pytest.raises(NotImplementedError):
        cb.RetinaFace(half=True)
