"""gpu: YOLOv5l-face on the conv engine against the CPU oracle (oracle/yolov5face_oracle.py, pinned to the reference by
tests/test_oracle_yolov5face.py), plus the new conv forms (SiLU epilogues, destination slices) against torch CPU fp32."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import codeformer_b200 as cb
from codeformer_b200 import _lib, yolov5face as Y
from oracle import yolov5face_oracle as YO

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = 'cuda:0'
OUT_SILU = 4
MIN_FACE = 2          # the random network's best-scoring boxes are small: keep those of 2 px and more


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _bar(out, ref):
    err = float((out.cpu() - ref).abs().max())
    assert err <= 6e-5 * float(ref.abs().max()), err
    return err


# per-tap engine: 1x1 and 3x3 stride 2 with SiLU into a channel slice of a wider buffer; the 32- and 48-channel convs of the
# network are zero-padded to 64 (real channels first, zero weights and bias after)
@pytest.mark.parametrize('h,w,cin,cout,real_in,real_out,k,stride,pitch,c0', [
    (40, 56, 64, 64, 64, 64, 1, 1, 128, 64),        # C3 cv2 into the second half of the concat
    (21, 27, 128, 128, 128, 128, 1, 1, 256, 0),     # ragged tiles, first half
    (40, 56, 64, 64, 64, 32, 1, 1, 64, 0),          # stem_2a: 64 -> 32 (padded to 64)
    (40, 56, 64, 64, 32, 64, 3, 2, 128, 0),         # stem_2b: 32 (padded to 64) -> 64, stride 2, into the stem concat
    (22, 28, 256, 256, 256, 256, 3, 2, 512, 0),     # head conv 17 into the layer-18 concat
    (12, 14, 256, 64, 256, 48, 1, 1, 64, 0),        # Detect: 256 -> 48 (padded to 64), no activation
])
def test_pertap_silu_into_a_slice(h, w, cin, cout, real_in, real_out, k, stride, pitch, c0):
    lib = _lib.load()
    g = torch.Generator().manual_seed(h * w + cin + k)
    x = torch.randn(2, cin, h, w, generator=g)
    x[:, real_in:] = 0
    wt = torch.zeros(cout, cin, k, k)
    wt[:real_out, :real_in] = torch.randn(real_out, real_in, k, k, generator=g) / (real_in * k * k) ** 0.5
    b = torch.zeros(cout)
    b[:real_out] = 0.1 * torch.randn(real_out, generator=g)
    act = 0 if real_out == 48 else OUT_SILU
    ref = F.conv2d(x, wt, b, stride, k // 2)
    if act:
        ref = F.silu(ref)
    ho, wo = ref.shape[2], ref.shape[3]
    xd = x.permute(0, 2, 3, 1).contiguous().to(DEV)
    out = torch.full((2, ho, wo, pitch), 7.0, device=DEV)
    need = lib.cfb_conv2d_pertap_workspace_bytes(2, h, w, cin, cout, k, stride)
    ws = torch.empty(int(need), dtype=torch.uint8, device=DEV)
    wd, bd = wt.to(DEV), b.to(DEV)
    _lib.check(lib.cfb_conv2d_pertap_slice_nhwc(_lib.ptr(xd), _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(out), 2, h, w, cin, cout, k,
                                                stride, act, pitch, c0, _lib.ptr(ws), ws.numel(), _stream()), 'pertap slice')
    torch.cuda.synchronize()
    o = out.cpu()
    print('pertap', h, w, k, stride, _bar(o[..., c0:c0 + cout].permute(0, 3, 1, 2), ref))
    assert bool((o[..., c0 + real_out:c0 + cout] == 0).all()), 'padded channels stay zero'
    rest = torch.cat((o[..., :c0], o[..., c0 + cout:]), -1)
    assert bool((rest == 7.0).all()), 'channels outside the slice are untouched'


def test_gen_silu_with_a_post_activation_residual():
    """Bottleneck: out = x + silu(conv3x3(t) + b), written into the first half of a 256-channel concat buffer."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(11)
    t = torch.randn(1, 128, 21, 27, generator=g)
    xres = torch.randn(1, 128, 21, 27, generator=g)
    wt = torch.randn(128, 128, 3, 3, generator=g) / (128 * 9) ** 0.5
    b = 0.1 * torch.randn(128, generator=g)
    ref = xres + F.silu(F.conv2d(t, wt, b, 1, 1))
    out = torch.zeros((1, 21, 27, 256), device=DEV)
    ws = torch.empty(int(lib.cfb_conv2d_gen_workspace_bytes(128, 128)), dtype=torch.uint8, device=DEV)
    td, wd, bd = t.permute(0, 2, 3, 1).contiguous().to(DEV), wt.to(DEV), b.to(DEV)
    rd = xres.permute(0, 2, 3, 1).contiguous().to(DEV)
    _lib.check(lib.cfb_conv2d_gen_nhwc(_lib.ptr(td), 128, _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(out), 256, 0, 1, 21, 27, 128, 128, 0,
                                       0, 0, OUT_SILU, None, 0, _lib.ptr(rd), 128, 1.0, _lib.ptr(ws), ws.numel(), _stream()), 'gen')
    torch.cuda.synchronize()
    _bar(out[..., :128].permute(0, 3, 1, 2), ref)
    assert float(out[..., 128:].abs().max()) == 0.0


def _net(seed=1):
    sd = Y.random_yolov5l_state_dict(seed)
    net = cb.YOLOv5lFace().to(DEV)
    net.load_state_dict(sd, strict=True)
    return sd, net


def _image(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize('h,w', [(672, 864), (352, 480), (64, 96)])
def test_forward_vs_oracle(h, w):
    sd, net = _net()
    img = _image(h, w, 0)
    x = torch.from_numpy(np.ascontiguousarray(img[..., ::-1].transpose(2, 0, 1))).unsqueeze(0).float() / 255.0   # RGB / 255
    ref_pred, ref_raw = YO.forward(sd, x)
    pred, raw = net(x.to(DEV))
    torch.cuda.synchronize()
    e_raw = max(float((a.cpu() - b).abs().max()) for a, b in zip(raw, ref_raw))
    d = (pred.cpu() - ref_pred).abs()
    e_score = float(d[..., [4, 15]].max())
    e_xy = float(torch.cat((d[..., 0:4], d[..., 5:15]), -1).max())
    print(f'{h}x{w} raw {e_raw:.2e} scores {e_score:.2e} coordinates {e_xy:.2e} px')
    assert e_raw <= 2e-4 and e_score <= 1e-4 and e_xy <= 5e-3
    assert all(tuple(r.shape) == (1, 3, h // s, w // s, 16) for r, s in zip(raw, Y.STRIDES))
    p8, r8 = net.forward_u8(torch.from_numpy(img).to(DEV).unsqueeze(0))
    assert torch.equal(pred, p8) and all(torch.equal(a, b) for a, b in zip(raw, r8)), 'uint8 input equals the fp32 one'


def test_letterboxed_u8_equals_the_fp32_canvas():
    _, net = _net()
    img = _image(333, 427, 3)
    _, second, (H, W), (top, left) = Y.letterbox_geometry(333, 427)
    x = YO.preprocess([img])
    assert tuple(x.shape[2:]) == (H, W)
    small = torch.from_numpy(img).to(DEV).unsqueeze(0)
    resized = Y._resize_u8(small, *second)
    a, _ = net(x.to(DEV))
    b, _ = net.forward_u8(resized, (H, W), (top, left), raw=False)
    assert torch.equal(a, b)


def test_batch_equals_single_images():
    _, net = _net()
    imgs = torch.from_numpy(np.stack([_image(96, 128, 1), _image(96, 128, 2)])).to(DEV)
    both, braw = net.forward_u8(imgs)
    for i in range(2):
        one, oraw = net.forward_u8(imgs[i:i + 1])
        assert torch.equal(both[i:i + 1], one)
        assert all(torch.equal(a[i:i + 1], b) for a, b in zip(braw, oraw))


def _reference(sd, imgs, target_size=None):
    """The oracle's detect_faces at the confidence threshold closest to 0.7 that no objectness and no obj * cls lies within
    1e-3 of (the midpoint of a gap of those scores) and that leaves at least one face, so that the GPU / oracle comparison
    means something: (thr, result)."""
    x = YO.preprocess(imgs, target_size)
    pred, _ = YO.forward(sd, x)
    scores = torch.cat((pred[..., 4].flatten(), (pred[..., 4] * pred[..., 15]).flatten())).double().sort().values
    gaps = (scores[1:] - scores[:-1]) >= 2e-3
    mids = ((scores[1:] + scores[:-1]) / 2)[gaps]
    for thr in sorted((float(t) for t in mids if 0.5 <= t <= 0.95), key=lambda t: abs(t - 0.7)):
        res = Y.finish_detections(YO.candidates(pred, thr), tuple(x.shape[2:]), [im.shape for im in imgs], thr, 0.5, MIN_FACE)
        if res is not None:
            return thr, res
    raise AssertionError('no threshold with a 1e-3 margin')


@pytest.mark.parametrize('h,w', [(640, 853), (333, 427)])
def test_detect_faces_vs_oracle(h, w):
    sd, net = _net()
    img = _image(h, w, 0)
    thr, ref = _reference(sd, [img])
    assert np.array_equal(ref, YO.detect_faces(sd, img, conf_thres=thr, min_face=MIN_FACE))
    det = cb.YoloDetector('facelib/detection/yolov5face/models/yolov5l.yaml', min_face=MIN_FACE, device=DEV)
    det.detector = net
    out = det.detect_faces(img, conf_thres=thr)
    print(f'{h}x{w}: threshold {thr}, {0 if ref is None else ref.shape[0]} detections')
    assert ref is not None and out is not None
    assert out.dtype == np.int64 and out.shape == ref.shape
    assert np.abs(out - ref).max() <= 1
    again = det.detect_faces([torch.from_numpy(img).to(DEV)], conf_thres=thr)
    assert np.array_equal(out, again), 'repeated runs (and numpy / CUDA input) are bit-identical'


def test_target_size_and_a_list_of_images():
    sd, net = _net()
    imgs = [_image(600, 801, 4), _image(600, 801, 5)]
    det = cb.YoloDetector('yolov5l.yaml', min_face=MIN_FACE, target_size=480, device=DEV)
    det.detector = net
    thr, ref = _reference(sd, imgs, 480)
    out = det.detect_faces(imgs, conf_thres=thr)
    assert out is not None and out.shape == ref.shape and np.abs(out - ref).max() <= 1


def test_errors():
    _, net = _net()
    with pytest.raises(NotImplementedError):
        cb.init_detection_model('YOLOv5n', device=DEV)
    with pytest.raises(NotImplementedError):
        cb.YoloDetector('facelib/detection/yolov5face/models/yolov5n.yaml')
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 64, 64))
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 64, 80, device=DEV))
    det = cb.YoloDetector('yolov5l.yaml', device=DEV)
    det.detector = net
    with pytest.raises(NotImplementedError):
        det.detect_faces(np.zeros((64, 64, 4), np.uint8))
    with pytest.raises(NotImplementedError):
        det.detect_faces(np.zeros((64, 64, 3), np.float32))
    x = torch.full((1, 3, 64, 64), float('nan'), device=DEV)
    pred, _ = net(x)
    torch.cuda.synchronize()
    assert net.candidates(pred, 64, 64)[0].shape[0] == 0
    assert net.candidates(torch.full_like(pred, float('nan')), 64, 64)[0].shape[0] == 0
    cb.check_async_status()
