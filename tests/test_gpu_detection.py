"""gpu: RetinaFace-ResNet50 on the conv engine against the CPU oracle (oracle/retinaface_oracle.py, pinned to the reference by
tests/test_oracle_detection.py), plus the new conv forms against torch CPU fp32."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import codeformer_b200 as cb
from codeformer_b200 import _lib, detection as D
from oracle import retinaface_oracle as RO

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = 'cuda:0'


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _bar(out, ref):
    err = float((out.cpu() - ref).abs().max())
    assert err <= 6e-5 * float(ref.abs().max()), err
    return err


@pytest.mark.parametrize('h,w,cin,cout,k,stride,res', [(37, 50, 64, 128, 1, 1, True), (21, 27, 256, 64, 1, 1, True),
                                                        (37, 50, 64, 64, 3, 2, False), (11, 14, 128, 256, 3, 2, False),
                                                        (37, 51, 128, 256, 1, 2, False)])
def test_pertap_conv_forms(h, w, cin, cout, k, stride, res):
    lib = _lib.load()
    g = torch.Generator().manual_seed(h * w + cin)
    x = torch.randn(2, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = 0.1 * torch.randn(cout, generator=g)
    ref = F.conv2d(x, wt, b, stride, k // 2)
    r = torch.randn(ref.shape, generator=g) if res else None
    if res:
        ref = ref + r
    ref = F.relu(ref)
    ho, wo = ref.shape[2], ref.shape[3]
    xd = x.permute(0, 2, 3, 1).contiguous().to(DEV)
    out = torch.empty((2, ho, wo, cout), device=DEV)
    rd = r.permute(0, 2, 3, 1).contiguous().to(DEV) if res else None
    need = lib.cfb_conv2d_pertap_workspace_bytes(2, h, w, cin, cout, k, stride)
    ws = torch.empty(int(need), dtype=torch.uint8, device=DEV)
    wd, bd = wt.to(DEV), b.to(DEV)          # kept alive until the stream has run the conv
    _lib.check(lib.cfb_conv2d_pertap_nhwc(_lib.ptr(xd), _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(out), 2, h, w, cin, cout,
                                          k, stride, 3, _lib.ptr(rd), _lib.ptr(ws), ws.numel(), _stream()), 'pertap')
    torch.cuda.synchronize()
    print('pertap', h, w, k, stride, _bar(out.permute(0, 3, 1, 2), ref))


def test_gen_conv_relu_into_a_slice():
    lib = _lib.load()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 64, 21, 27, generator=g)
    wt = torch.randn(64, 64, 3, 3, generator=g) / 24.
    b = 0.1 * torch.randn(64, generator=g)
    ref = F.relu(F.conv2d(x, wt, b, 1, 1))
    out = torch.zeros((1, 21, 27, 256), device=DEV)
    ws = torch.empty(int(lib.cfb_conv2d_gen_workspace_bytes(64, 64)), dtype=torch.uint8, device=DEV)
    xd, wd, bd = x.permute(0, 2, 3, 1).contiguous().to(DEV), wt.to(DEV), b.to(DEV)
    _lib.check(lib.cfb_conv2d_gen_nhwc(_lib.ptr(xd), 64, _lib.ptr(wd), _lib.ptr(bd),
                                       _lib.ptr(out), 256, 192, 1, 21, 27, 64, 64, 0, 0, 0, 3, None, 0, None, 0, 1.0,
                                       _lib.ptr(ws), ws.numel(), _stream()), 'gen')
    torch.cuda.synchronize()
    _bar(out[..., 192:].permute(0, 3, 1, 2), ref)
    assert float(out[..., :192].abs().max()) == 0.0


def _net(seed=1):
    sd = D.random_retinaface_state_dict(seed)
    net = cb.RetinaFace().to(DEV)
    net.load_state_dict(sd, strict=True)
    return sd, net


def _image(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize('h,w', [(333, 427), (640, 853), (37, 50)])
def test_forward_vs_oracle(h, w):
    sd, net = _net()
    img = _image(h, w, 0)
    x = RO.input_from_u8(img)
    ref = RO.forward(sd, x)
    out = net(x.to(DEV))
    out_u8 = net.forward_u8(torch.from_numpy(img).to(DEV).unsqueeze(0))
    torch.cuda.synchronize()
    errs = [float((o.cpu() - r).abs().max()) for o, r in zip(out, ref)]
    print(f'{h}x{w} loc {errs[0]:.2e} conf {errs[1]:.2e} landms {errs[2]:.2e}')
    assert errs[0] <= 2e-4 and errs[1] <= 1e-4 and errs[2] <= 2e-4
    for a, b in zip(out, out_u8):
        assert torch.equal(a, b), 'the fused uint8 input path equals the fp32 one'


@pytest.mark.parametrize('h,w', [(333, 427), (640, 853)])
def test_detect_faces_vs_oracle(h, w):
    sd, net = _net()
    img = _image(h, w, 0)
    ref = RO.detect_faces(sd, img)
    out = net.detect_faces(img)
    print(f'{h}x{w}: {ref.shape[0]} detections')
    assert out.dtype == np.float32 and out.shape == ref.shape
    assert np.abs(out[:, 4] - ref[:, 4]).max(initial=0) <= 1e-4
    assert np.abs(out[:, :4] - ref[:, :4]).max(initial=0) <= 0.05
    assert np.abs(out[:, 5:] - ref[:, 5:]).max(initial=0) <= 0.05
    again = net.detect_faces(torch.from_numpy(img).to(DEV))
    assert np.array_equal(out, again), 'repeated runs (and numpy / CUDA input) are bit-identical'


def test_batch_equals_single_images():
    _, net = _net()
    imgs = torch.from_numpy(np.stack([_image(96, 130, 1), _image(96, 130, 2)])).to(DEV)
    both = net.forward_u8(imgs)
    for i in range(2):
        one = net.forward_u8(imgs[i:i + 1])
        for a, b in zip(both, one):
            assert torch.equal(a[i:i + 1], b)


def test_errors():
    _, net = _net()
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 64, 64))
    with pytest.raises(NotImplementedError):
        cb.RetinaFace('mobile0.25')
    with pytest.raises(NotImplementedError):
        cb.RetinaFace(half=True)
    with pytest.raises(NotImplementedError):
        net.detect_faces(_image(64, 64, 0), use_origin_size=False)
    with pytest.raises(NotImplementedError):
        net.detect_faces(np.zeros((64, 64, 4), np.uint8))
    with pytest.raises(NotImplementedError):
        net.detect_faces(np.zeros((64, 64, 3), np.float32))
    with pytest.raises(NotImplementedError):
        cb.init_detection_model('retinaface_mobile0.25', device=DEV)
    x = torch.full((1, 3, 64, 64), float('nan'), device=DEV)
    loc, conf, landms = net(x)
    torch.cuda.synchronize()
    cand = net.candidates(loc, torch.full_like(conf, float('nan')), landms, 64, 64)
    assert cand[0].shape[0] == 0
    cb.check_async_status()
