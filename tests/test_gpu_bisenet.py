"""-m gpu: BiSeNet on the conv engine (``BiSeNet.forward`` / ``masks_u8``, ``cfb_bisenet_*``) against the torch CPU oracle
(oracle/bisenet_oracle.py, bit-identical to the reference class), its SIMT kernels against torch, batch invariance, the
fused masks against the unfused chain, and the callers (parse_masks, paste_faces_to_input_image, restore_images) against a
wrapper parser that takes the generic path."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import codeformer_b200 as cb
from codeformer_b200 import _lib
from codeformer_b200 import pasteback as PB
from oracle import bisenet_oracle as BO
from oracle import pasteback_oracle as O
from tests.test_gpu_wholeimage import _affines, nets, whole_images   # noqa: F401  (nets: fixture)
from tests.util import golden

cv2 = pytest.importorskip('cv2')
pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
torch.set_num_threads(16)
DEV = 'cuda'
REL_BOUND = 1e-4          # max-abs error of each output <= REL_BOUND * max |logit| of the oracle


def _net(sd=None):
    net = cb.BiSeNet(num_class=19)
    net.load_state_dict(sd if sd is not None else BO.random_bisenet_state_dict(1), strict=True)
    return net.eval().to(DEV)


@pytest.fixture(scope='module')
def bise():
    sd = BO.random_bisenet_state_dict(1)
    return SimpleNamespace(sd=sd, net=_net(sd))


def _faces(n, hw=(512, 512)):
    """n uint8 BGR faces from the committed RGB fixtures: the four faces, then rolled and mirrored copies; cropped to hw."""
    f = golden('faces.npz')['faces'][..., ::-1]
    out = [np.roll(f[i % 4], 37 * (i // 4), axis=1)[:, ::(-1 if (i // 4) % 2 else 1)][:hw[0], :hw[1]] for i in range(n)]
    return torch.from_numpy(np.ascontiguousarray(np.stack(out))).to(DEV)


def _input(faces):
    """cfb_u8_to_input of uint8 BGR faces [N,H,W,3]: what parse_masks feeds the network."""
    N, H, W, _ = faces.shape
    x = torch.empty((N, 3, H, W), dtype=torch.float32, device=DEV)
    _lib.check(_lib.load().cfb_u8_to_input(_lib.ptr(faces.contiguous()), _lib.ptr(x), N, H * W,
                                           ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'cfb_u8_to_input')
    return x


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---- forward against the oracle ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('batch,hw', [(1, (512, 512)), (3, (512, 512)), (2, (96, 160))])
def test_forward_vs_oracle(bise, batch, hw):
    x = _input(_faces(batch, hw))
    outs = bise.net(x)
    torch.cuda.synchronize()
    cb.check_async_status()
    ref = BO.forward(bise.sd, x.cpu())
    for name, a, r in zip(('out', 'out16', 'out32'), outs, ref):
        assert a.shape == r.shape == (batch, 19) + hw
        err, top = float((a.cpu() - r).abs().max()), float(r.abs().max())
        print(f'bisenet {name} B={batch} {hw}: max-abs {err:.3e} (|logit|max {top:.3f}, ratio {err / top:.2e})')
        assert err <= REL_BOUND * top, name
    if batch == 3:
        margin = ref[0].topk(2, dim=1).values
        sure = (margin[:, 0] - margin[:, 1]) > 2 * REL_BOUND * float(ref[0].abs().max())
        cls = cb.face_parse_mask(outs[0])[0].cpu().long()
        print(f'bisenet classes: {float((cls != ref[0].argmax(1)).float().mean()) * 100:.4f} % differ from the oracle, '
              f'{float(sure.float().mean()) * 100:.2f} % of pixels have a margin above the bound')
        assert torch.equal(cls[sure], ref[0].argmax(1)[sure])


def test_batch_invariance(bise):
    x = _input(_faces(3))
    outs = bise.net(x)
    cls, mask = bise.net.masks_u8(_faces(3))
    for k in range(3):
        one = bise.net(x[k:k + 1])
        for a, b in zip(outs, one):
            assert torch.equal(a[k], b[0]), f'face {k}'
        c1, m1 = bise.net.masks_u8(_faces(3)[k:k + 1])
        assert torch.equal(c1[0], cls[k]) and torch.equal(m1[0], mask[k])
    again = bise.net(x)
    assert all(torch.equal(a, b) for a, b in zip(outs, again)), 'deterministic'


# ---- the SIMT kernels against torch ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('hw,out', [((16, 16), (512, 512)), ((64, 64), (512, 512)), ((3, 5), (96, 160))])
def test_bilinear_vs_torch(hw, out):
    g = torch.Generator().manual_seed(hw[0])
    x = torch.randn(2, 19, *hw, generator=g)
    ref = F.interpolate(x, out, mode='bilinear', align_corners=True)
    src = torch.zeros(2, hw[0], hw[1], 64)
    src[..., :19] = x.permute(0, 2, 3, 1)
    src = src.to(DEV)
    y = torch.empty((2, 19) + out, device=DEV)
    _lib.check(_lib.load().cfb_debug_bisenet_bilinear(_lib.ptr(src), 64, 2, hw[0], hw[1], 19, _lib.ptr(y), out[0], out[1], _stream()),
               'cfb_debug_bisenet_bilinear')
    err = float((y.cpu() - ref).abs().max())
    print(f'bilinear {hw} -> {out}: max-abs {err:.3e}, bit-equal {torch.equal(y.cpu(), ref)}')
    assert err <= 1e-6 * float(ref.abs().max())


def _fold(sd, w, bn):
    s = sd[bn + '.weight'] / torch.sqrt(sd[bn + '.running_var'] + 1e-5)
    return (w.flatten(1) * s[:, None]).contiguous(), (sd[bn + '.bias'] - sd[bn + '.running_mean'] * s).contiguous()


def _attention(feat, w1, b1, act1, w2=None, b2=None, act2=0):
    N, C, H, W = feat.shape
    f = feat.permute(0, 2, 3, 1).contiguous().to(DEV)
    d = lambda t: None if t is None else t.contiguous().to(DEV)   # noqa: E731
    w1, b1, w2, b2 = d(w1), d(b1), d(w2), d(b2)
    c1 = w1.shape[0]
    c2 = w2.shape[0] if w2 is not None else 0
    mean = torch.empty((N, C), device=DEV)
    att = torch.empty((N, c2 or c1), device=DEV)
    _lib.check(_lib.load().cfb_debug_bisenet_attention(_lib.ptr(f), N, H * W, C, _lib.ptr(w1), _lib.ptr(b1), c1, act1, _lib.ptr(w2),
                                                       _lib.ptr(b2), c2, act2, _lib.ptr(mean), _lib.ptr(att), _stream()),
               'cfb_debug_bisenet_attention')
    return mean.cpu(), att.cpu()


def test_arm_and_ffm_attention_vs_torch(bise):
    sd = bise.sd
    g = torch.Generator().manual_seed(3)
    for p, hw in (('cp.arm32', (16, 16)), ('cp.arm16', (32, 32)), ('cp.arm16', (3, 5))):
        feat = torch.relu(torch.randn(3, 128, *hw, generator=g))
        w, b = _fold(sd, sd[p + '.conv_atten.weight'], p + '.bn_atten')
        mean, att = _attention(feat, w, b, 2)
        ref = BO.arm_attention(sd, p, feat).flatten(1)
        assert float((mean - feat.mean((2, 3))).abs().max()) <= 1e-6
        err = float((att - ref).abs().max())
        print(f'{p} attention {hw}: max-abs {err:.3e}')
        assert err <= 1e-6
    feat = torch.relu(torch.randn(3, 256, 64, 64, generator=g))
    _, att = _attention(feat, sd['ffm.conv1.weight'].flatten(1), None, 1, sd['ffm.conv2.weight'].flatten(1), None, 2)
    err = float((att - BO.ffm_attention(sd, feat).flatten(1)).abs().max())
    print(f'ffm attention: max-abs {err:.3e}')
    assert err <= 1e-6
    v = torch.relu(torch.randn(3, 512, 16, 16, generator=g))
    w, b = _fold(sd, sd['cp.conv_avg.conv.weight'], 'cp.conv_avg.bn')
    _, avg = _attention(v, w, b, 1)
    ref = BO._cbr(F.avg_pool2d(v, v.size()[2:]), sd, 'cp.conv_avg', pad=0).flatten(1)
    assert float((avg - ref).abs().max()) <= 1e-5 * float(ref.abs().max())


# ---- masks_u8: byte-equal to the unfused chain ----------------------------------------------------------------------------
@pytest.mark.parametrize('batch', [1, 3, 32])
def test_masks_u8_equals_chain(bise, batch):
    faces = _faces(batch)
    cls, mask = bise.net.masks_u8(faces)
    rc, rm = cb.face_parse_mask(bise.net(_input(faces))[0])
    torch.cuda.synchronize()
    cb.check_async_status()
    assert cls.shape == rc.shape == (batch, 512, 512) and mask.shape == rm.shape
    assert torch.equal(cls, rc), f'classes: {int((cls != rc).sum())} pixels differ'
    assert torch.equal(mask, rm), f'mask: {int((mask != rm).sum())} pixels differ'
    assert len(torch.unique(mask)) == 2 and len(torch.unique(cls)) >= 3


def test_masks_u8_small_faces(bise):
    faces = _faces(2, (96, 160))
    cls, mask = bise.net.masks_u8(faces)
    rc, rm = cb.face_parse_mask(bise.net(_input(faces))[0])
    assert torch.equal(cls, rc) and torch.equal(mask, rm)


# ---- the loader and the callers -------------------------------------------------------------------------------------------
def test_init_parsing_model_loads_strictly(bise, tmp_path):
    path = tmp_path / 'parsing_bisenet.pth'
    torch.save(bise.sd, path)
    net = cb.init_parsing_model('bisenet', model_path=str(path))
    assert isinstance(net, cb.BiSeNet) and not net.training
    assert all(torch.equal(v.cpu(), bise.sd[k]) for k, v in net.state_dict().items())
    faces = _faces(2)
    assert torch.equal(net.masks_u8(faces)[0], bise.net.masks_u8(faces)[0])
    bad = dict(bise.sd)
    bad['module.extra'] = torch.zeros(1)
    torch.save(bad, path)
    with pytest.raises(RuntimeError):
        cb.init_parsing_model('bisenet', model_path=str(path))
    assert isinstance(cb.init_parsing_model(device=DEV), cb.ParseNet), 'the default stays ParseNet'


def test_parse_masks_equals_wrapper(bise):
    parser = bise.net
    faces = _faces(5)
    big = PB.resize_linear(faces, (1024, 1024))
    for f in (faces, big):
        assert torch.equal(PB.parse_masks(f, parser), PB.parse_masks(f, lambda x: parser(x)))


def test_paste_faces_to_input_image_equals_wrapper(bise):
    rng = np.random.default_rng(2)
    img = O.synthetic_background(300, 420, 5)
    aff = _affines(rng, 3, 300, 420)
    faces = list(_faces(3).cpu().numpy())

    def paste(parser):
        helper = SimpleNamespace(input_img=img, upscale_factor=2, face_size=(512, 512), restored_faces=list(faces),
                                 inverse_affine_matrices=[cv2.invertAffineTransform(a) * 2 for a in aff], use_parse=True,
                                 face_parse=parser)
        return PB.paste_faces_to_input_image(helper)
    a, b = paste(bise.net), paste(lambda x: bise.net(x))
    assert a.shape == (600, 840, 3) and np.array_equal(a, b)


def test_restore_images_equals_wrapper(nets, bise):
    base = whole_images()
    imgs = [base[0], cv2.cvtColor(cv2.cvtColor(base[1], cv2.COLOR_BGR2GRAY), cv2.COLOR_GRAY2BGR), base[2], base[-1]]
    a, _, faces = cb.restore_images(imgs, nets.net, nets.det, parser=bise.net, max_batch=4, return_faces=True)
    assert sum(len(f) for f in faces) >= 2
    b = cb.restore_images(imgs, nets.net, nets.det, parser=lambda x: bise.net(x), max_batch=4)
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), f'image {i}: {int((x != y).sum())} bytes differ'


# ---- errors --------------------------------------------------------------------------------------------------------------
def test_errors(bise):
    net = bise.net
    x = _input(_faces(1))
    with pytest.raises(RuntimeError, match='CUDA'):
        net(x.cpu())
    with pytest.raises(RuntimeError, match='float32'):
        net(x.double())
    with pytest.raises(RuntimeError, match='float32'):
        net(x[:, :2])
    for hw in [(500, 512), (512, 520), (16, 16)]:
        with pytest.raises(RuntimeError, match='multiples of 32'):
            net(torch.zeros((1, 3) + hw, device=DEV))
        with pytest.raises(RuntimeError, match='multiples of 32'):
            net.masks_u8(torch.zeros((1,) + hw + (3,), dtype=torch.uint8, device=DEV))
    with pytest.raises(NotImplementedError):
        net(x, return_feat=True)
    good = _faces(1)
    with pytest.raises(RuntimeError, match='CUDA'):
        net.masks_u8(good.cpu())
    for bad in (good.float(), torch.zeros((1, 512, 512), dtype=torch.uint8, device=DEV),
                torch.zeros((1, 512, 512, 4), dtype=torch.uint8, device=DEV)):
        with pytest.raises(RuntimeError, match='uint8'):
            net.masks_u8(bad)
    lib = _lib.load()
    with pytest.raises(RuntimeError, match='NULL'):
        _lib.check(lib.cfb_bisenet_masks_u8(net._net, _lib.ptr(good), None, None, 1, 512, 512, None, 0, None), 'masks_u8')
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    with pytest.raises(RuntimeError, match='multiples of 32'):
        _lib.check(lib.cfb_bisenet_masks_u8(net._net, _lib.ptr(good), _lib.ptr(good), None, 1, 500, 512, _lib.ptr(ws), ws.numel(), None),
                   'masks_u8')
    with pytest.raises(RuntimeError, match='workspace'):
        _lib.check(lib.cfb_bisenet_masks_u8(net._net, _lib.ptr(good), _lib.ptr(good), None, 1, 512, 512, _lib.ptr(ws), ws.numel(), None),
                   'masks_u8')
    assert not lib.cfb_bisenet_create(0) and not lib.cfb_bisenet_create(65)
    with pytest.raises(NotImplementedError):
        cb.init_parsing_model('bisenet_v2')
    c, m = net.masks_u8(torch.empty((0, 512, 512, 3), dtype=torch.uint8, device=DEV))
    assert c.shape == (0, 512, 512) and m.shape == (0, 512, 512)
    # the device context stays usable after every refusal
    assert torch.equal(net.masks_u8(good)[0], bise.net.masks_u8(good)[0])


def test_nan_input(bise):
    x = torch.full((1, 3, 64, 64), float('nan'), device=DEV)
    outs = bise.net(x)
    cls, mask = cb.face_parse_mask(outs[0])
    torch.cuda.synchronize()
    cb.check_async_status()
    assert int(cls.max()) < 19 and set(torch.unique(mask).tolist()) <= {0, 255}
    assert torch.equal(bise.net.masks_u8(_faces(1))[0], bise.net.masks_u8(_faces(1))[0]), 'the next call works'
