"""-m gpu: ParseNet's parse masks straight from uint8 faces (``ParseNet.masks_u8`` / ``cfb_parsenet_masks_u8``) and its fp16
precision (``ParseNet.set_precision('fp16')``).  In fp32 the fused path is byte-equal to cfb_u8_to_input -> forward ->
face_parse_mask, and the callers (parse_masks, paste_faces_to_input_image, restore_images) give the bytes of the unfused
chain, which a thin wrapper parser still takes.  fp16 logits are held to twice the error of the float64 emulation
(tests/parsenet_fp16_emul.py) against the reference golden."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import _lib
from codeformer_b200 import parsing as P
from codeformer_b200 import pasteback as PB
from oracle import pasteback_oracle as O
from tests import parsenet_fp16_emul as PE
from tests.test_gpu_wholeimage import _affines, nets, whole_images   # noqa: F401  (nets: fixture)
from tests.util import golden, maxabs

cv2 = pytest.importorskip('cv2')
pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = 'cuda'


def _net(sd, size=512, precision=None):
    net = cb.ParseNet(in_size=size, out_size=size, parsing_ch=19)
    net.load_state_dict(sd, strict=True)
    net = net.eval().to(DEV)
    return net.set_precision(precision) if precision else net


@pytest.fixture(scope='module')
def shipped():
    from oracle import gen_golden as GG
    sd, x = GG.parsenet_inputs()
    return SimpleNamespace(sd=sd, x=x, net=_net(sd))


def _faces(n):
    """n uint8 BGR 512x512 faces from the committed RGB fixtures: the four faces, then rolled and mirrored copies."""
    f = golden('faces.npz')['faces'][..., ::-1]
    out = [np.roll(f[i % 4], 37 * (i // 4), axis=1)[:, ::(-1 if (i // 4) % 2 else 1)] for i in range(n)]
    return torch.from_numpy(np.ascontiguousarray(np.stack(out))).to(DEV)


def _input(faces):
    """cfb_u8_to_input of uint8 BGR faces [N,H,W,3]: what parse_masks feeds the network."""
    N, H, W, _ = faces.shape
    x = torch.empty((N, 3, H, W), dtype=torch.float32, device=DEV)
    _lib.check(_lib.load().cfb_u8_to_input(_lib.ptr(faces.contiguous()), _lib.ptr(x), N, H * W,
                                           ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'cfb_u8_to_input')
    return x


def _chain(net, faces):
    """The unfused chain: cfb_u8_to_input -> forward -> face_parse_mask."""
    return cb.face_parse_mask(net(_input(faces))[0])


def _check_equal(net, faces):
    cls, mask = net.masks_u8(faces)
    rc, rm = _chain(net, faces)
    torch.cuda.synchronize()
    cb.check_async_status()
    assert cls.shape == rc.shape and mask.shape == rm.shape
    assert torch.equal(cls, rc), f'classes: {int((cls != rc).sum())} pixels differ'
    assert torch.equal(mask, rm), f'mask: {int((mask != rm).sum())} pixels differ'
    return cls, mask


# ---- fp32: byte-equal to the unfused chain ---------------------------------------------------------------------------
@pytest.mark.parametrize('batch', [1, 3, 40])
def test_masks_u8_equals_chain_shipped(shipped, batch):
    faces = _faces(batch)
    cls, mask = _check_equal(shipped.net, faces)
    assert len(torch.unique(mask)) == 2, 'the faces must give both mask values'
    # batch invariance and determinism
    for k in sorted({0, batch // 2, batch - 1}):
        one = shipped.net.masks_u8(faces[k:k + 1])
        assert torch.equal(one[0][0], cls[k]) and torch.equal(one[1][0], mask[k]), f'face {k} alone'
    again = shipped.net.masks_u8(faces)
    assert torch.equal(again[0], cls) and torch.equal(again[1], mask)


@pytest.mark.parametrize('size,batch,hw', [(64, 3, (64, 64)), (128, 2, (128, 128)), (128, 2, (96, 160))])
def test_masks_u8_equals_chain_small_configs(size, batch, hw):
    """1 and 2 down/up steps, and a non-square face."""
    net = _net(P.random_parsenet_state_dict(P.parsenet_spec(size, size), 5), size)
    faces = torch.from_numpy(np.random.default_rng(size + batch).integers(0, 256, (batch,) + hw + (3,), dtype=np.uint8)).to(DEV)
    cls, _ = _check_equal(net, faces)
    assert torch.equal(net.masks_u8(faces[1:2])[0][0], cls[1])


# ---- callers ----------------------------------------------------------------------------------------------------------
def test_parse_masks_equals_wrapper(shipped):
    """A wrapper parser (not a ParseNet) takes the unfused chain: the same bytes, for 512 faces and for faces a face upsampler
    made (resized to 512 first)."""
    parser = shipped.net
    faces = _faces(5)
    big = PB.resize_linear(faces, (1024, 1024))
    for f in (faces, big):
        assert torch.equal(PB.parse_masks(f, parser), PB.parse_masks(f, lambda x: parser(x)))


def test_paste_faces_to_input_image_equals_wrapper(shipped):
    rng = np.random.default_rng(2)
    for gray in (False, True):
        img = O.synthetic_background(300, 420, 5)
        if gray:
            img = cv2.cvtColor(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), cv2.COLOR_GRAY2BGR)
        aff = _affines(rng, 3, 300, 420)
        faces = list(_faces(3).cpu().numpy())

        def paste(parser):
            helper = SimpleNamespace(input_img=img, upscale_factor=2, face_size=(512, 512), restored_faces=list(faces),
                                     inverse_affine_matrices=[cv2.invertAffineTransform(a) * 2 for a in aff], use_parse=True,
                                     face_parse=parser)
            return PB.paste_faces_to_input_image(helper)
        a, b = paste(shipped.net), paste(lambda x: shipped.net(x))
        assert a.shape == (600, 840, 3) and np.array_equal(a, b), f'gray={gray}'


def test_restore_images_equals_wrapper(nets):
    base = whole_images()
    imgs = [base[0], cv2.cvtColor(cv2.cvtColor(base[1], cv2.COLOR_BGR2GRAY), cv2.COLOR_GRAY2BGR), base[2], base[-1]]
    a, _, faces = cb.restore_images(imgs, nets.net, nets.det, parser=nets.parser, max_batch=4, return_faces=True)
    assert sum(len(f) for f in faces) >= 2
    b = cb.restore_images(imgs, nets.net, nets.det, parser=lambda x: nets.parser(x), max_batch=4)
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), f'image {i}: {int((x != y).sum())} bytes differ'


# ---- fp16 ------------------------------------------------------------------------------------------------------------
def test_fp16_vs_reference_golden(shipped):
    """fp16 logits against the reference's fp32 logits: error <= 2x that of the float64 emulation of ParseNet in fp16, +1e-4;
    classes equal the golden's wherever the golden top-1/top-2 margin exceeds that bound."""
    net = _net(shipped.sd, precision='fp16')
    logits = net(shipped.x.to(DEV))[0]
    torch.cuda.synchronize()
    cb.check_async_status()
    g = golden('parsenet.npz')
    err = maxabs(logits[..., ::4, ::4].cpu(), g['mask_s4'])
    emul = PE.parsenet_forward(shipped.sd, shipped.x.to(DEV), P.parsenet_plan(512, 512)[0])
    err_emul = maxabs(emul[..., ::4, ::4].cpu(), g['mask_s4'])
    bound = 2 * err_emul + 1e-4
    print(f'parsenet fp16: max-abs {err:.3e}, emulation {err_emul:.3e} (|logit|max {float(np.abs(g["mask_s4"]).max()):.3f})')
    assert logits.shape == (1, 19, 512, 512) and err <= bound
    cls = cb.face_parse_mask(logits)[0].cpu()
    gc = torch.from_numpy(g['classes'])
    sure = torch.from_numpy(g['margin'].astype(np.float32)) > bound
    print(f'parsenet fp16: {float((cls != gc).float().mean()) * 100:.3f} % of pixels change class '
          f'({float(sure.float().mean()) * 100:.1f} % have a margin above {bound:.2e})')
    assert torch.equal(cls[sure], gc[sure])
    assert torch.equal(net(shipped.x.to(DEV))[0], logits), 'deterministic'


def test_fp16_masks_u8_equals_fp16_chain(shipped):
    net = _net(shipped.sd, precision='fp16')
    faces = _faces(3)
    cls, mask = _check_equal(net, faces)
    assert torch.equal(PB.parse_masks(faces, net), mask), 'parse_masks takes masks_u8 in fp16 too'
    assert not torch.equal(cls, shipped.net.masks_u8(faces)[0]), 'fp16 must take effect'


def test_precision_switching_keeps_fp32_bits(shipped):
    sd = P.random_parsenet_state_dict(P.parsenet_spec(128, 128), 3)
    x = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(1)).to(DEV) * 2 - 1
    net = _net(sd, 128)
    assert net.precision == 'fp32'
    a = net(x)[0]
    assert net.set_precision('fp16') is net and net.precision == 'fp16'
    h = net(x)[0]
    net.set_precision('fp32')
    assert torch.equal(net(x)[0], a), 'fp32 -> fp16 -> fp32 gives the fp32 bits back'
    assert torch.equal(a, _net(sd, 128)(x)[0]) and torch.equal(h, _net(sd, 128, 'fp16')(x)[0])
    assert not torch.equal(a, h)
    net.set_precision('fp16')
    net.load_state_dict(sd)
    net = net.to(DEV)
    assert net.precision == 'fp16' and torch.equal(net(x)[0], h), 'kept across load_state_dict and .to()'
    for bad in ('bf16', 'half', 1, None):
        with pytest.raises(ValueError):
            net.set_precision(bad)
    assert net.precision == 'fp16'
    with pytest.raises(RuntimeError, match='precision'):
        _lib.check(_lib.load().cfb_parsenet_set_precision(net._net, 2), 'cfb_parsenet_set_precision')


def test_masks_u8_input_errors(shipped):
    net = shipped.net
    good = _faces(1)
    with pytest.raises(RuntimeError, match='CUDA'):
        net.masks_u8(good.cpu())
    with pytest.raises(RuntimeError, match='uint8'):
        net.masks_u8(good.float())
    for shape in [(1, 512, 512), (1, 512, 512, 4), (512, 512, 3)]:
        with pytest.raises(RuntimeError, match='uint8'):
            net.masks_u8(torch.zeros(shape, dtype=torch.uint8, device=DEV))
    for hw in [(500, 512), (512, 520), (16, 16)]:
        with pytest.raises(RuntimeError, match='multiples'):
            net.masks_u8(torch.zeros((1,) + hw + (3,), dtype=torch.uint8, device=DEV))
    lib = _lib.load()
    with pytest.raises(RuntimeError, match='NULL'):
        _lib.check(lib.cfb_parsenet_masks_u8(net._net, _lib.ptr(good), None, None, 1, 512, 512, None, 0, None), 'masks_u8')
    c, m = net.masks_u8(torch.empty((0, 512, 512, 3), dtype=torch.uint8, device=DEV))
    assert c.shape == (0, 512, 512) and m.shape == (0, 512, 512)
