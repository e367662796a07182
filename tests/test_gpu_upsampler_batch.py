"""gpu: RealESRGANer on the device for batches of uint8 images (cfb_rrdb_forward_u8_tiles, RealESRGANer.enhance_batch) against
the generic pre_process / tile_process / post_process chain with the reference's uint8 conversion, and restore_images with
a RealESRGANer background / face upsampler against the per-image reference loop."""
import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import spec as S
from oracle import pasteback_oracle as O

cv2 = pytest.importorskip('cv2')
pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _net(scale, num_block=1, seed=11, precision='fp32'):
    """A seeded small RRDBNet whose outputs spread over [0, 1] and past both ends, so that the clamp and the rounding of
    the uint8 conversion are exercised."""
    sd = S.random_state_dict(S.rrdbnet_spec(3, 3, scale, 64, num_block, 32), seed)
    sd['conv_last.weight'] = sd['conv_last.weight'] * 12
    sd['conv_last.bias'] = sd['conv_last.bias'] + 0.5
    net = cb.RRDBNet(3, 3, scale=scale, num_block=num_block)
    net.load_state_dict(sd)
    return net.to(DEV).eval().set_precision(precision)


def _imgs(n, h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, 3), dtype=np.uint8)


def _to_u8(out_rgb_chw):
    """The reference's conversion of a model output (realesrgan_utils.py:203-210): clamp, RGB -> BGR, * 255, round, uint8."""
    out = out_rgb_chw.float().cpu().clamp_(0, 1).numpy()
    return (np.transpose(out[[2, 1, 0]], (1, 2, 0)) * 255.0).round().astype(np.uint8)


def generic_enhance(er, img):
    """enhance() through the generic chain: pre_process, tile_process (or process), post_process, uint8 conversion."""
    rgb = cv2.cvtColor(img.astype(np.float32) / 255, cv2.COLOR_BGR2RGB)
    return (er._run(rgb) * 255.0).round().astype(np.uint8)


class HostChain:
    """An upsampler object that is not this package's: the generic chain, one image per call; counts its calls."""

    def __init__(self, er):
        self.er, self.calls = er, 0

    def enhance(self, img, outscale=None):
        self.calls += 1
        return generic_enhance(self.er, img), 'RGB'


# ---- the entry point ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('precision', ['fp32', 'fp16'])
@pytest.mark.parametrize('scale', [2, 4])
def test_u8_tiles_equal_the_float_forward_on_the_host_prepared_tile(scale, precision):
    net = _net(scale, precision=precision)
    H, W, pre = 45, 38, 10
    img = _imgs(1, H, W, scale)
    er = cb.RealESRGANer(scale=scale, model=net, tile=0, pre_pad=pre, device=DEV)
    rgb = cv2.cvtColor(img[0].astype(np.float32) / 255, cv2.COLOR_BGR2RGB)
    er.pre_process(rgb)                                   # the host-prepared padded image [1,3,Hm,Wm]
    padded = er.img
    th, tw, iy, ix = 24, 20, 30, 26                       # a window over the bottom / right pads
    ref = _to_u8(net(padded[:, :, iy:iy + th, ix:ix + tw].contiguous())[0])
    images = torch.from_numpy(img).to(DEV)
    s = scale
    # the whole tile output at the canvas origin
    out = torch.full((1, H * s, W * s, 3), 77, dtype=torch.uint8, device=DEV)
    net.forward_u8_tiles(images, pre, [(0, iy, ix, 0, 0, th * s, tw * s, 0, 0)], th, tw, out)
    got = out.cpu().numpy()
    assert np.array_equal(got[0, :th * s, :tw * s], ref)
    assert (got[0, th * s:] == 77).all() and (got[0, :, tw * s:] == 77).all(), 'writes only the crop'
    # a crop placed elsewhere, partly past the canvas (discarded, as post_process does)
    out.fill_(77)
    cy, cx, ch, cw, oy, ox = 4, 6, 20, 16, H * s - 12, 12
    net.forward_u8_tiles(images, pre, [(0, iy, ix, cy, cx, ch, cw, oy, ox)], th, tw, out)
    got = out.cpu().numpy()
    assert np.array_equal(got[0, oy:, ox:ox + cw], ref[cy:cy + 12, cx:cx + cw])
    keep = np.ones(got.shape[1:3], bool)
    keep[oy:, ox:ox + cw] = False
    assert (got[0][keep] == 77).all()
    torch.cuda.synchronize()
    cb.check_async_status()


# ---- enhance_batch --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('precision', ['fp32', 'fp16'])
@pytest.mark.parametrize('pre_pad', [0, 10])
@pytest.mark.parametrize('tile', [0, 24])
@pytest.mark.parametrize('scale', [2, 4])
def test_enhance_batch_equals_the_generic_chain(scale, tile, pre_pad, precision):
    net = _net(scale, precision=precision)
    er = cb.RealESRGANer(scale=scale, model=net, tile=tile, tile_pad=6, pre_pad=pre_pad, device=DEV)
    H, W = 37, 45                                         # odd: mod pad at x2; tile 24 / pad 6 leaves ragged edge tiles
    imgs = _imgs(3, H, W, scale * 100 + tile + pre_pad)
    refs = [generic_enhance(er, im) for im in imgs]
    x = torch.from_numpy(imgs).to(DEV)
    outs = {}
    for mt in (1, 3, None, 10 ** 6):
        out = er.enhance_batch(x, max_tiles=mt)
        assert out.is_cuda and out.dtype == torch.uint8 and out.shape == (3, H * scale, W * scale, 3)
        outs[mt] = out.cpu().numpy()
        for i in range(3):
            d = outs[mt][i] != refs[i]
            assert not d.any(), f'max_tiles {mt}, image {i}: {int(d.sum())} bytes differ'
    one = er.enhance_batch(x[1:2], outscale=scale).cpu().numpy()
    assert np.array_equal(one[0], refs[1])
    # enhance() routes uint8 3-channel images through the same device path
    e, mode = er.enhance(imgs[2], outscale=scale)
    assert mode == 'RGB' and np.array_equal(e, refs[2])
    r = np.stack(refs)
    assert ((r > 0) & (r < 255)).mean() > 0.2 and (r == 0).any() and (r == 255).any(), 'clamp and rounding exercised'
    torch.cuda.synchronize()
    cb.check_async_status()


def test_enhance_batch_of_faces_at_the_production_tile():
    """512 x 512 faces with tile=400, tile_pad=40: four window shapes, two of them 152 pixels wide."""
    net = _net(2)
    er = cb.RealESRGANer(scale=2, model=net, tile=400, tile_pad=40, pre_pad=0, device=DEV)
    imgs = _imgs(3, 512, 512, 5)
    out = er.enhance_batch(torch.from_numpy(imgs).to(DEV)).cpu().numpy()
    for i in range(3):
        assert np.array_equal(out[i], generic_enhance(er, imgs[i])), f'face {i}'


def test_threads_share_one_upsampler():
    import threading
    net = _net(2)
    er = cb.RealESRGANer(scale=2, model=net, tile=24, tile_pad=6, pre_pad=10, device=DEV)
    imgs = [_imgs(2, 30 + 4 * k, 41, k) for k in range(4)]
    refs = [er.enhance_batch(torch.from_numpy(im).to(DEV)).cpu().numpy() for im in imgs]
    res = [None] * 4

    def run(k):
        res[k] = er.enhance_batch(torch.from_numpy(imgs[k]).to(DEV)).cpu().numpy()
    ts = [threading.Thread(target=run, args=(k,)) for k in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for k in range(4):
        assert np.array_equal(res[k], refs[k])


def test_errors():
    net = _net(2)
    er = cb.RealESRGANer(scale=2, model=net, tile=0, pre_pad=10, device=DEV)
    x = torch.from_numpy(_imgs(1, 20, 24, 1)).to(DEV)
    with pytest.raises(NotImplementedError):
        er.enhance_batch(x, outscale=3)                   # INTER_LANCZOS4 is not built
    with pytest.raises(NotImplementedError):
        er.enhance_batch(x.to(torch.int16))
    with pytest.raises(NotImplementedError):
        er.enhance_batch(torch.zeros(1, 20, 24, 4, dtype=torch.uint8, device=DEV))
    with pytest.raises(NotImplementedError):
        er.enhance_batch(x[..., 0])
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        er.enhance_batch(x.cpu())
    with pytest.raises(RuntimeError, match='pre_pad'):     # pad not smaller than the dimension it reflects
        er.enhance_batch(x[:, :10])
    odd = cb.RealESRGANer(scale=2, model=net, tile=16, tile_pad=3, pre_pad=0, device=DEV)
    with pytest.raises(AssertionError):                   # 19-pixel windows at x2: not a multiple of the unshuffle factor
        odd.enhance_batch(x)
    four = cb.RRDBNet(3, 3, scale=2, num_block=1).to(DEV)
    other = cb.RealESRGANer(scale=2, model=torch.nn.Identity(), tile=0, pre_pad=0, device=DEV)
    with pytest.raises(NotImplementedError):
        other.enhance_batch(x)
    lib = cb._lib.load()
    four._prepare(x.device)
    ws = four._workspace(1, 20, 24, x.device)
    out = torch.empty(1, 40, 48, 3, dtype=torch.uint8, device=DEV)
    import ctypes
    bad = (ctypes.c_int32 * 9)(0, 2, 0, 0, 0, 40, 48, 0, 0)          # window past the padded image
    assert lib.cfb_rrdb_forward_u8_tiles(four._net, cb._lib.ptr(x), 1, 20, 24, 0, bad, 1, 20, 24, cb._lib.ptr(out),
                                         cb._lib.ptr(ws), ws.numel(), None) != 0
    assert b'outside the padded image' in lib.cfb_last_error()
    # the generic chain keeps 16-bit images
    img16 = (_imgs(1, 20, 24, 3)[0].astype(np.uint16) * 257)
    o16, mode = er.enhance(img16)
    assert o16.dtype == np.uint16 and o16.shape == (40, 48, 3) and mode == 'RGB'
    torch.cuda.synchronize()
    cb.check_async_status()


# ---- restore_images -------------------------------------------------------------------------------------------------
from tests.test_gpu_wholeimage import nets, reference_loop, whole_images  # noqa: E402,F401  (the module fixture)


def _spy(er):
    calls = []
    orig = er.enhance

    def enhance(*a, **k):
        calls.append(1)
        return orig(*a, **k)
    er.enhance = enhance
    return calls


def test_restore_images_with_device_upsamplers(nets, monkeypatch):
    from codeformer_b200 import pasteback as PB
    bg = cb.RealESRGANer(scale=2, model=_net(2, seed=11), tile=400, tile_pad=40, pre_pad=0, device=DEV)
    face = cb.RealESRGANer(scale=2, model=_net(2, seed=12), tile=400, tile_pad=40, pre_pad=0, device=DEV)
    # frames that read_image does not enlarge (the reference resizes an upsampled background of another size with LANCZOS4)
    imgs = whole_images()[-2:] + [np.ascontiguousarray(whole_images()[-1][::-1]), O.synthetic_background(512, 600, 7)]
    host_bg, host_face = HostChain(bg), HostChain(face)
    orig = PB.paste_faces_to_input_image
    monkeypatch.setattr(PB, 'paste_faces_to_input_image',
                        lambda h, upsample_img=None: orig(h, upsample_img=upsample_img, face_upsampler=host_face))
    refs = [reference_loop(im, nets.net, nets.det, nets.parser, bg_upsampler=host_bg) for im in imgs]
    monkeypatch.setattr(PB, 'paste_faces_to_input_image', orig)
    n_faces = sum(n for _, n in refs)
    print('faces per image', [n for _, n in refs])
    assert n_faces > 0
    bg_calls, face_calls = _spy(bg), _spy(face)
    for cuda_inputs in (False, True):
        for max_batch in (1, 4):
            inputs = [torch.from_numpy(im).to(DEV) for im in imgs] if cuda_inputs else imgs
            res = cb.restore_images(inputs, nets.net, nets.det, parser=nets.parser, bg_upsampler=bg, face_upsampler=face,
                                    max_batch=max_batch)
            for i, ((ref, _), out) in enumerate(zip(refs, res)):
                out = out.cpu().numpy() if cuda_inputs else out
                assert np.array_equal(out, ref), f'image {i} (cuda {cuda_inputs}, max_batch {max_batch}): ' \
                                                 f'{int((out != ref).sum())} bytes differ'
    assert not bg_calls and not face_calls, 'the host enhance is not called on the device path'
    # other upsampler objects keep their per-image / per-face host calls and give the same bytes
    host_bg.calls = host_face.calls = 0
    res = cb.restore_images(imgs, nets.net, nets.det, parser=nets.parser, bg_upsampler=host_bg, face_upsampler=host_face,
                            max_batch=4)
    assert host_bg.calls == len(imgs) and host_face.calls == n_faces
    for (ref, _), out in zip(refs, res):
        assert np.array_equal(out, ref)
    torch.cuda.synchronize()
    cb.check_async_status()


def test_restore_images_other_outscale_keeps_the_host_call(nets):
    """A x4 upsampler at upscale 2 needs the reference's LANCZOS4 resize inside enhance: it stays a host call per image."""
    bg = cb.RealESRGANer(scale=4, model=_net(4), tile=0, pre_pad=0, device=DEV)
    img = np.ascontiguousarray(whole_images()[-1][:600, :600])
    ref, _ = reference_loop(img, nets.net, nets.det, nets.parser, bg_upsampler=bg)
    calls = _spy(bg)
    out = cb.restore_images([img], nets.net, nets.det, parser=nets.parser, bg_upsampler=bg, upscale=2)[0]
    assert calls == [1] and np.array_equal(out, ref)
