"""-m gpu: the face-only scripts on the device -- inpainting (``forward_u8(inpaint=True)``, the blend fused into the last
conv), the --has_aligned loop over crops of any size (``restore_aligned``), the batched gray test (``cfb_is_gray_u8``) and
colorization -- against the scripts' loops restated with the reference's arithmetic (tests/aligned_restate.py and
oracle/plumbing_oracle.py, pinned on the reference by tests/test_aligned_restate_cpu.py)."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import _lib
from codeformer_b200 import spec as S
from codeformer_b200.wholeimage import _device_is_gray, _gray_sums, is_gray
from oracle import plumbing_oracle as P
from tests.aligned_restate import aligned_crop, inpaint_blend
from tests.util import golden

cv2 = pytest.importorskip('cv2')
pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
WHOLE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'whole_imgs')
C3 = ('32', '64', '128')


def _net(seed, **kw):
    net = cb.CodeFormer(**{k: (list(v) if k == 'connect_list' else v) for k, v in kw.items()}).to(DEV).eval()
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(**kw), seed))
    return net


@pytest.fixture(scope='module')
def net_inpaint():          # inference_inpainting.py:45-46: codebook 512, three connections
    return _net(4, codebook_size=512, connect_list=C3)


@pytest.fixture(scope='module')
def net_c3():               # inference_colorization.py:45-46: codebook 1024, three connections
    return _net(3, connect_list=C3)


@pytest.fixture(scope='module')
def net_main():
    return _net(1)


def faces_bgr():
    return np.ascontiguousarray(golden('faces.npz')['faces'][..., ::-1])        # committed faces are RGB


def inpaint_faces(B):
    """Faces with white holes: painted blocks, isolated (255,255,255) pixels beside near-white ones, an all-white face and a
    face without any white pixel, cycled to B faces."""
    f = faces_bgr()
    kinds = []
    a = f[0].copy()
    a[100:180, 150:300] = 255
    a[300:340, 60:90] = 255
    kinds.append(a)
    b = f[1].copy()
    ys, xs = np.mgrid[20:500:24, 20:500:24]
    b[ys, xs] = 255
    b[ys, xs + 1] = (255, 255, 254)
    b[ys, xs + 2] = (255, 254, 255)
    b[ys + 1, xs] = (254, 255, 255)
    kinds.append(b)
    kinds.append(np.full((512, 512, 3), 255, np.uint8))
    kinds.append(np.minimum(f[2], 254))
    c = f[3].copy()
    c[200:260, 200:260] = 255
    c[400:, :] = 255
    kinds.append(c)
    return np.stack([kinds[i % len(kinds)] for i in range(B)])


def script_inpaint(net, faces):
    """inference_inpainting.py:64-75 restated on the device for a batch: u8_to_input, forward(w=1, adain=False), mask, blend,
    tensor2img."""
    x = torch.from_numpy(P.face_to_input(faces)).to(DEV)
    out = net(x, w=1, adain=False)[0]
    return P.output_to_face(inpaint_blend(x, out).cpu().numpy())


@pytest.mark.parametrize('precision', ['fp32', 'fp16'])
@pytest.mark.parametrize('B,graph', [(1, True), (1, False), (3, True), (3, False), (32, False)])
def test_inpaint_equals_the_script(net_inpaint, monkeypatch, B, graph, precision):
    if not graph:
        monkeypatch.setenv('CFB_CUDA_GRAPH', '0')
    faces = inpaint_faces(B)
    net_inpaint.set_precision(precision)
    try:
        want = script_inpaint(net_inpaint, faces)
        got = net_inpaint.forward_u8(torch.from_numpy(faces).to(DEV), w=1, adain=False, inpaint=True)
        torch.cuda.synchronize()
        cb.check_async_status()
    finally:
        net_inpaint.set_precision('fp32')
    assert got.dtype == torch.uint8 and tuple(got.shape) == (B, 512, 512, 3)
    got = got.cpu().numpy()
    assert np.array_equal(got, want)
    white = (faces == 255).all(-1)
    assert np.array_equal(got[~white], faces[~white])          # the input face wherever it is not (255, 255, 255)
    if B == 32:                                                 # every kind of face is in the batch
        assert white[0].any() and white[2].all() and not white[3].any() and not white[1].all()


def test_inpaint_and_plain_graphs_are_separate(net_inpaint):
    """The same batch, w and adain with and without the blend: two CUDA graphs, each with its own result."""
    faces = inpaint_faces(2)
    d = torch.from_numpy(faces).to(DEV)
    plain_want = P.output_to_face(net_inpaint(torch.from_numpy(P.face_to_input(faces)).to(DEV), w=1, adain=False)[0].cpu().numpy())
    for _ in range(2):
        inp = net_inpaint.forward_u8(d, w=1, adain=False, inpaint=True).cpu().numpy()
        plain = net_inpaint.forward_u8(d, w=1, adain=False).cpu().numpy()
        assert np.array_equal(plain, plain_want)
        assert np.array_equal(inp, script_inpaint(net_inpaint, faces))
        assert not np.array_equal(inp, plain)


def test_restore_faces_inpaint_and_fallback(net_inpaint):
    faces = inpaint_faces(7)
    want = script_inpaint(net_inpaint, faces)
    got = net_inpaint.restore_faces(list(faces), w=1, adain=False, max_batch=4, inpaint=True)
    assert len(got) == 7 and np.array_equal(np.stack(got), want)
    assert net_inpaint.last_restore_errors == []
    orig = net_inpaint.forward_u8

    def boom(*a, **k):
        assert k.get('inpaint') is True
        raise RuntimeError('injected failure')
    net_inpaint.forward_u8 = boom
    try:
        got = net_inpaint.restore_faces(list(faces), w=1, adain=False, max_batch=4, inpaint=True)
    finally:
        net_inpaint.forward_u8 = orig
    assert np.array_equal(np.stack(got), faces)                # inference_inpainting.py:78-80 saves the input face
    assert [lo for lo, _ in net_inpaint.last_restore_errors] == [0, 4]


def test_inpaint_c_entry_checks_arguments(net_inpaint):
    lib = _lib.load()
    net_inpaint.forward_u8(torch.from_numpy(inpaint_faces(1)).to(DEV), w=1, adain=False, inpaint=True)
    assert lib.cfb_codeformer_inpaint_u8(net_inpaint._net, None, None, None, None, None, 1, 1.0, 0, None, 0, None) != 0
    assert b'cfb_codeformer_inpaint_u8: NULL image pointer' in lib.cfb_last_error()
    assert lib.cfb_codeformer_inpaint_u8(None, None, None, None, None, None, 1, 1.0, 0, None, 0, None) != 0


def test_colorization_equals_the_script(net_c3):
    """inference_colorization.py:60-75: w=0, adain=True on the 3-connect net, plain tensor2img."""
    faces = faces_bgr()
    x = torch.from_numpy(P.face_to_input(faces)).to(DEV)
    want = P.output_to_face(net_c3(x, w=0, adain=True)[0].cpu().numpy())
    got = net_c3.restore_faces(list(faces), w=0, adain=True, max_batch=3)
    assert np.array_equal(np.stack(got), want)


# ---- the --has_aligned loop ----------------------------------------------------------------------------------------
SIZES = [(512, 512), (256, 256), (1024, 1024), (300, 400), (511, 513)]         # (w, h) of the crops


def aligned_inputs():
    """Crops of every size, cut from the committed whole images; every other one is made gray as an old photograph is."""
    imgs = [cv2.imread(os.path.join(WHOLE, f'{n}.jpg'), cv2.IMREAD_COLOR) for n in ('00', '01', '03', '04', '05')]
    out = []
    for k, (w, h) in enumerate(SIZES * 2):
        img = imgs[k % len(imgs)]
        crop = cv2.resize(img, (w, h), interpolation=cv2.INTER_AREA)
        if k % 2:
            crop = cv2.cvtColor(cv2.cvtColor(crop, cv2.COLOR_BGR2GRAY), cv2.COLOR_GRAY2BGR)
        out.append(np.ascontiguousarray(crop))
    return out


def reference_aligned(crops, net, w=0.5):
    """inference_codeformer.py:180-213 with --has_aligned, one crop at a time: host cv2.resize, is_gray, restore_faces,
    add_restored_face."""
    res, flags, resized = [], [], []
    for img in crops:
        crop, g = aligned_crop(img)
        restored = net.restore_faces([crop], w=w, adain=True)[0]
        helper = SimpleNamespace(is_gray=g, restored_faces=[])
        cb.add_restored_face(helper, restored, crop)
        res.append(helper.restored_faces[0])
        flags.append(g)
        resized.append(crop)
    return res, flags, resized


@pytest.fixture(scope='module')
def aligned_ref(net_main):
    crops = aligned_inputs()
    return crops, reference_aligned(crops, net_main)


@pytest.mark.parametrize('max_batch', [1, 4, 32])
def test_restore_aligned_host_inputs(net_main, aligned_ref, max_batch):
    crops, (want, flags, resized) = aligned_ref
    assert any(flags) and not all(flags)
    got, dcrops, gray = cb.restore_aligned(crops, net_main, w=0.5, max_batch=max_batch, return_crops=True)
    assert gray == flags
    assert np.array_equal(dcrops.cpu().numpy(), np.stack(resized))
    assert cb.restore_aligned.last_errors == []
    for g, r, f in zip(got, want, flags):
        assert isinstance(g, np.ndarray) and g.dtype == (np.float64 if f else np.uint8) and g.shape == (512, 512, 3)
        assert g.dtype == r.dtype and np.array_equal(g, r)


def test_restore_aligned_cuda_inputs(net_main, aligned_ref):
    crops, (want, _, _) = aligned_ref
    got = cb.restore_aligned([torch.from_numpy(c).to(DEV) for c in crops], net_main, w=0.5, max_batch=4)
    for g, r in zip(got, want):
        assert torch.is_tensor(g) and g.is_cuda
        assert np.array_equal(g.cpu().numpy(), r)
    mixed = [torch.from_numpy(c).to(DEV) if k % 3 == 0 else c for k, c in enumerate(crops)]
    got = cb.restore_aligned(mixed, net_main, w=0.5, max_batch=32)
    for k, (g, r) in enumerate(zip(got, want)):
        assert torch.is_tensor(g) == (k % 3 == 0)
        assert np.array_equal(g.cpu().numpy() if torch.is_tensor(g) else g, r)


def test_restore_aligned_w_adain_and_fallback(net_main):
    crops = aligned_inputs()[:4]
    x = [aligned_crop(c)[0] for c in crops]
    want = net_main.restore_faces(x, w=0.0, adain=False)
    got, _, gray = cb.restore_aligned(crops, net_main, w=0.0, adain=False, return_crops=True)
    for g, r, f in zip(got, want, gray):
        if not f:
            assert np.array_equal(g, r)
    orig = net_main.forward_u8

    def boom(*a, **k):
        raise RuntimeError('injected failure')
    net_main.forward_u8 = boom
    try:
        got, dcrops, gray = cb.restore_aligned(crops, net_main, max_batch=3, return_crops=True)
    finally:
        net_main.forward_u8 = orig
    assert [lo for lo, _ in cb.restore_aligned.last_errors] == [0, 3]
    assert 'injected failure' in cb.restore_aligned.last_errors[0][1]
    for g, c, f in zip(got, x, gray):
        if not f:
            assert np.array_equal(g, c)           # the reference's fallback: tensor2img of the input is the crop itself
    torch.cuda.synchronize()
    cb.check_async_status()


def test_restore_aligned_errors(net_main):
    crop = aligned_inputs()[1]
    with pytest.raises(RuntimeError):
        cb.restore_aligned([torch.from_numpy(crop)], net_main)
    with pytest.raises(NotImplementedError):
        cb.restore_aligned([crop.astype(np.uint16)], net_main)
    with pytest.raises(NotImplementedError):
        cb.restore_aligned([crop[:, :, 0]], net_main)
    with pytest.raises(NotImplementedError):
        cb.restore_aligned([np.zeros((300, 300, 4), np.uint8)], net_main)
    with pytest.raises(NotImplementedError):
        cb.restore_aligned([torch.from_numpy(crop[:, :, 0].copy()).to(DEV)], net_main)
    assert cb.restore_aligned([], net_main) == []


# ---- cfb_is_gray_u8 ------------------------------------------------------------------------------------------------
def _numpy_sums(imgs):
    c = imgs.astype(np.int64)
    d = [c[..., 0] - c[..., 1], c[..., 1] - c[..., 2], c[..., 2] - c[..., 0]]
    return np.stack([x.sum(axis=(1, 2)) for x in d] + [(x * x).sum(axis=(1, 2)) for x in d], axis=1)


def threshold_images():
    """G = R = base and B = base + e with e = +5 / -5 / 0 on 30 / 30 / 40 % of the pixels: the variances are 15, 0 and 15, so
    the score is exactly 10 (gray, ``<=``).  The second image moves one pixel to e = +6 and lands just above."""
    rng = np.random.default_rng(11)
    base = rng.integers(10, 240, (100, 100)).astype(np.int64)
    e = np.zeros(10000, np.int64)
    e[:3000], e[3000:6000] = 5, -5
    e = rng.permutation(e).reshape(100, 100)
    at = np.stack([base + e, base, base], -1).astype(np.uint8)
    above = at.copy()
    y, x = np.argwhere(e == 5)[0]
    above[y, x, 0] += 1
    return np.stack([at, above])


def test_is_gray_sums_exact():
    rng = np.random.default_rng(5)
    frames = rng.integers(0, 256, (3, 1080, 1920, 3), dtype=np.uint8)
    frames[1] = frames[1, :, :, :1]                                # a gray frame
    frames[2, :, :, 0] = 255                                       # sums far from zero
    frames[2, :, :, 2] = 0
    for imgs in (frames, threshold_images(), rng.integers(0, 256, (1, 7, 5, 3), dtype=np.uint8)):
        got = _gray_sums(torch.from_numpy(imgs).to(DEV))
        assert got.dtype == np.int64 and np.array_equal(got, _numpy_sums(imgs))
    t = threshold_images()
    assert [is_gray(im) for im in t] == [True, False]
    assert _device_is_gray(torch.from_numpy(t).to(DEV)) == [True, False]
    assert _device_is_gray(torch.from_numpy(t[0]).to(DEV)) is True
    assert _device_is_gray(torch.from_numpy(frames).to(DEV)) == [is_gray(f) for f in frames] == [False, True, False]
