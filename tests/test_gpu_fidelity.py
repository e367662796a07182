"""gpu: per-face fidelity weights.  A call with one ``w`` per face must give, for every face, exactly what the scalar call on
that face alone gives with its own ``w`` (``torch.equal``), for ``forward`` (also ``code_only``), ``forward_u8`` and the
inpainting path, in both precisions, on the three engines and on the graph, eager and multi-lane paths; a face with w <= 0 or
NaN gets the skipped-fusion result.  Also: the SFT epilogue alone (``cfb_debug_conv_tc_prec_wv`` against the scalar entry),
one CUDA graph for every w vector, ``restore_images`` / ``restore_aligned`` / ``restore_faces`` with per-image / per-crop /
per-face weights, and the argument errors."""
import ctypes
import math

import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import _lib
from codeformer_b200 import spec as S
from tests.test_gpu_aligned import inpaint_faces
from tests.test_gpu_wholeimage import nets, whole_images      # noqa: F401  (module fixture and inputs)
from tests.test_gpu_wide_tiles import plane_bytes
from tests.util import golden

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = 'cuda:0'
# mixed weights: inside (0, 1], 0, negative and NaN (both skip the fusion in the scalar call)
W_MIX = [0.5, 0.0, 1.0, -0.3, float('nan'), 0.7, 0.25, 0.5, 0.0]


def _weights(B, shift=0):
    return [W_MIX[(i + shift) % len(W_MIX)] for i in range(B)]


@pytest.fixture(scope='module')
def net():
    n = cb.CodeFormer().to(DEV).eval()
    n.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1))
    return n


@pytest.fixture(scope='module')
def net_inpaint():          # inference_inpainting.py:45-46: codebook 512, three connections
    kw = dict(codebook_size=512, connect_list=['32', '64', '128'])
    n = cb.CodeFormer(**kw).to(DEV).eval()
    n.load_state_dict(S.random_state_dict(S.codeformer_spec(**kw), 4))
    return n


@pytest.fixture
def mode(net, request):
    """(engine, precision) of the module for one test; restored afterwards."""
    def set_mode(engine, precision):
        net.set_engine(engine)
        net.set_precision(precision)
    yield set_mode
    net.set_engine('auto')
    net.set_precision('fp32')
    net._cfb_graphs.clear()


def faces_u8(B):
    f = np.ascontiguousarray(golden('faces.npz')['faces'][..., ::-1])
    return np.stack([f[i % len(f)] for i in range(B)])


def faces_x(B):
    x = torch.from_numpy(faces_u8(B)[..., ::-1].astype(np.float32) / 255.).permute(0, 3, 1, 2).contiguous()
    return ((x - 0.5) / 0.5).to(DEV)


def _groups(ws):
    """face indices grouped by weight (NaN is one group)."""
    g = {}
    for i, v in enumerate(ws):
        g.setdefault('nan' if math.isnan(v) else v, []).append(i)
    return g


def scalar_reference(call, B, ws, alone):
    """Per face, the scalar call's result for that face with its own w: face by face when ``alone``, else one scalar call per
    distinct w over the faces that share it (faces are independent in every forward: the batch-invariance tests pin this)."""
    outs = None
    for key, idx in _groups(ws).items():
        w = float('nan') if key == 'nan' else key
        for sel in ([[i] for i in idx] if alone else [idx]):
            res = call(sel, w)
            if outs is None:
                outs = [torch.empty((B,) + r.shape[1:], dtype=r.dtype, device=r.device) for r in res]
            for o, r in zip(outs, res):
                o[sel] = r
    return outs


PATHS = [(1, 'graph'), (1, 'eager'), (3, 'graph'), (3, 'eager'), (32, 'eager'), (32, 'lanes')]


def _path(monkeypatch, path):
    if path != 'graph':
        monkeypatch.setenv('CFB_CUDA_GRAPH', '0')
    if path == 'lanes':
        monkeypatch.setenv('CFB_STREAM_LANES', '2')


@pytest.mark.parametrize('engine,precision', [('auto', 'fp32'), ('tc', 'fp32'), ('f32', 'fp32'), ('auto', 'fp16'), ('tc', 'fp16')])
@pytest.mark.parametrize('B,path', PATHS)
def test_forward_per_face_equals_scalar(net, mode, monkeypatch, engine, precision, B, path):
    mode(engine, precision)
    _path(monkeypatch, path)
    x = faces_x(B)
    ws = _weights(B, B)
    got = net(x, w=ws, adain=True)
    cb.check_async_status()
    ref = scalar_reference(lambda sel, w: net(x[sel], w=w, adain=True), B, ws, alone=B <= 3)
    for name, g, r in zip(('out', 'logits', 'lq_feat'), got, ref):
        assert torch.equal(g, r), name


@pytest.mark.parametrize('engine', ['auto', 'f32'])
def test_forward_code_only(net, mode, engine):
    mode(engine, 'fp32')
    x = faces_x(3)
    ws = torch.tensor([0.5, 0.0, 1.0], device=DEV)
    logits, lq = net(x, w=ws, code_only=True)
    rl, rq = net(x, w=0.3, code_only=True)           # code_only never depends on w
    assert torch.equal(logits, rl) and torch.equal(lq, rq)


@pytest.mark.parametrize('precision', ['fp32', 'fp16'])
@pytest.mark.parametrize('inpaint', [False, True])
@pytest.mark.parametrize('B,path', [(1, 'graph'), (3, 'graph'), (3, 'eager'), (32, 'eager')])
def test_forward_u8_per_face_equals_scalar(net, net_inpaint, mode, monkeypatch, precision, inpaint, B, path):
    m = net_inpaint if inpaint else net
    m.set_precision(precision)
    try:
        _path(monkeypatch, path)
        faces = torch.from_numpy(inpaint_faces(B) if inpaint else faces_u8(B)).to(DEV)
        ws = _weights(B, 2 * B + inpaint)
        got = m.forward_u8(faces, w=np.asarray(ws), adain=not inpaint, inpaint=inpaint)
        cb.check_async_status()
        ref, = scalar_reference(lambda sel, w: (m.forward_u8(faces[sel], w=w, adain=not inpaint, inpaint=inpaint),),
                                B, ws, alone=B <= 3)
        assert torch.equal(got, ref)
    finally:
        m.set_precision('fp32')
        m._cfb_graphs.clear()


def test_one_graph_for_every_w_vector(net):
    net._cfb_graphs.clear()
    faces = torch.from_numpy(faces_u8(2)).to(DEV)
    x = faces_x(2)
    vecs = [[0.5, 0.0], [1.0, 0.25], [float('nan'), 0.7], [0.1, 0.9]]
    got_u8 = [net.forward_u8(faces, w=v) for v in vecs]
    got_f = [net(x, w=torch.tensor(v), adain=True)[0] for v in vecs]
    assert sorted(k[0] for k in net._cfb_graphs) == ['u8wv', 'wv']       # one graph per entry point, whatever the values
    for v, gu, gf in zip(vecs, got_u8, got_f):
        for i, wi in enumerate(v):
            assert torch.equal(gu[i], net.forward_u8(faces[i:i + 1], w=wi)[0])
            assert torch.equal(gf[i], net(x[i:i + 1], w=wi, adain=True)[0][0])
    net._cfb_graphs.clear()


# ---- the SFT epilogue alone ----------------------------------------------------------------------------------------
def _debug_conv(entry, x, wt, b, dec, scl, sw, N, H, C, precision):
    lib = _lib.load()
    out = torch.empty(N, H, H, C, device=DEV)
    pl = torch.zeros(2 * plane_bytes(N, H, C), dtype=torch.uint8, device=DEV)
    gp = torch.zeros(N * H * H // 128 * 4 * 64, device=DEV)
    wsb = lib.cfb_conv2d_workspace_bytes(N, H, H, C, C, 3, 0)
    ws = torch.empty(int(wsb), dtype=torch.uint8, device=DEV)
    tn = ctypes.c_int32(0)
    _lib.check(getattr(lib, entry)(_lib.ptr(x), None, 0, _lib.ptr(wt), _lib.ptr(b), _lib.ptr(out), N, H, H, C, C, 0, 0, None,
                                   None, 0, None, _lib.ptr(dec), _lib.ptr(scl), sw, _lib.ptr(pl), _lib.ptr(gp), _lib.ptr(ws), wsb,
                                   _lib.stream(), ctypes.byref(tn), 3, 0, precision), entry)
    torch.cuda.synchronize()
    cb.check_async_status()
    return out, pl, gp, tn.value


@pytest.mark.parametrize('precision', [0, 1])
@pytest.mark.parametrize('C,H,tile', [(128, 32, 128), (256, 16, 128), (64, 32, -64)])
def test_sft_conv_per_image(precision, C, H, tile):
    """shift.2 of a Fuse_sft_block (raw planes in, SFT epilogue, planes and GroupNorm partials out) with one w per image
    equals the scalar entry with that image's w, image by image; w <= 0 / NaN gives dec exactly."""
    N = 5
    g = torch.Generator().manual_seed(C + H)
    x, dec, scl = [torch.randn(N, H, H, C, generator=g).to(DEV) for _ in range(3)]
    wt = (torch.randn(C, C, 3, 3, generator=g) / math.sqrt(9 * C)).to(DEV)
    b = torch.randn(C, generator=g).to(DEV)
    ws = [0.5, 0.0, -1.0, float('nan'), 1.0]
    wv = torch.tensor(ws, device=DEV)
    out, pl, gp, tn = _debug_conv('cfb_debug_conv_tc_prec_wv', x, wt, b, dec, scl, _lib.ptr(wv), N, H, C, precision)
    assert tn == tile
    img_pl = H * H * C * 2                                           # bytes of one image in one plane
    half = plane_bytes(N, H, C)
    for i, wi in enumerate(ws):
        # the scalar entry applies its w as given: w <= 0 / NaN images compare with w = 0, the blend the vector applies
        ro, rpl, rgp, _ = _debug_conv('cfb_debug_conv_tc_prec', x, wt, b, dec, scl, wi if wi > 0 else 0.0, N, H, C, precision)
        assert torch.equal(out[i], ro[i]), f'image {i}'
        for base in (0, half):
            assert torch.equal(pl[base + i * img_pl: base + (i + 1) * img_pl], rpl[base + i * img_pl: base + (i + 1) * img_pl])
        per = gp.numel() // N
        assert torch.equal(gp[i * per:(i + 1) * per], rgp[i * per:(i + 1) * per])
        if not wi > 0:
            assert torch.equal(out[i], dec[i])


# ---- front-ends ----------------------------------------------------------------------------------------------------
def test_restore_faces_per_face(net):
    faces = faces_u8(6)
    ws = _weights(6, 1)
    got = net.restore_faces(list(faces), w=ws, max_batch=4)
    assert net.last_restore_errors == []
    for i in range(6):
        assert np.array_equal(got[i], net.restore_faces([faces[i]], w=ws[i])[0]), f'face {i}'


def test_restore_faces_fp16_falls_back_per_chunk(net, monkeypatch):
    """A chunk whose status check fails (simulated on the host: the first status read reports an error, as an fp16 operand
    overflow of the Fuse_sft_blocks would) gives its input faces back; the other chunk keeps its per-face results."""
    faces = faces_u8(4)
    ws = [0.5, 0.0, 1.0, 0.3]
    calls = {'n': 0}
    real = _lib.load()

    class Lib:
        def __getattr__(self, k):
            return getattr(real, k)

        def cfb_check_async_status(self):
            calls['n'] += 1
            return 1 if calls['n'] == 1 else real.cfb_check_async_status()
    monkeypatch.setattr(_lib, 'load', lambda _l=Lib(): _l)
    got = net.restore_faces(list(faces), w=ws, max_batch=2)
    monkeypatch.undo()
    assert [lo for lo, _ in net.last_restore_errors] == [0]
    assert np.array_equal(got[0], faces[0]) and np.array_equal(got[1], faces[1])
    ref = net.restore_faces(list(faces[2:]), w=ws[2:], max_batch=2)
    assert np.array_equal(got[2], ref[0]) and np.array_equal(got[3], ref[1])


def test_restore_aligned_per_crop(net):
    rng = np.random.default_rng(3)
    crops = [rng.integers(0, 256, (s, s, 3), dtype=np.uint8) for s in (256, 512, 300, 256)]
    crops[2] = np.repeat(crops[2][..., :1], 3, axis=2)           # a gray crop
    ws = [0.5, 0.0, 1.0, float('nan')]
    got = cb.restore_aligned(crops, net, w=ws, max_batch=3)
    for i, c in enumerate(crops):
        ref = cb.restore_aligned([c], net, w=ws[i])[0]
        assert got[i].dtype == ref.dtype and np.array_equal(got[i], ref), f'crop {i}'


def test_restore_images_per_image(nets):
    imgs = whole_images()[:4]
    ws = [0.5, 0.0, 1.0, 0.8]
    got = cb.restore_images(imgs, nets.net, nets.det, parser=nets.parser, w=ws, max_batch=4)
    for i, im in enumerate(imgs):
        ref = cb.restore_images([im], nets.net, nets.det, parser=nets.parser, w=ws[i])[0]
        assert np.array_equal(got[i], ref), f'image {i}'


# ---- errors --------------------------------------------------------------------------------------------------------
def test_errors(net):
    x = faces_x(2)
    faces = torch.from_numpy(faces_u8(2)).to(DEV)
    with pytest.raises(RuntimeError, match='one fidelity weight per face'):
        net(x, w=[0.5, 0.5, 0.5])
    with pytest.raises(RuntimeError, match='one fidelity weight per face'):
        net.forward_u8(faces, w=torch.tensor([0.5], device=DEV))
    with pytest.raises(ValueError, match='floating point'):
        net.forward_u8(faces, w=torch.tensor([1, 0], device=DEV))
    with pytest.raises(ValueError, match='floating point'):
        net(x, w=np.array([1, 0]))
    with pytest.raises(RuntimeError, match='one fidelity weight per face'):
        net.restore_faces(list(faces_u8(3)), w=[0.5, 0.5])
    with pytest.raises(RuntimeError, match='one fidelity weight per face'):
        cb.restore_aligned(list(faces_u8(2)), net, w=[0.5])
    lib = _lib.load()
    assert lib.cfb_codeformer_forward_u8_wv(net._net, _lib.ptr(faces), _lib.ptr(faces), None, None, None, 2, None, 1, None, 0,
                                            _lib.stream()) != 0
    assert b'NULL w_dev' in lib.cfb_last_error()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs a second CUDA device')
def test_weights_on_another_device(net):
    with pytest.raises(RuntimeError, match='per-face fidelity weights are on'):
        net(faces_x(2), w=torch.tensor([0.5, 0.5], device='cuda:1'))
