"""gpu: fidelity sweeps.  ``CodeFormer.forward_u8_sweep`` must give, for every face b and weight k, exactly what
``forward_u8(face_b[None], w=ws[k])`` and the per-face-weight call give (``torch.equal``) on the 4-connect, 3-connect and
codebook-512 nets, at several batch sizes and sweep lengths, with AdaIN on and off, in both precisions, on every engine and on
the graph and eager paths; the encoder side runs once whatever K is.  ``restore_images_sweep`` must give, per weight, exactly
what ``restore_images`` gives at that weight, while detection and the background upsample run once per chunk of images."""
import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import spec as S
from codeformer_b200 import wholeimage as WI
from tests.test_gpu_fidelity import faces_u8
from tests.test_gpu_wholeimage import nets, whole_images      # noqa: F401  (module fixture and inputs)

cv2 = pytest.importorskip('cv2')
pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = 'cuda:0'
# inside (0, 1], 0, above 1, negative and NaN (the last two skip the fusion in a scalar call)
W_SWEEP = [0.5, 0.0, 1.0, -0.3, float('nan'), 1.7]


def sweep_ws(K, shift=0):
    return [W_SWEEP[(i + shift) % len(W_SWEEP)] for i in range(K)]


_NETS = []          # CodeFormer modules of this file: their graphs and workspaces are freed after every test


@pytest.fixture(autouse=True)
def clean_status():
    yield
    torch.cuda.synchronize()
    cb.check_async_status()
    for n in _NETS:     # decoder batches of B*K faces: graph-pinned workspaces of earlier tests would pile up
        n._cfb_graphs.clear()
        n._cfb_ws.clear()
    torch.cuda.empty_cache()


def _make(seed, **kw):
    n = cb.CodeFormer(**kw).to(DEV).eval()
    n.load_state_dict(S.random_state_dict(S.codeformer_spec(**kw), seed))
    _NETS.append(n)
    return n


@pytest.fixture(scope='module')
def net():
    return _make(1)


@pytest.fixture(scope='module')
def variants(net):
    return {'main': net,
            'conn3': _make(2, connect_list=['32', '64', '128']),
            'cb512': _make(4, codebook_size=512, connect_list=['32', '64', '128'])}


@pytest.fixture
def mode(net):
    def set_mode(engine, precision):
        net.set_engine(engine)
        net.set_precision(precision)
    yield set_mode
    net.set_engine('auto')
    net.set_precision('fp32')
    net._cfb_graphs.clear()


def check_sweep(n, B, ws, adain=True):
    """the sweep against the scalar call on each face alone and against one per-face-w call over the repeated faces"""
    faces = torch.from_numpy(faces_u8(B)).to(DEV)
    K = len(ws)
    got = n.forward_u8_sweep(faces, ws, adain=adain)
    assert got.shape == (B, K, 512, 512, 3) and got.dtype == torch.uint8
    per_face = n.forward_u8(faces.repeat_interleave(K, 0), w=ws * B, adain=adain).view(B, K, 512, 512, 3)
    assert torch.equal(got, per_face)
    for b in range(B):
        for k in range(K):
            ref = n.forward_u8(faces[b:b + 1], w=ws[k], adain=adain)[0]
            assert torch.equal(got[b, k], ref), f'face {b}, w {ws[k]}'
    return got


@pytest.mark.parametrize('B', [1, 3, 6])
@pytest.mark.parametrize('K', [1, 2, 5])
def test_sweep_equals_scalar_calls(net, B, K):
    check_sweep(net, B, sweep_ws(K, shift=B))          # B <= cuda_graph_max_batch: graph replay; B = 6: eager


@pytest.mark.parametrize('which,B,K', [('conn3', 1, 5), ('conn3', 6, 2), ('cb512', 3, 2), ('cb512', 6, 5)])
def test_sweep_other_nets(variants, which, B, K):
    check_sweep(variants[which], B, sweep_ws(K, shift=K))


@pytest.mark.parametrize('adain', [False, True])
def test_sweep_adain(net, adain):
    check_sweep(net, 2, sweep_ws(3, shift=3), adain=adain)


@pytest.mark.parametrize('engine,precision', [('tc', 'fp32'), ('f32', 'fp32'), ('auto', 'fp16'), ('tc', 'fp16')])
@pytest.mark.parametrize('B,K', [(2, 3), (5, 2)])
def test_sweep_engines_and_precisions(net, mode, engine, precision, B, K):
    mode(engine, precision)
    check_sweep(net, B, sweep_ws(K, shift=1))


def test_sweep_batch_invariance(net):
    ws = sweep_ws(4, shift=2)
    faces = torch.from_numpy(faces_u8(6)).to(DEV)
    six = net.forward_u8_sweep(faces, ws)
    for b in range(6):
        assert torch.equal(net.forward_u8_sweep(faces[b:b + 1], ws)[0], six[b]), f'face {b}'


def test_sweep_graph_serves_every_ws(net):
    faces = torch.from_numpy(faces_u8(2)).to(DEV)
    net._cfb_graphs.clear()
    a = net.forward_u8_sweep(faces, [0.5, 1.0])
    b = net.forward_u8_sweep(faces, torch.tensor([1.0, 0.5], device=DEV))
    assert [k[0] for k in net._cfb_graphs] == ['u8sweep']
    assert torch.equal(a[:, 0], b[:, 1]) and torch.equal(a[:, 1], b[:, 0])


def test_encoder_side_runs_once(net):
    """the w-independent part is launched once: a sweep's launch count does not grow with K"""
    faces = torch.from_numpy(faces_u8(5)).to(DEV)      # B > cuda_graph_max_batch: every call launches
    counts = []
    for K in (2, 5):
        net.forward_u8_sweep(faces, sweep_ws(K))
        counts.append(net.last_launch_count)
    assert counts[0] == counts[1] > 0


def test_sweep_argument_errors(net):
    faces = torch.from_numpy(faces_u8(1)).to(DEV)
    for bad in ([], [[0.5, 1.0]], np.zeros((2, 2), np.float32), torch.tensor([1, 2]), np.array([1, 2]), 0.5, 'ab'):
        with pytest.raises(ValueError):
            net.forward_u8_sweep(faces, bad)
    with pytest.raises(RuntimeError):
        net.forward_u8_sweep(faces.cpu(), [0.5])
    with pytest.raises(RuntimeError):
        net.forward_u8_sweep(faces.float(), [0.5])
    with pytest.raises(RuntimeError):
        net.forward_u8_sweep(faces[:, :256], [0.5])
    assert net.forward_u8_sweep(faces[:0], [0.5, 1.0]).shape == (0, 2, 512, 512, 3)
    if torch.cuda.device_count() > 1:
        with pytest.raises(RuntimeError):
            net.forward_u8_sweep(faces, torch.tensor([0.5], device='cuda:1'))


# ---- whole images ------------------------------------------------------------------------------------------------
WS = [0.5, 0.0, 1.0]


def _counting(monkeypatch, obj, name):
    calls = []
    orig = getattr(obj, name)

    def spy(*a, **k):
        calls.append(1)
        return orig(*a, **k)
    monkeypatch.setattr(obj, name, spy)
    return calls


def check_images(imgs, net, det, ws=WS, monkeypatch=None, bg=None, **kw):
    if net not in _NETS:
        _NETS.append(net)
    refs = [cb.restore_images(imgs, net, det, w=w, bg_upsampler=bg, return_faces=True, **kw) for w in ws]
    det_calls = bg_calls = None
    if monkeypatch is not None:
        inner = det.detector if isinstance(det, cb.YoloDetector) else det
        det_calls = _counting(monkeypatch, inner, 'forward_u8')
        if bg is not None:
            bg_calls = _counting(monkeypatch, bg, 'enhance_batch')
    res, crops, faces = cb.restore_images_sweep(imgs, net, det, ws, bg_upsampler=bg, return_faces=True, **kw)
    assert len(res) == len(faces) == len(ws)
    for k, (ref, ref_crops, ref_faces) in enumerate(refs):
        for i in range(len(imgs)):
            a, b = res[k][i], ref[i]
            assert type(a) is type(b) and a.dtype == b.dtype and a.shape == b.shape, f'w {ws[k]}, image {i}'
            if torch.is_tensor(a):
                a, b = a.cpu().numpy(), b.cpu().numpy()
            assert np.array_equal(a, b), f'w {ws[k]}, image {i}: {int((a != b).sum())} elements differ'
            assert np.array_equal(np.asarray(crops[i].cpu() if torch.is_tensor(crops[i]) else crops[i]),
                                  np.asarray(ref_crops[i].cpu() if torch.is_tensor(ref_crops[i]) else ref_crops[i]))
            fa, fb = faces[k][i], ref_faces[i]
            fa, fb = (fa.cpu().numpy(), fb.cpu().numpy()) if torch.is_tensor(fa) else (fa, fb)
            assert fa.dtype == fb.dtype and np.array_equal(fa, fb)
    assert not cb.restore_images_sweep.last_errors
    n_chunks = len(WI._chunks([np.empty(im.shape, np.uint8) for im in imgs], max(1, int(kw.get('max_batch', 32)))))
    if det_calls is not None:
        assert len(det_calls) == n_chunks
    if bg_calls is not None:
        assert len(bg_calls) == n_chunks
    return crops


@pytest.mark.parametrize('max_batch', [1, 4, 32])
def test_restore_images_sweep_equals_restore_images(nets, monkeypatch, max_batch):
    crops = check_images(whole_images(), nets.net, nets.det, monkeypatch=monkeypatch, parser=nets.parser, max_batch=max_batch)
    assert sum(c.shape[0] for c in crops) >= 3


def test_restore_images_sweep_options(nets):
    imgs = whole_images()[3:]
    check_images(imgs, nets.net, nets.det, ws=[1.0, 0.25], upscale=1, only_center_face=True, max_batch=4)
    # CUDA inputs give CUDA outputs
    check_images([torch.from_numpy(im).to(DEV) for im in whole_images()[-2:]], nets.net, nets.det, parser=None, max_batch=4)


def test_restore_images_sweep_yolo_and_faceless_image(nets, monkeypatch):
    from codeformer_b200.yolov5face import random_yolov5l_state_dict
    det = cb.init_detection_model('YOLOv5l', device=DEV)
    det.detector.load_state_dict(random_yolov5l_state_dict(2, obj_bias=(1.25, -4.0, -4.0)), strict=True)
    crops = check_images(whole_images()[-2:], nets.net, det, monkeypatch=monkeypatch, parser=nets.parser, max_batch=4)
    assert sorted(c.shape[0] for c in crops)[0] == 0 and sum(c.shape[0] for c in crops) > 0


def test_restore_images_sweep_upsamplers_and_gray(nets, monkeypatch):
    from tests.test_gpu_lanczos_gray import _to_gray
    rrdb = cb.RRDBNet(3, 3, scale=2, num_block=1)
    rrdb.load_state_dict(S.random_state_dict(S.rrdbnet_spec(3, 3, 2, 64, 1, 32), 11))
    bg = cb.RealESRGANer(scale=2, model=rrdb, tile=0, pre_pad=0, device=DEV)
    fu = cb.RealESRGANer(scale=2, model=rrdb, tile=0, pre_pad=0, device=DEV)
    base = whole_images()
    imgs = [(_to_gray(base[-1]) * 0.5).astype(np.uint8), base[-1], base[4]]
    check_images(imgs, nets.net, nets.det, monkeypatch=monkeypatch, bg=bg, parser=nets.parser, face_upsampler=fu,
                 max_batch=4)
    # gray images without a face upsampler: float64 faces and the float64 paste
    check_images([_to_gray(base[-1]), base[1]], nets.net, nets.det, ws=[0.7, 0.0], parser=nets.parser)


def test_restore_images_sweep_fallback(nets, monkeypatch):
    img = whole_images()[-1]

    def boom(*a, **k):
        raise RuntimeError('injected failure')
    monkeypatch.setattr(nets.net, 'forward_u8_sweep', boom)
    out, crops, faces = cb.restore_images_sweep([img], nets.net, nets.det, WS, max_batch=4, return_faces=True)
    assert crops[0].shape[0] > 0
    for k in range(len(WS)):
        assert np.array_equal(crops[0], faces[k][0])
    errs = cb.restore_images_sweep.last_errors
    assert errs and all('injected failure' in m for _, m in errs)
    assert [lo for lo, _ in errs] == [lo for lo, _ in WI.sweep_chunks(crops[0].shape[0], len(WS), 4)]


def test_restore_images_sweep_errors(nets):
    img = whole_images()[-1]
    with pytest.raises(ValueError):
        cb.restore_images_sweep([img], nets.net, nets.det, [])
    with pytest.raises(RuntimeError):
        cb.restore_images_sweep([torch.from_numpy(img)], nets.net, nets.det, [0.5])
    with pytest.raises(NotImplementedError):
        cb.restore_images_sweep([img.astype(np.uint16)], nets.net, nets.det, [0.5])
    assert cb.restore_images_sweep([], nets.net, nets.det, [0.5, 1.0]) == [[], []]
