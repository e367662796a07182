"""SURVEY.md section 8 rows f1 / f2 on the GPU: the caller's uint8 plumbing fused into the first / last conv and the
batched caller loop, against oracle/plumbing_oracle.py (pinned on the reference's img2tensor / normalize / tensor2img)."""
import ctypes

import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import _lib
from codeformer_b200 import spec as S
from tests.util import faces_input, golden

pytestmark = pytest.mark.gpu


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope='module')
def net_main():
    net = cb.CodeFormer().cuda().eval()
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1))
    return net


def faces_bgr(sel=slice(None)):
    return np.ascontiguousarray(golden('faces.npz')['faces'][sel][..., ::-1])       # committed faces are RGB


def test_plumbing_kernels_bit_exact_vs_golden():
    """cfb_u8_to_input / cfb_output_to_u8 == the reference's own functions on every byte value and every rounding
    half-way point (tests/golden/plumbing.npz, generated from basicsr/utils/img_util.py + torchvision normalize)."""
    lib = _lib.load()
    g = golden('plumbing.npz')
    face = torch.from_numpy(g['face_bgr'][None].copy()).cuda()
    x = torch.empty((1, 3, 64, 64), device='cuda')
    _lib.check(lib.cfb_u8_to_input(_lib.ptr(face), _lib.ptr(x), 1, 64 * 64, _stream()), 'cfb_u8_to_input')
    assert np.array_equal(x.cpu().numpy()[0], g['x'])
    out = torch.from_numpy(g['out'].copy()).cuda()
    img = torch.empty((1, 64, 64, 3), dtype=torch.uint8, device='cuda')
    _lib.check(lib.cfb_output_to_u8(_lib.ptr(out), _lib.ptr(img), 1, 64 * 64, _stream()), 'cfb_output_to_u8')
    assert np.array_equal(img.cpu().numpy()[0], g['restored_bgr'])


def test_plumbing_kernels_vs_oracle_full_size():
    from oracle import plumbing_oracle as P
    lib = _lib.load()
    f = faces_bgr(slice(0, 2))
    d = torch.from_numpy(f).cuda()
    x = torch.empty((2, 3, 512, 512), device='cuda')
    _lib.check(lib.cfb_u8_to_input(_lib.ptr(d), _lib.ptr(x), 2, 512 * 512, _stream()), 'cfb_u8_to_input')
    assert np.array_equal(x.cpu().numpy(), P.face_to_input(f))
    assert torch.equal(x.cpu(), faces_input(slice(0, 2)))
    o = (torch.randn(2, 3, 512, 512, generator=torch.Generator().manual_seed(5)) * 0.8)
    img = torch.empty((2, 512, 512, 3), dtype=torch.uint8, device='cuda')
    od = o.cuda()
    _lib.check(lib.cfb_output_to_u8(_lib.ptr(od), _lib.ptr(img), 2, 512 * 512, _stream()), 'cfb_output_to_u8')
    assert np.array_equal(img.cpu().numpy(), P.output_to_face(o.numpy()))


@pytest.mark.parametrize('batch', [1, 6])       # 1: CUDA-graph replay path, 6: plain launches
def test_fused_u8_forward_equals_fp32_path_plus_plumbing(net_main, batch):
    """The fused entry point must equal plumbing(oracle) o forward(fp32) o plumbing(oracle) bit for bit: the first conv
    sees the same fp32 input values, the last conv rounds the same fp32 accumulators."""
    from oracle import plumbing_oracle as P
    sel = [i % 4 for i in range(batch)]
    f = faces_bgr()[sel]
    x = torch.from_numpy(P.face_to_input(f)).cuda()
    out = net_main(x, w=0.5, adain=True)[0]
    want = P.output_to_face(out.cpu().numpy())
    got = net_main.forward_u8(torch.from_numpy(f).cuda(), w=0.5, adain=True)
    assert got.dtype == torch.uint8 and tuple(got.shape) == (batch, 512, 512, 3)
    assert np.array_equal(got.cpu().numpy(), want)


def test_fused_u8_forward_vs_reference_golden(net_main):
    """End of the chain against the UNMODIFIED reference: restored u8 face vs tensor2img(reference out) on golden face 0.
    out differs from the reference by <= 1e-3 (here ~1e-4) in [-1,1] => at most one grey level, and only next to a
    rounding boundary."""
    from oracle import plumbing_oracle as P
    g = golden('codeformer_main.npz')
    want = P.output_to_face(g['out'])
    got = net_main.forward_u8(torch.from_numpy(faces_bgr(slice(0, 1))).cuda(), w=0.5, adain=True).cpu().numpy()
    diff = np.abs(got.astype(np.int16) - want.astype(np.int16))
    assert diff.max() <= 1
    assert (diff != 0).mean() < 0.02


def test_restore_faces_front_end(net_main):
    """Row f2: a list of cropped faces in, list of restored faces out, chunked; == one forward_u8 per face."""
    f = faces_bgr()
    faces = [f[i % 4] for i in range(7)]
    res = net_main.restore_faces(faces, w=0.5, adain=True, max_batch=3)
    assert len(res) == 7 and all(r.dtype == np.uint8 and r.shape == (512, 512, 3) for r in res)
    single = [net_main.forward_u8(torch.from_numpy(f[i:i + 1]).cuda(), w=0.5, adain=True).cpu().numpy()[0] for i in range(4)]
    for i in range(7):
        assert np.array_equal(res[i], single[i % 4])
    assert net_main.restore_faces([], w=0.5) == []
    with pytest.raises(RuntimeError):
        net_main.restore_faces([np.zeros((256, 256, 3), np.uint8)])


def test_restore_faces_error_fallback_returns_input(net_main, monkeypatch):
    """inference_codeformer.py:209-211: on failure the restored face is the (round-tripped) input face."""
    f = faces_bgr(slice(0, 2))

    def boom(*a, **k):
        raise RuntimeError('injected failure')
    monkeypatch.setattr(net_main, 'forward_u8', boom)
    res = net_main.restore_faces(list(f), w=0.5, on_error='input')
    assert np.array_equal(np.stack(res), f) and len(net_main.last_restore_errors) == 1
    with pytest.raises(RuntimeError):
        net_main.restore_faces(list(f), w=0.5, on_error='raise')


def test_restore_host_c_entry(net_main):
    """cfb_codeformer_restore_host (host uint8 in / out through the C ABI) == forward_u8."""
    lib = _lib.load()
    f = faces_bgr(slice(1, 3))
    want = net_main.forward_u8(torch.from_numpy(f).cuda(), w=0.5, adain=True).cpu().numpy()
    hin = torch.from_numpy(f).pin_memory()
    hout = torch.empty_like(hin).pin_memory()
    iob = lib.cfb_host_io_bytes(net_main._net, 2)
    io = torch.empty(int(iob), dtype=torch.uint8, device='cuda')
    wsb = lib.cfb_workspace_bytes(net_main._net, 2)
    ws = torch.empty(int(wsb), dtype=torch.uint8, device='cuda')
    _lib.check(lib.cfb_codeformer_restore_host(net_main._net, _lib.ptr(hin), _lib.ptr(hout), 2, 0.5, 1, _lib.ptr(io), iob,
                                               _lib.ptr(ws), wsb, _stream()), 'cfb_codeformer_restore_host')
    assert np.array_equal(hout.numpy(), want)
