"""gpu: ResNetArcFace on the conv engine against the CPU oracle (oracle/arcface_oracle.py, pinned to the reference by
tests/test_oracle_arcface.py), its new conv forms against torch CPU fp32, the fused uint8 path, and identity_similarity."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import codeformer_b200 as cb
from codeformer_b200 import _lib, arcface as A, spec as S
from oracle import arcface_oracle as AO
from oracle import gen_golden_arcface as G

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
DEV = 'cuda:0'
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
# split-fp16 operands (fp32 parity): the embedding bound of the nets on the engine, relative to max(1, |ref|max); measured
# 2.3e-6 .. 3.9e-6 on the seeded weights (|ref|max ~0.9 .. 1.04) on an H100 80GB HBM3
EMB_BAR = 2e-4


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _bar(out, ref):
    err = float((out.cpu() - ref).abs().max())
    assert err <= 6e-5 * float(ref.abs().max()), err
    return err


def _conv(x, wt, b, stride, scale=None, shift=None, act=0, slope=0.0, res=None):
    """cfb_debug_arcface_conv on NCHW CPU tensors; scale / shift per-(image, channel) [n, cin]."""
    lib = _lib.load()
    n, cin, h, w = x.shape
    cout, k = wt.shape[0], wt.shape[2]
    ho, wo = (h + 1) // 2 if stride == 2 else h, (w + 1) // 2 if stride == 2 else w
    need = lib.cfb_conv2d_gen_workspace_bytes(cin, cout) if (k == 3 and stride == 1) else \
        lib.cfb_conv2d_pertap_workspace_bytes(n, h, w, cin, cout, k, stride)
    ws = torch.empty(int(need), dtype=torch.uint8, device=DEV)
    xd = x.permute(0, 2, 3, 1).contiguous().to(DEV)
    out = torch.empty((n, ho, wo, cout), device=DEV)
    wd, bd = wt.to(DEV), b.to(DEV)
    sd = scale.contiguous().to(DEV) if scale is not None else None
    hd = shift.contiguous().to(DEV) if shift is not None else None
    rd = res.permute(0, 2, 3, 1).contiguous().to(DEV) if res is not None else None
    _lib.check(lib.cfb_debug_arcface_conv(_lib.ptr(xd), _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(out), n, h, w, cin, cout, k, stride,
                                          _lib.ptr(sd), _lib.ptr(hd), act, float(slope), _lib.ptr(rd), _lib.ptr(ws), ws.numel(),
                                          _stream()), 'cfb_debug_arcface_conv')
    torch.cuda.synchronize()
    return out.permute(0, 3, 1, 2)


def _data(n, cin, cout, h, w, k, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = 0.1 * torch.randn(cout, generator=g)
    return g, x, wt, b


@pytest.mark.parametrize('h,w,cin,cout', [(64, 64, 64, 64), (16, 16, 256, 256), (8, 8, 512, 512), (13, 21, 128, 64)])
def test_halo_affine_only_transform_and_prelu(h, w, cin, cout):
    """bn0 -> conv1 -> PReLU: the per-(image, channel) affine without activation inside the image, zero padding outside it
    (not a weight fold), the PReLU epilogue; 8 x 8 and 13 x 21 maps run as ragged tiles."""
    g, x, wt, b = _data(2, cin, cout, h, w, 3, h * cin)
    sc = 0.5 + torch.rand(2, cin, generator=g)
    sh = 0.3 * torch.randn(2, cin, generator=g)
    ref = F.prelu(F.conv2d(x * sc[:, :, None, None] + sh[:, :, None, None], wt, b, 1, 1), torch.tensor([0.21]))
    print('affine+prelu', h, w, _bar(_conv(x, wt, b, 1, sc, sh, 5, 0.21), ref))
    ref = F.conv2d(x * sc[:, :, None, None] + sh[:, :, None, None], wt, b, 1, 1)          # affine only, no activation
    _bar(_conv(x, wt, b, 1, sc, sh), ref)


@pytest.mark.parametrize('h,w,cin,cout', [(64, 64, 64, 64), (8, 8, 512, 512), (11, 9, 128, 128)])
def test_halo_residual_prelu(h, w, cin, cout):
    g, x, wt, b = _data(3, cin, cout, h, w, 3, h + cin)
    r = torch.randn(3, cout, h, w, generator=g)
    ref = F.prelu(F.conv2d(x, wt, b, 1, 1) + r, torch.tensor([0.13]))
    print('halo residual+prelu', h, w, _bar(_conv(x, wt, b, 1, act=5, slope=0.13, res=r), ref))


@pytest.mark.parametrize('h,w,cin,cout,k', [(64, 64, 64, 128, 3), (32, 32, 128, 256, 3), (16, 16, 256, 512, 3),
                                            (16, 16, 256, 512, 1), (15, 17, 64, 64, 3)])
def test_pertap_stride2_residual_prelu(h, w, cin, cout, k):
    """conv2 3x3 stride 2 + residual + PReLU and the 1x1 stride-2 downsample on the per-tap engine; layer4's 8 x 8 output is
    a ragged tile (64 of 128 pixels)."""
    g, x, wt, b = _data(2, cin, cout, h, w, k, h * cout + k)
    ref = F.conv2d(x, wt, b, 2, k // 2)
    r = torch.randn(ref.shape, generator=g)
    out = _conv(x, wt, b, 2, act=5, slope=0.27, res=r)
    print('pertap s2 residual+prelu', h, w, k, _bar(out, F.prelu(ref + r, torch.tensor([0.27]))))
    _bar(_conv(x, wt, b, 2), ref)


def test_conv_form_errors():
    g, x, wt, b = _data(1, 64, 64, 16, 16, 3, 1)
    with pytest.raises(RuntimeError):          # the input affine is built for 3x3 stride 1 only
        _conv(x, wt, b, 2, torch.ones(1, 64), torch.zeros(1, 64))
    with pytest.raises(RuntimeError):          # activation must be none or PReLU
        _conv(x, wt, b, 1, act=1)


def _net(layers=(2, 2, 2, 2), seed=1):
    net = cb.ResNetArcFace('IRBlock', layers, use_se=False)
    net.load_state_dict(A.random_arcface_state_dict(layers, seed=seed), strict=True)
    return net.to(DEV).eval()


def _check_emb(emb, ref, what):
    emb = emb.cpu()
    err = float((emb - ref).abs().max())
    cos = float(F.cosine_similarity(emb, ref, dim=1).min())
    print(f'{what}: max-abs {err:.3e} (|ref|max {float(ref.abs().max()):.3f}), min cosine {cos:.8f}')
    assert err <= EMB_BAR * max(1.0, float(ref.abs().max())) and cos >= 0.99999
    return err


@pytest.mark.parametrize('B', [1, 3, 32])
def test_forward_against_golden(B):
    x, ref = G.inputs()[:B], torch.from_numpy(np.load(os.path.join(GOLDEN, 'arcface.npz'))['emb'][:B])
    _check_emb(_net()(x.to(DEV)), ref, f'forward B={B}')


def test_forward_other_layers_against_oracle():
    layers = (1, 2, 3, 1)
    sd = A.random_arcface_state_dict(layers, seed=5)
    x = 0.5 * torch.randn(5, 1, 128, 128, generator=torch.Generator().manual_seed(2))
    _check_emb(_net(layers, 5)(x.to(DEV)), AO.arcface_forward(sd, x, layers), 'forward layers (1,2,3,1)')


def _faces(n):
    f = np.load(os.path.join(GOLDEN, 'faces.npz'))['faces']
    g = np.random.default_rng(4)
    extra = g.integers(0, 256, size=(max(0, n - len(f)), 512, 512, 3), dtype=np.uint8)
    return torch.from_numpy(np.concatenate([f, extra])[:n]).to(DEV)


def _unfused_input(faces):
    """The caller's steps as separate fp32 device passes: img2tensor(face / 255.), normalize(0.5, 0.5), gray_resize_for_identity."""
    x = (faces.double() / 255.).float().flip(-1).permute(0, 3, 1, 2).contiguous()
    x = (x - 0.5) / 0.5
    gray = (0.2989 * x[:, 0, :, :] + 0.5870 * x[:, 1, :, :] + 0.1140 * x[:, 2, :, :]).unsqueeze(1)
    return F.interpolate(gray, (128, 128), mode='bilinear', align_corners=False)


def test_forward_u8_bit_equal_to_the_unfused_chain_and_batch_invariant():
    net, faces = _net(), _faces(7)
    x = _unfused_input(faces)
    assert torch.equal(x.cpu(), AO.gray_resize_for_identity(AO.faces_to_input(faces.cpu())))
    e8 = net.forward_u8(faces)
    assert torch.equal(e8, net(x))
    for i in range(7):                                               # batch invariance
        assert torch.equal(net.forward_u8(faces[i:i + 1]), e8[i:i + 1])
    assert torch.equal(net.forward_u8(faces[2:5]), e8[2:5])
    for _ in range(3):                                               # repeated runs
        assert torch.equal(net.forward_u8(faces), e8)
    _check_emb(e8, AO.arcface_forward(A.random_arcface_state_dict(seed=1), x.cpu()), 'forward_u8 B=7')


def test_identity_similarity_single_and_sweep():
    net, faces = _net(), _faces(3)
    g = torch.Generator(device=DEV).manual_seed(3)
    noisy = (faces.int() + torch.randint(-20, 21, faces.shape, generator=g, device=DEV, dtype=torch.int32)).clamp(0, 255).byte()
    sim = cb.identity_similarity(net, faces, noisy)
    want = F.cosine_similarity(net.forward_u8(noisy), net.forward_u8(faces), dim=-1)
    assert sim.shape == (3,) and torch.equal(sim, want)
    assert torch.equal(cb.identity_similarity(net, faces, faces), F.cosine_similarity(*(net.forward_u8(faces),) * 2, dim=-1))
    # a real sweep: CodeFormer at K weights, scored in chunks that straddle the inputs and the candidates
    cf = cb.CodeFormer().to(DEV).eval()
    cf.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    ws = [0.0, 0.5, 1.0]
    sweep = cf.forward_u8_sweep(faces, ws)
    sims = cb.identity_similarity(net, faces, sweep, max_batch=4)
    e_in = net.forward_u8(faces)
    assert sims.shape == (3, 3)
    for k in range(3):
        assert torch.equal(sims[:, k], F.cosine_similarity(net.forward_u8(sweep[:, k].contiguous()), e_in, dim=-1))
    print('sweep similarities', sims.cpu().numpy())


def test_strict_load_and_errors():
    Sd = A.random_arcface_state_dict(seed=2)
    net = cb.ResNetArcFace(layers=[2, 2, 2, 2], use_se=False)
    net.load_state_dict(Sd, strict=True)
    bad = dict(Sd)
    bad['fc5.weight'] = torch.zeros(512, 100)
    with pytest.raises(RuntimeError):
        net.load_state_dict(bad, strict=True)
    net = net.to(DEV)
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 1, 128, 128))                            # CPU input
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 1, 112, 112, device=DEV))                # wrong shape
    with pytest.raises(RuntimeError):
        net.forward_u8(torch.zeros(1, 256, 256, 3, dtype=torch.uint8, device=DEV))
    with pytest.raises(RuntimeError):
        net.forward_u8(torch.zeros(1, 512, 512, 3, dtype=torch.uint8))   # CPU faces
    cpu_net = cb.ResNetArcFace(layers=[2, 2, 2, 2], use_se=False)
    with pytest.raises(RuntimeError):                                # parameters on the CPU, input on the GPU
        cpu_net(torch.zeros(1, 1, 128, 128, device=DEV))
    with pytest.raises(NotImplementedError):
        cb.ResNetArcFace('IRBlock', [2, 2, 2, 2], use_se=True)
    with pytest.raises(RuntimeError):
        net.train()
    assert net(torch.zeros(0, 1, 128, 128, device=DEV)).shape == (0, 512)
    with pytest.raises(RuntimeError):
        cb.identity_similarity(net, _faces(2), _faces(3))
