"""-m gpu: the encoder alone (VQAutoEncoder.encoder / CodeFormer.encoder), the latent codes of uint8 faces with the fused mirror
(latent_codes_u8, generate_latent_gt) and the code-prediction scores of CodeFormer's stage 2 (code_scores)."""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import codeformer_b200 as cb
from codeformer_b200 import _lib
from codeformer_b200 import spec as S
from oracle.plumbing_oracle import face_to_input
from tests.latent_restate import cross_entropy_f64, feat_mse_f64, script_latent_gt
from tests.util import faces_input, golden, maxabs

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
TOL_LAT = 2e-4          # the VQAE / CodeFormer latent bar of test_gpu_e2e.py


def _vq(seed=2):
    v = cb.VQAutoEncoder(512, 64, [1, 2, 2, 4, 4, 8], 'nearest', 2, [16], 1024).cuda().eval()
    v.load_state_dict(S.random_state_dict(S.vqae_spec(), seed), strict=True)
    return v


@pytest.fixture(scope='module')
def vq():
    return _vq()


@pytest.fixture(scope='module')
def cf():
    net = cb.CodeFormer().cuda().eval()
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    return net


def _faces(n, seed=0):
    """n uint8 [512,512,3] BGR faces: the committed faces, shifted and with a little noise so that no two are equal."""
    base = golden('faces.npz')['faces'][..., ::-1]
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        f = np.roll(base[i % base.shape[0]], 9 * i, axis=1).astype(np.int16) + rng.integers(-3, 4, (512, 512, 3))
        out.append(np.clip(f, 0, 255).astype(np.uint8))
    return np.stack(out)


def _chain(faces):
    """img2tensor(img / 255., bgr2rgb=True, float32=True) + normalize(0.5, 0.5) of uint8 BGR faces, on the device."""
    return torch.from_numpy(face_to_input(faces)).cuda()


def _codes(v, x):
    return v.quantize(v.encoder(x))[2]['min_encoding_indices'].view(-1, 16, 16)


# ---- the encoder alone ----------------------------------------------------------------------------------------------------
def test_vq_encoder_vs_oracle():
    """Golden VQAE weights on a committed face, and a seeded net on a seeded input, against the oracle's Encoder.forward."""
    from oracle import codeformer_oracle as O
    for seed, x in ((2, faces_input(slice(0, 1))), (5, torch.randn(1, 3, 512, 512, generator=torch.Generator().manual_seed(5)).clamp_(-1, 1))):
        v = _vq(seed)
        z = v.encoder(x.cuda())
        rz, _ = O.encoder_forward(S.random_state_dict(S.vqae_spec(), seed), x)
        assert z.shape == (1, 256, 16, 16) and z.dtype == torch.float32
        err = maxabs(z.cpu(), rz)
        print(f'seed {seed}: encoder max-abs {err:.3e} (|z|max {float(rz.abs().max()):.2f})')
        assert err < TOL_LAT


def test_vq_encoder_is_the_forward_latent(vq):
    """encoder(x) is, bit for bit, the latent VQAutoEncoder.forward quantizes (its last encoder stage, read through capture)."""
    x = faces_input(slice(0, 3)).cuda()
    last = len(vq.encoder.blocks) - 1
    vq(x[:1])                                             # the handle exists once a forward ran
    cap = torch.empty(3 * 16 * 16 * 256, device='cuda')
    vq.capture(f'enc.{last}', cap)
    try:
        _, _, st = vq(x, return_min_encodings=False)
        torch.cuda.synchronize()
    finally:
        vq.capture(f'enc.{last}', None)
    z = vq.encoder(x)
    assert torch.equal(z.permute(0, 2, 3, 1).reshape(-1), cap)
    # quantize(encoder(x)) runs VectorQuantizer.forward's fused kernel, the forward its distance GEMM + argmin: the two may
    # part only on near-ties, within the distance error of the two fp32 kernels (1e-5 of |z|^2 + |e|^2, about 100 fp32 ulps)
    idx = vq.quantize(z)[2]['min_encoding_indices']
    ref = st['min_encoding_indices']
    diff = (idx != ref).view(-1).nonzero().view(-1)
    print(f'quantize(encoder(x)) vs forward: {diff.numel()} of {idx.numel()} tokens differ')
    if diff.numel():
        zt = z.permute(0, 2, 3, 1).reshape(-1, 256).double()[diff]
        E = vq.quantize.embedding.weight.detach().double()
        a, b = E[idx.view(-1)[diff]], E[ref.view(-1)[diff]]
        d_a, d_b = ((zt - a) ** 2).sum(1), ((zt - b) ** 2).sum(1)
        scale = (zt ** 2).sum(1) + torch.maximum((a ** 2).sum(1), (b ** 2).sum(1))
        assert bool(((d_a - d_b).abs() <= 1e-5 * scale).all()), 'the selections differ beyond a near-tie'


def test_codeformer_encoder_is_lq_feat(cf):
    x = faces_input(slice(0, 2)).cuda()
    _, lq = cf(x, w=0, code_only=True)
    z = cf.encoder(x)
    assert torch.equal(z, lq)
    assert torch.equal(cf.encoder(x[1:2]), lq[1:2])


def test_encoder_surface(vq):
    with pytest.raises(TypeError):
        vq.encoder(faces_input(slice(0, 1)).cuda(), True)          # generate_latent_gt.py:55 fails in the reference too
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        vq.encoder(torch.zeros(1, 3, 512, 512))
    with pytest.raises(RuntimeError, match='expected input'):
        vq.encoder(torch.zeros(1, 3, 256, 256, device='cuda'))
    with pytest.raises(RuntimeError, match='parameter holder'):
        vq.encoder.blocks[0](torch.zeros(1, 3, 8, 8, device='cuda'))
    assert vq.encoder(torch.zeros(0, 3, 512, 512, device='cuda')).shape == (0, 256, 16, 16)


# ---- latent codes of uint8 faces ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B', [1, 3, 32])
def test_latent_codes_u8_equal_fp32_chain(vq, B):
    """Equal to quantize(encoder(fp32 chain)) bit for bit; hflip to the same chain on img[:, ::-1].  At odd B the mirror of face
    0 is image B of the 2B-image pass, so orig and mirror meet inside a batch."""
    faces = _faces(B, seed=B)
    dev = torch.from_numpy(faces).cuda()
    plain = vq.latent_codes_u8(dev)
    orig, flip = vq.latent_codes_u8(dev, hflip=True)
    assert plain.shape == orig.shape == flip.shape == (B, 16, 16) and plain.dtype == torch.int64
    ref_o = torch.cat([_codes(vq, _chain(faces[i:i + 4])) for i in range(0, B, 4)])
    ref_f = torch.cat([_codes(vq, _chain(np.ascontiguousarray(faces[i:i + 4, :, ::-1]))) for i in range(0, B, 4)])
    assert torch.equal(plain, ref_o) and torch.equal(orig, ref_o)
    assert torch.equal(flip, ref_f)
    assert not torch.equal(orig, flip)


def test_latent_codes_u8_batch_invariant(vq):
    faces = torch.from_numpy(_faces(32, seed=7)).cuda()
    o32, f32 = vq.latent_codes_u8(faces, hflip=True)
    for lo, hi in ((0, 1), (5, 6), (31, 32), (3, 7), (10, 27)):
        o, f = vq.latent_codes_u8(faces[lo:hi], hflip=True)
        assert torch.equal(o, o32[lo:hi]) and torch.equal(f, f32[lo:hi])


def test_latent_codes_u8_errors(vq):
    with pytest.raises(RuntimeError, match='CUDA uint8'):
        vq.latent_codes_u8(torch.zeros(1, 512, 512, 3, dtype=torch.uint8))
    with pytest.raises(RuntimeError, match='CUDA uint8'):
        vq.latent_codes_u8(torch.zeros(1, 512, 512, 3, device='cuda'))
    with pytest.raises(RuntimeError, match='HWC BGR'):
        vq.latent_codes_u8(torch.zeros(1, 3, 512, 512, dtype=torch.uint8, device='cuda'))
    e = torch.zeros(0, 512, 512, 3, dtype=torch.uint8, device='cuda')
    o, f = vq.latent_codes_u8(e, hflip=True)
    assert o.shape == f.shape == (0, 16, 16)
    lib = _lib.load()
    with pytest.raises(RuntimeError, match='mirror'):
        _lib.check(lib.cfb_latent_codes_u8(vq._net, ctypes.c_void_p(1), ctypes.c_void_p(1), None, 2, 3, None, 0, None),
                   'cfb_latent_codes_u8')


def test_generate_latent_gt(vq, tmp_path):
    faces = _faces(6, seed=11)
    names = ['00012', '00003', 'b', 'a', '00100', 'z_last']
    ref = script_latent_gt(list(faces), names, vq, 'cuda')
    got = cb.generate_latent_gt(list(faces), names, vq)
    assert list(got) == ['orig', 'hflip'] and list(got['orig']) == names and list(got['hflip']) == names
    for kind in ('orig', 'hflip'):
        for n in names:
            a = got[kind][n]
            assert isinstance(a, np.ndarray) and a.dtype == np.int64 and a.shape == (16, 16)
            assert np.array_equal(a, ref[kind][n]), (kind, n)
    for mb in (1, 4):
        g2 = cb.generate_latent_gt(faces, names, vq, max_batch=mb)
        assert all(np.array_equal(g2[k][n], got[k][n]) for k in got for n in names)
    g3 = cb.generate_latent_gt(torch.from_numpy(faces).cuda(), names, vq, max_batch=4)
    assert all(np.array_equal(g3[k][n], got[k][n]) for k in got for n in names)
    path = tmp_path / 'latent_gt_code1024.pth'
    torch.save(got, path)
    back = torch.load(path, weights_only=False)
    assert list(back) == ['orig', 'hflip'] and list(back['hflip']) == names
    assert all(np.array_equal(back[k][n], got[k][n]) and back[k][n].dtype == np.int64 for k in got for n in names)
    with pytest.raises(ValueError, match='names'):
        cb.generate_latent_gt(faces, names[:-1], vq)


# ---- code-prediction scores -----------------------------------------------------------------------------------------------
def test_code_scores_vs_float64(cf):
    B = 3
    faces = _faces(B, seed=21)
    x = _chain(faces)
    gt = cf.latent_codes_u8(torch.from_numpy(_faces(B, seed=30)).cuda())   # the faces' own VQGAN codes: an imperfect target
    r = cb.code_scores(cf, x, gt)
    logits, lq = cf(x, w=0, code_only=True)
    g = gt.view(B, 256)
    ce64 = F.cross_entropy(logits.double().permute(0, 2, 1), g, reduction='none').mean(1)
    assert r['cross_entropy'].dtype == torch.float64 and r['cross_entropy'].shape == (B,)
    assert bool(((r['cross_entropy'] - ce64).abs() <= 1e-12 * ce64.abs()).all())
    assert torch.allclose(cross_entropy_f64(logits, g), ce64, rtol=1e-12, atol=0)
    # torch's fp32 value, within its own error bound: per token, a few fp32 ulps of max|logit| + log K
    ce32 = F.cross_entropy(logits.permute(0, 2, 1), g, reduction='none').mean(1).double()
    bound = 64 * 2.0 ** -24 * (float(logits.abs().max()) + math.log(1024))
    print(f'cross-entropy {r["cross_entropy"].tolist()} fp32 torch off by {float((ce32 - r["cross_entropy"]).abs().max()):.3e} '
          f'(bound {bound:.3e})')
    assert float((ce32 - r['cross_entropy']).abs().max()) <= bound
    assert torch.equal(r['top_idx'], logits.argmax(2))
    assert torch.equal(r['accuracy'], (r['top_idx'] == g).double().mean(1))
    mse64 = feat_mse_f64(cf.quantize.embedding.weight.detach(), g, lq)
    assert bool(((r['feat_mse'] - mse64).abs() <= 1e-12 * mse64).all())
    # the two stage-2 losses of codeformer_idx_model.py:100-115 on this batch, as the docstring builds them
    l_ce = F.cross_entropy(logits.permute(0, 2, 1), g) * 0.5
    l_feat = torch.mean((cf.quantize.get_codebook_feat(g, shape=[B, 16, 16, 256]) - lq) ** 2)
    assert abs(float(0.5 * r['cross_entropy'].mean()) - float(l_ce)) <= 0.5 * bound
    assert abs(float(r['feat_mse'].mean()) - float(l_feat)) <= 1e-5 * float(l_feat)


def test_code_scores_u8_equals_fp32_chain_and_batch_invariant(cf):
    faces = _faces(32, seed=41)
    dev = torch.from_numpy(faces).cuda()
    gt = cf.latent_codes_u8(torch.from_numpy(_faces(32, seed=42)).cuda())
    r8 = cb.code_scores(cf, dev, gt)
    r32 = cb.code_scores(cf, _chain(faces), gt.view(32, 256))
    keys = ('cross_entropy', 'accuracy', 'feat_mse', 'top_idx')
    assert all(torch.equal(r8[k], r32[k]) for k in keys)
    for mb in (1, 4):
        rm = cb.code_scores(cf, dev[:9], gt[:9], max_batch=mb)
        assert all(torch.equal(rm[k], r8[k][:9]) for k in keys)
    for lo, hi in ((0, 1), (7, 10), (31, 32)):
        rb = cb.code_scores(cf, dev[lo:hi], gt[lo:hi])
        assert all(torch.equal(rb[k], r8[k][lo:hi]) for k in keys)


def test_code_scores_own_codes_give_accuracy_one(cf):
    dev = torch.from_numpy(_faces(3, seed=51)).cuda()
    own = cb.code_scores(cf, dev, torch.zeros(3, 256, dtype=torch.int64, device='cuda'))['top_idx']
    r = cb.code_scores(cf, dev, own)
    assert torch.equal(r['accuracy'], torch.ones(3, dtype=torch.float64, device='cuda'))
    assert bool((r['cross_entropy'] >= 0).all())


def test_code_scores_kernel_nan_and_bad_index():
    """cfb_code_scores on crafted logits: a NaN logit makes that face's cross-entropy NaN (no fault, the other face is
    untouched); an index outside [0, K) is never read and is reported as RuntimeError."""
    lib = _lib.load()
    gen = torch.Generator().manual_seed(3)
    B, T, K, D = 2, 256, 1024, 256
    logits = (3 * torch.randn(B, T, K, generator=gen)).cuda()
    E = torch.randn(K, D, generator=gen).cuda()
    feat = torch.randn(B, T, D, generator=gen).cuda()
    gt = torch.randint(0, K, (B, T), generator=gen).cuda()
    top = logits.argmax(2)

    def run(lg, g):
        out = torch.empty(B, 3, dtype=torch.float64, device='cuda')
        _lib.check(lib.cfb_code_scores(_lib.ptr(lg), _lib.ptr(top), _lib.ptr(g), _lib.ptr(feat), _lib.ptr(E), B, T, K, D,
                                       _lib.ptr(out), _lib.stream()), 'cfb_code_scores')
        torch.cuda.synchronize()
        return out
    clean = run(logits, gt)
    assert torch.allclose(clean[:, 0], cross_entropy_f64(logits, gt), rtol=1e-12, atol=0)
    assert torch.equal(clean[:, 1], (top == gt).double().sum(1))
    nan = logits.clone()
    nan[1, 17, 400] = float('nan')
    r = run(nan, gt)
    cb.check_async_status()
    assert math.isnan(float(r[1, 0])) and torch.equal(r[0], clean[0]) and torch.equal(r[1, 1:], clean[1, 1:])
    for bad in (K, -1, 1 << 40):
        g = gt.clone()
        g[1, 200] = bad
        r = run(logits, g)
        with pytest.raises(RuntimeError, match='out of range'):
            cb.check_async_status()
        assert torch.equal(r[0], clean[0]) and bool(torch.isnan(r[1]).all())
    cb.check_async_status()                             # the report cleared the condition


def test_code_scores_bad_index_and_errors(cf):
    dev = torch.from_numpy(_faces(2, seed=61)).cuda()
    gt = torch.zeros(2, 16, 16, dtype=torch.int64, device='cuda')
    gt[1, 3, 4] = 1024
    with pytest.raises(RuntimeError, match='out of range'):
        cb.code_scores(cf, dev, gt)
    gt[1, 3, 4] = 0
    assert torch.isfinite(cb.code_scores(cf, dev, gt)['cross_entropy']).all()
    with pytest.raises(RuntimeError, match='CUDA'):
        cb.code_scores(cf, dev.cpu(), gt)
    with pytest.raises(RuntimeError, match='CUDA'):
        cb.code_scores(cf, dev, gt.cpu())
    with pytest.raises(RuntimeError, match='int64'):
        cb.code_scores(cf, dev, gt.int())
    with pytest.raises(RuntimeError, match='gt_codes must be'):
        cb.code_scores(cf, dev, gt[:1])
    with pytest.raises(RuntimeError, match='uint8 or float32'):
        cb.code_scores(cf, dev.double(), gt)
    with pytest.raises(RuntimeError, match='HWC BGR'):
        cb.code_scores(cf, dev[:, :256], gt)
    with pytest.raises(RuntimeError, match='CodeFormer'):
        cb.code_scores(_vq(), dev, gt)
