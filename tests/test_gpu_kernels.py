"""-m gpu: every kernel of libcfb200 against the same op of the reference's math backend (torch CPU fp32),
called through the C ABI.  Tolerances are written next to each check; integer/index results are bit-exact."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from codeformer_b200 import _lib
from tests import gpu_util as G
from tests.util import golden, maxabs, vq_micro_inputs

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


def _rand(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


# (N, Cin, Cout, H, k, mode)  -- small instances of the conv families of SURVEY.md Appendix A
CONV_CASES = [
    (2, 64, 64, 32, 3, 0), (1, 128, 128, 32, 3, 0), (1, 256, 128, 16, 3, 0), (1, 512, 256, 16, 3, 0),
    (1, 512, 512, 16, 3, 0), (1, 256, 512, 16, 3, 0), (1, 64, 128, 32, 1, 0), (1, 512, 256, 16, 1, 0),
    (1, 512, 512, 16, 1, 0), (2, 64, 64, 32, 3, 1), (1, 128, 128, 16, 3, 1), (1, 256, 256, 16, 3, 1),
    (1, 128, 128, 16, 3, 2), (1, 512, 512, 8, 3, 2), (3, 64, 64, 20, 3, 0),
]


@pytest.mark.parametrize('engine', [1, 2])
@pytest.mark.parametrize('case', CONV_CASES)
def test_conv_matches_torch(case, engine):
    N, Cin, Cout, H, k, mode = case
    x = _rand(N, Cin, H, H, seed=1)
    w = _rand(Cout, Cin, k, k, seed=2, scale=1.0 / math.sqrt(Cin * k * k))
    b = _rand(Cout, seed=3, scale=0.1)
    if mode == 0:
        ref = F.conv2d(x, w, b, padding=k // 2)
    elif mode == 1:
        ref = F.conv2d(F.pad(x, (0, 1, 0, 1)), w, b, stride=2)              # vqgan_arch.py:122-126
    else:
        ref = F.conv2d(F.interpolate(x, scale_factor=2.0, mode='nearest'), w, b, padding=1)   # :134-138
    try:
        out = G.conv2d(x, w, b, mode=mode, engine=engine).cpu()
    except RuntimeError as e:
        if engine == 2 and 'not supported by the wgmma engine' in str(e):
            pytest.skip('shape not on the tensor-core engine')
        raise
    tol = 2e-5 if engine == 1 else 6e-5     # fp32 FMA vs split-fp16 (3 MMAs, ~22-bit operands)
    assert maxabs(out, ref) < tol * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize('engine', [1, 2])
def test_conv_fused_groupnorm_silu_residual_epilogues(engine):
    """GN(32,C,1e-6)+swish fused on load, bias+residual / LeakyReLU / GELU epilogues (ResBlock, Fuse_sft, FFN)."""
    N, C, H = 2, 128, 32
    x = _rand(N, C, H, H, seed=4) * 2 + 0.5
    gamma, beta = 1 + 0.1 * _rand(C, seed=5), 0.1 * _rand(C, seed=6)
    w = _rand(C, C, 3, 3, seed=7, scale=1 / math.sqrt(9 * C))
    b = _rand(C, seed=8, scale=0.1)
    res = _rand(N, C, H, H, seed=9)
    h = F.group_norm(x, 32, gamma, beta, eps=1e-6)
    ref = F.conv2d(h * torch.sigmoid(h), w, b, padding=1) + res
    xin, scale, shift = G.gn_coef(x, gamma, beta)
    # scale/shift reproduce group_norm
    hn = (xin * scale[:, None, None, :] + shift[:, None, None, :]).permute(0, 3, 1, 2).cpu()
    assert maxabs(hn, h) < 5e-6 * float(h.abs().max())
    try:
        out = G.conv2d(x, w, b, in_scale=scale, in_shift=shift, in_act=1, residual=res, engine=engine).cpu()
        assert maxabs(out, ref) < 6e-5 * float(ref.abs().max())
        out = G.conv2d(x, w, b, out_act=1, engine=engine).cpu()
        assert maxabs(out, F.leaky_relu(F.conv2d(x, w, b, padding=1), 0.2)) < 2e-4
        out = G.conv2d(x, w[:, :, 1:2, 1:2].contiguous(), b, out_act=2, engine=engine).cpu()
        assert maxabs(out, F.gelu(F.conv2d(x, w[:, :, 1:2, 1:2], b))) < 2e-4
    except RuntimeError as e:
        if engine == 2 and 'not supported by the wgmma engine' in str(e):
            pytest.skip('shape not on the tensor-core engine')
        raise


# (N, Cin, Cout, H, act): the in-kernel operand transform (fp32 activation -> GroupNorm affine (+SiLU) -> fp16 hi/lo inside the
# conv kernel) on both tile widths, with border tiles, several k-blocks and one-tile-high images
XF_CASES = [(2, 64, 64, 64, 1), (1, 128, 64, 32, 1), (2, 256, 128, 32, 1), (1, 64, 128, 32, 0), (2, 512, 512, 16, 1),
            (4, 128, 128, 16, 0)]


@pytest.mark.parametrize('case', XF_CASES)
def test_conv_in_kernel_operand_transform(case):
    """vqgan_arch.py:14-20,153-160: conv(swish(GroupNorm(x))) with the normalisation applied inside the wgmma conv kernel
    (engine 2) against torch CPU fp32 and against the fp32 CUDA-core engine.  x has a large per-channel offset so that a
    wrong affine or a missing zero-padding of the NORMALISED tensor is visible at the image border."""
    N, Cin, Cout, H, act = case
    x = _rand(N, Cin, H, H, seed=11) * 1.5 + _rand(1, Cin, 1, 1, seed=12) * 3
    gamma, beta = 1 + 0.2 * _rand(Cin, seed=13), 0.5 * _rand(Cin, seed=14)
    w = _rand(Cout, Cin, 3, 3, seed=15, scale=1 / math.sqrt(9 * Cin))
    b = _rand(Cout, seed=16, scale=0.1)
    res = _rand(N, Cout, H, H, seed=17)
    h = F.group_norm(x, 32, gamma, beta, eps=1e-6)
    ref = F.conv2d(h * torch.sigmoid(h) if act else h, w, b, padding=1) + res
    _, scale, shift = G.gn_coef(x, gamma, beta)
    out_tc = G.conv2d(x, w, b, in_scale=scale, in_shift=shift, in_act=act, residual=res, engine=2).cpu()
    out_f32 = G.conv2d(x, w, b, in_scale=scale, in_shift=shift, in_act=act, residual=res, engine=1).cpu()
    bound = 6e-5 * float(ref.abs().max())
    assert maxabs(out_tc, ref) < bound, 'tensor-core engine with the fused operand transform'
    assert maxabs(out_f32, ref) < bound
    from codeformer_b200 import _lib as L
    _lib_status = L.load().cfb_check_async_status()
    assert _lib_status == 0, L.load().cfb_last_error()


@pytest.mark.parametrize('C,H', [(64, 64), (128, 32), (256, 16), (512, 16), (512, 64)])
def test_group_norm_coef(C, H):
    x = _rand(2, C, H, H, seed=C + H) * 3 + 1
    gamma, beta = 1 + 0.1 * _rand(C, seed=1), 0.1 * _rand(C, seed=2)
    ref = F.group_norm(x, 32, gamma, beta, eps=1e-6)
    xin, scale, shift = G.gn_coef(x, gamma, beta)
    y = torch.empty_like(xin)
    lib = _lib.load()
    _lib.check(lib.cfb_affine_act(_lib.ptr(xin), _lib.ptr(scale), _lib.ptr(shift), _lib.ptr(y), 2, H * H, C, 1, G.stream()))
    assert maxabs(G.nchw(y).cpu(), ref * torch.sigmoid(ref)) < 1e-5 * float(ref.abs().max())


@pytest.mark.parametrize('heads,d', [(1, 512), (8, 64)])
def test_attention_core(heads, d):
    B, S = 2, 256
    E = heads * d
    q, k, v = _rand(B, S, E, seed=1), _rand(B, S, E, seed=2), _rand(B, S, E, seed=3)
    scale = d ** -0.5
    qh = q.view(B, S, heads, d).transpose(1, 2)
    kh = k.view(B, S, heads, d).transpose(1, 2)
    vh = v.view(B, S, heads, d).transpose(1, 2)
    ref = (F.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1) @ vh).transpose(1, 2).reshape(B, S, E)
    out = torch.empty(B, S, E, device='cuda')
    lib = _lib.load()
    qd, kd, vd = q.cuda(), k.cuda(), v.cuda()          # keep device copies alive across the call
    _lib.check(lib.cfb_attention(_lib.ptr(qd), _lib.ptr(kd), _lib.ptr(vd), _lib.ptr(out), B, S, heads, d,
                                 E, E, E, E, scale, G.stream()))
    assert maxabs(out.cpu(), ref) < 2e-5


def test_layer_norm_and_pos():
    T, C = 512, 512
    x = _rand(T, C, seed=1) * 2 + 0.3
    g, b, pos = 1 + 0.1 * _rand(C, seed=2), 0.1 * _rand(C, seed=3), 0.02 * _rand(256, C, seed=4)
    ref = F.layer_norm(x, (C,), g, b)
    y, y2 = torch.empty(T, C, device='cuda'), torch.empty(T, C, device='cuda')
    lib = _lib.load()
    xd, gd, bd, pd = x.cuda(), g.cuda(), b.cuda(), pos.cuda()
    _lib.check(lib.cfb_layer_norm(_lib.ptr(xd), _lib.ptr(gd), _lib.ptr(bd), _lib.ptr(y), _lib.ptr(y2),
                                  _lib.ptr(pd), 256, T, C, G.stream()))
    assert maxabs(y.cpu(), ref) < 5e-6
    assert maxabs(y2.cpu(), ref + pos.repeat(2, 1)) < 5e-6


def test_adain_and_layout():
    from oracle import codeformer_oracle as O
    c, s = _rand(2, 256, 16, 16, seed=1), _rand(2, 256, 16, 16, seed=2) * 3 + 1
    out = torch.empty(2, 16, 16, 256, device='cuda')
    lib = _lib.load()
    cd, sdv = G.nhwc(c), G.nhwc(s)
    _lib.check(lib.cfb_adain_nhwc(_lib.ptr(cd), _lib.ptr(sdv), _lib.ptr(out), 2, 256, 256, G.stream()))
    assert maxabs(G.nchw(out).cpu(), O.adain(c, s)) < 2e-5
    x = _rand(3, 40, 7, 9, seed=3).cuda()
    y = torch.empty(3, 63, 40, device='cuda')
    _lib.check(lib.cfb_nchw_to_nhwc(_lib.ptr(x), _lib.ptr(y), 3, 40, 63, G.stream()))
    assert torch.equal(y.view(3, 7, 9, 40), x.permute(0, 2, 3, 1))
    z = torch.empty_like(x)
    _lib.check(lib.cfb_nhwc_to_nchw(_lib.ptr(y), _lib.ptr(z), 3, 40, 63, G.stream()))
    assert torch.equal(z, x)


@pytest.mark.parametrize('case', ['B', 'C'])
def test_vq_nearest_config3_bit_exact_indices(case):
    """BASELINE.json configs[2]: 32x256x16x16 vs 1024 codes; indices bit-exact vs the reference golden."""
    import codeformer_b200 as cb
    g = golden('vq_micro.npz')
    E, z = vq_micro_inputs(case)
    vq = cb.VectorQuantizer(1024, 256, 0.25)
    vq.embedding.weight.data.copy_(E)
    vq = vq.cuda()
    zq, loss, st = vq(z.cuda())
    idx = st['min_encoding_indices'].cpu().numpy()
    assert idx.shape == (8192, 1) and idx.dtype == np.int64
    assert np.array_equal(idx, g[f'{case}_idx'])
    assert maxabs(zq[0].cpu(), g[f'{case}_zq_b0']) <= 2.4e-7 * 8       # reference's z+(zq-z) is <=2.4e-7 off E[idx]
    assert abs(float(loss) - float(g[f'{case}_loss'])) < 1e-5 * max(1.0, float(g[f'{case}_loss']))
    assert abs(float(st['perplexity']) - float(g[f'{case}_perplexity'])) < 1e-3 * float(g[f'{case}_perplexity'])
    assert abs(float(st['mean_distance']) - float(g[f'{case}_mean_distance'])) < 1e-4 * float(g[f'{case}_mean_distance'])
    oh = st['min_encodings']
    assert oh.shape == (8192, 1024) and float(oh.sum()) == 8192.0
    assert torch.equal(oh.argmax(1, keepdim=True).cpu(), torch.from_numpy(idx))
    # get_codebook_feat (vqgan_arch.py:72-84) reproduces E[idx] bit-for-bit
    feat = vq.get_codebook_feat(st['min_encoding_indices'], [32, 16, 16, 256]).cpu()
    assert torch.equal(feat, E[torch.from_numpy(idx[:, 0])].view(32, 16, 16, 256).permute(0, 3, 1, 2))


def test_vq_edge_cases():
    import codeformer_b200 as cb
    vq = cb.VectorQuantizer(1000, 256, 0.25)          # ragged: codes not a multiple of the 256-code tile
    vq.embedding.weight.data.normal_(generator=torch.Generator().manual_seed(1))
    vq = vq.cuda()
    z = _rand(1, 256, 3, 5, seed=2)                   # ragged token count (15 tokens, tile is 32)
    zq, loss, st = vq(z.cuda())
    E = vq.embedding.weight.detach().cpu()
    zf = z.permute(0, 2, 3, 1).reshape(-1, 256)
    d = (zf.double() ** 2).sum(1, keepdim=True) + (E.double() ** 2).sum(1) - 2 * zf.double() @ E.double().t()
    assert torch.equal(st['min_encoding_indices'].cpu()[:, 0], d.argmin(1))
    # duplicate codes => first index wins (torch.argmin semantics)
    vq.embedding.weight.data[7] = vq.embedding.weight.data[500]
    z2 = vq.embedding.weight.data[500].view(1, 256, 1, 1).clone()
    assert int(vq(z2)[2]['min_encoding_indices'][0, 0]) == 7
    # empty batch
    zq, loss, st = vq(torch.empty(0, 256, 16, 16, device='cuda'))
    assert zq.shape == (0, 256, 16, 16) and st['min_encoding_indices'].shape == (0, 1)


# (dim, codes, seed, one kernel): the config-3 shape and inputs (seed 0 = vq_micro_inputs('B')); codes % 128 == 64 inside the
# one kernel's limits; emb_dim 320 and 2048 codes outside them, where the module runs cfb_vq_nearest (the SIMT kernel at
# emb_dim 320, whose width the tensor-core operand prep does not take; stored dot products at 2048 codes).  The other seeds keep every token's two nearest codes >= 8e-4 apart in float64 (for E and -E), far above the
# rounding of the fp32 distances, so the float64 argmin is a fair check.
VQ_PATH_CASES = [(256, 1024, 0, 1), (256, 960, 3, 1), (320, 1024, 5, 0), (256, 2048, 3, 0)]


@pytest.mark.parametrize('dim,codes,seed,one_kernel', VQ_PATH_CASES)
def test_vq_fused_path_equals_the_unfused_one(dim, codes, seed, one_kernel):
    """VectorQuantizer.forward -- the ONE-kernel fused path (z tile in shared memory, argmin from the wgmma accumulators,
    statistics by the last CTA) with the prepared codebook where the shape allows it -- called twice, against the unfused path
    (stored dot products) and a float64 argmin: same indices, z_q and statistics; a changed embedding is picked up."""
    import codeformer_b200 as cb
    lib = _lib.load()
    g = torch.Generator().manual_seed(seed)
    E = torch.randn(codes, dim, generator=g)
    z = torch.randn(32, dim, 16, 16, generator=g)
    zf = z.permute(0, 2, 3, 1).reshape(-1, dim).double()
    vq = cb.VectorQuantizer(codes, dim, 0.25)
    vq.embedding.weight.data.copy_(E)
    vq = vq.cuda()
    zd = z.cuda()
    assert lib.cfb_vq_fast_supported(32, 16, 16, dim, codes) == one_kernel
    zq, loss, st = vq(zd)
    zq2, loss2, st2 = vq(zd)                                        # prepared codebook and workspace reused
    assert torch.equal(zq, zq2) and torch.equal(st['min_encoding_indices'], st2['min_encoding_indices']) and float(loss) == float(loss2)
    Ed = vq.embedding.weight.detach().contiguous()
    zq_o = torch.empty_like(zd)
    idx_o = torch.empty((8192, 1), dtype=torch.int64, device='cuda')
    stats_o = torch.empty(4, device='cuda')
    wsb = lib.cfb_vq_workspace_bytes(32, 256, dim, codes)
    ws = torch.empty(int(wsb), dtype=torch.uint8, device='cuda')
    _lib.check(lib.cfb_vq_nearest(_lib.ptr(zd), _lib.ptr(Ed), 32, 16, 16, dim, codes, 0.25, _lib.ptr(zq_o), _lib.ptr(idx_o),
                                  _lib.ptr(stats_o), None, _lib.ptr(ws), wsb, G.stream()), 'cfb_vq_nearest')
    torch.cuda.synchronize()
    assert torch.equal(st['min_encoding_indices'], idx_o) and torch.equal(zq, zq_o)
    assert abs(float(loss) - float(stats_o[0])) < 1e-6 * float(stats_o[0])
    assert abs(float(st['mean_distance']) - float(stats_o[2])) < 1e-5 * float(stats_o[2])
    d = (zf ** 2).sum(1, keepdim=True) + (E.double() ** 2).sum(1) - 2 * zf @ E.double().t()
    assert torch.equal(st['min_encoding_indices'].cpu()[:, 0], d.argmin(1))
    with torch.no_grad():
        vq.embedding.weight.mul_(-1.0)                              # in-place update bumps the version: re-prepared
    idx_neg = vq(zd)[2]['min_encoding_indices']
    assert not torch.equal(idx_neg, st['min_encoding_indices'])
    d = (zf ** 2).sum(1, keepdim=True) + (E.double() ** 2).sum(1) + 2 * zf @ E.double().t()
    assert torch.equal(idx_neg.cpu()[:, 0], d.argmin(1))
