"""-m gpu: CodeFormer / VQAutoEncoder ``set_precision('fp16')`` -- the generator and Fuse_sft_block convs on the single-pass
fp16 variants of the 128-wide, channel-major and per-tap tiles.

Unit convs go through cfb_debug_conv_tc_prec (it reports the tile it launched) and are compared with the float64 emulation of
tests/fp16_emul.py (operands rounded as the kernel rounds them).  Networks are compared with the reference golden vectors
against twice the error the float64 emulation of the whole fp16 mode makes there (tests/golden/codeformer_fp16.npz, written by
tools/gen_codeformer_fp16_golden.py), and with the same module in fp32 mode: logits, lq_feat and the code indices must be
bit-identical, because the encoder and the Transformer stay split."""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import codeformer_b200 as cb
from codeformer_b200 import _lib
from codeformer_b200 import spec as S
from tests import fp16_emul as E
from tests.test_gpu_wide_tiles import assert_gn_partials, plane_bytes
from tests.util import faces_input, golden, maxabs

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

SFT_W = 0.5
TILE_CM = -64
# (N, Cin, Cout, H, mode, operand, cin1, residual, sft, out planes, GroupNorm partials, LeakyReLU, ksize, tile)
# operand: 'gnsilu' / 'split' = fused transform with GroupNorm-affine + SiLU / plain; 'planes' = raw operand planes.
# cin1 > 0: channels [cin1, Cin) come from a second tensor (Fuse_sft_block's torch.cat).  Every form the fp16 forward launches.
CASES = [
    (2, 256, 256, 32, 0, 'gnsilu', 0, True, False, False, True, False, 3, 128),      # generator ResBlock conv2, CPG 8
    (1, 128, 128, 32, 0, 'gnsilu', 0, False, False, False, True, False, 3, 128),     # CPG 4
    (1, 512, 512, 16, 0, 'gnsilu', 0, True, False, True, True, False, 3, 128),       # CPG 16, planes for an Upsample
    (1, 256, 512, 16, 0, 'split', 0, False, False, False, True, False, 3, 128),      # generator conv_in on the code features
    (1, 512, 256, 32, 0, 'gnsilu', 256, False, False, False, True, False, 3, 128),   # Fuse encode_enc.conv1 on the concat
    (1, 512, 512, 16, 2, 'planes', 0, False, False, True, True, False, 3, 128),      # Upsample, CPG 16
    (2, 128, 128, 32, 2, 'planes', 0, False, False, True, True, False, 3, 128),      # Upsample, CPG 4
    (1, 256, 256, 32, 0, 'planes', 0, False, False, True, False, True, 3, 128),      # Fuse scale.0 / shift.0 (LeakyReLU)
    (1, 128, 128, 32, 0, 'planes', 0, False, False, False, False, False, 3, 128),    # Fuse scale.2
    (1, 256, 256, 32, 0, 'planes', 0, False, True, True, True, False, 3, 128),       # Fuse shift.2 (SFT), CPG 8
    (2, 128, 64, 32, 0, 'gnsilu', 0, True, False, False, True, False, 3, TILE_CM),   # 512^2 ResBlock, CPG 2
    (1, 128, 64, 32, 0, 'gnsilu', 64, False, False, False, True, False, 3, TILE_CM), # Fuse 512 encode_enc.conv1
    (1, 64, 64, 32, 0, 'planes', 0, False, False, True, False, True, 3, TILE_CM),    # Fuse 512 scale.0
    (1, 64, 64, 32, 0, 'planes', 0, False, True, True, True, False, 3, TILE_CM),     # Fuse 512 shift.2 (SFT), CPG 2
    (1, 512, 256, 32, 0, 'planes', 0, False, False, False, False, False, 1, 64),     # ResBlock conv_out 1x1
    (2, 128, 64, 32, 0, 'planes', 0, False, False, False, False, False, 1, 64),      # 1x1 to 64 channels
]


def _rand(*shape, seed, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def case_inputs(case):
    """NHWC x, OIHW w, bias, per-(n, cin) scale / shift, NHWC residual, SFT dec / scale (None where the case has none)."""
    N, Cin, Cout, H, mode, operand, cin1, resid, sft, planes, gn, act, k, tile = case
    Ho = 2 * H if mode == 2 else H
    x = _rand(N, H, H, Cin, seed=11) * 2 + 0.5
    w = _rand(Cout, Cin, k, k, seed=12, scale=1.0 / math.sqrt(Cin * k * k))
    b = _rand(Cout, seed=13, scale=0.1)
    sc = 1 + 0.1 * _rand(N, Cin, seed=14) if operand == 'gnsilu' else None
    sh = 0.1 * _rand(N, Cin, seed=15) if operand == 'gnsilu' else None
    r = _rand(N, Ho, Ho, Cout, seed=16) if resid else None
    dec = _rand(N, Ho, Ho, Cout, seed=17) if sft else None
    scl = 0.5 * _rand(N, Ho, Ho, Cout, seed=18) if sft else None
    return x, w, b, sc, sh, r, dec, scl


def emulated(case):
    """float64 single-pass model of the case (NHWC): the conv input and the weights rounded as the kernel rounds them.
    -> (reference, slack).  The kernel forms a GroupNorm-affine + SiLU operand in fp32 (SiLU to about 2^-21); where that
    value lies within its fp32 error of an fp16 rounding boundary, the kernel may take the neighbouring fp16 value.  slack
    bounds, per output, what those flips can move: sum over the receptive field of |w_hi| x the gap of the two candidates."""
    N, Cin, Cout, H, mode, operand, cin1, resid, sft, planes, gn, act, k, tile = case
    x, w, b, sc, sh, r, dec, scl = [None if t is None else t.double() for t in case_inputs(case)]
    slack = torch.zeros(1, dtype=torch.float64)
    if operand == 'gnsilu':
        assert mode == 0 and k == 3
        xs, s = x * sc[:, None, None, :], sh[:, None, None, :]
        x = F.silu(xs + s)
        delta = 2.0 ** -20 * x.abs() + 2.0 ** -22 * (xs.abs() + s.abs())
        gap = (E.fp16_round(x + delta) - E.fp16_round(x - delta)).abs().permute(0, 3, 1, 2)
        slack = F.conv2d(gap, E.weight_hi(w).abs(), padding=1).permute(0, 2, 3, 1)
    x = x.permute(0, 3, 1, 2)
    v = E.conv3x3(x, w, up=mode == 2) if k == 3 else F.conv2d(E.fp16_round(x), E.weight_hi(w))
    v = (v + b.view(1, -1, 1, 1)).permute(0, 2, 3, 1)
    if resid:
        v = v + r
    if act:
        v = F.leaky_relu(v, 0.2)
    if sft:
        v = dec + SFT_W * (dec * scl + v)
        slack = slack * SFT_W
    return v, slack


def run_case(case, precision, legacy=False):
    """-> (out NHWC, planes or None, GroupNorm partials or None, tile) of cfb_debug_conv_tc_prec (legacy: cfb_debug_conv_tc)"""
    N, Cin, Cout, H, mode, operand, cin1, resid, sft, planes, gn, act, k, tile = case
    lib = _lib.load()
    x, w, b, sc, sh, r, dec, scl = [None if t is None else t.cuda() for t in case_inputs(case)]
    Ho = 2 * H if mode == 2 else H
    x0 = x[..., :cin1].contiguous() if cin1 else x
    x1 = x[..., cin1:].contiguous() if cin1 else None
    out = torch.empty(N, Ho, Ho, Cout, device='cuda')
    pl = torch.zeros(2 * plane_bytes(N, Ho, Cout), dtype=torch.uint8, device='cuda') if planes else None
    gp = torch.zeros(N * Ho * Ho // 128 * 4 * 64, device='cuda') if gn else None
    wsb = lib.cfb_conv2d_workspace_bytes(N, H, H, Cin, Cout, k, mode)
    ws = torch.empty(int(wsb), dtype=torch.uint8, device='cuda')
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    tn = ctypes.c_int32(0)
    args = (_lib.ptr(x0), _lib.ptr(x1), cin1, _lib.ptr(w), _lib.ptr(b), _lib.ptr(out), N, H, H, Cin, Cout, mode,
            0 if operand == 'planes' else 1, _lib.ptr(sc), _lib.ptr(sh), 1 if operand == 'gnsilu' else 0, _lib.ptr(r),
            _lib.ptr(dec), _lib.ptr(scl), SFT_W, _lib.ptr(pl), _lib.ptr(gp), _lib.ptr(ws), wsb, st, ctypes.byref(tn))
    if legacy:
        _lib.check(lib.cfb_debug_conv_tc(*args), 'cfb_debug_conv_tc')
    else:
        _lib.check(lib.cfb_debug_conv_tc_prec(*args, k, 1 if act else 0, precision), 'cfb_debug_conv_tc_prec')
    torch.cuda.synchronize()
    cb.check_async_status()
    return out.cpu(), (None if pl is None else pl.cpu().numpy()), (None if gp is None else gp.cpu().numpy()), tn.value


def _case_id(c):
    N, Cin, Cout, H, mode, operand, cin1, resid, sft, planes, gn, act, k, tile = c
    return '-'.join([('up' if mode == 2 else 'same') + str(k), f'cin{Cin}', f'cout{Cout}', operand] + (['cat'] if cin1 else []) +
                    (['res'] if resid else []) + (['lrelu'] if act else []) + (['sft'] if sft else []) +
                    (['pl'] if planes else []) + (['gn'] if gn else []))


@pytest.mark.parametrize('case', CASES, ids=[_case_id(c) for c in CASES])
def test_fp16_conv_matches_emulation(case):
    """fp16 within 2e-5 max|ref| of the emulation on the expected tile; its planes and GroupNorm partials describe its own
    output; precision 0 of the new entry point is the existing one bit for bit; and the two precisions differ."""
    N, Cin, Cout, H, mode, operand, cin1, resid, sft, planes, gn, act, k, tile = case
    out, pl, gp, tn = run_case(case, 1)
    assert tn == tile, f'launched tile {tn}, expected {tile}'
    ref, slack = emulated(case)
    dev = (out.double() - ref).abs()
    err, excess = float(dev.max()), float((dev - slack).max())
    print(f'{_case_id(case)}: fp16 vs emulation max-abs {err:.3e}, beyond the operand-flip slack {excess:.3e} '
          f'(slack max {float(slack.max()):.2e}, |ref|max {float(ref.abs().max()):.3f})')
    assert excess <= 2e-5 * float(ref.abs().max())
    o = out.numpy()
    if planes:
        nb = plane_bytes(N, o.shape[1], Cout)
        hi = pl[:nb].view(np.float16)[:o.size].astype(np.float32)
        assert np.array_equal(hi, o.reshape(-1).astype(np.float16).astype(np.float32)), 'hi plane = fp16(out)'
    if gn:
        assert_gn_partials(gp, o, N, Cout)
    split = run_case(case, 0)
    assert split[3] == tile
    if not act and k == 3:
        legacy = run_case(case, 0, legacy=True)
        assert torch.equal(split[0], legacy[0]), 'precision 0 is cfb_debug_conv_tc'
        if planes:
            assert np.array_equal(split[1], legacy[1])
        if gn:
            assert np.array_equal(split[2], legacy[2])
    assert not torch.equal(out, split[0]), 'fp16 mode must take effect'


def test_fp16_conv_rejects_forms_it_is_not_built_for():
    """A 3x3 conv on the per-tap engine (24 x 24: no halo tiles), which the fp16 decoder never launches, is an error in fp16
    mode -- never a silent split run; a bad precision value is an error too."""
    case = (1, 64, 64, 24, 0, 'planes', 0, False, False, False, False, False, 3, 64)
    assert run_case(case, 0)[3] == 64
    with pytest.raises(RuntimeError, match='single-pass'):
        run_case(case, 1)
    with pytest.raises(RuntimeError, match='precision'):
        run_case(CASES[0], 2)


# ---------------------------------------------------------------------------------------------------------------- networks
@pytest.fixture(scope='module')
def emul():
    return golden('codeformer_fp16.npz')


@pytest.fixture(scope='module')
def net_main():
    net = cb.CodeFormer().cuda().eval()
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    return net


def _both(net, x, **kw):
    """(fp32 result, fp16 result) of one module, switching in between; the module is left in fp32 mode"""
    a = [t.clone() for t in net.set_precision('fp32')(x, **kw)]
    h = [t.clone() for t in net.set_precision('fp16')(x, **kw)]
    net.set_precision('fp32')
    torch.cuda.synchronize()
    cb.check_async_status()
    return a, h


def _check_codeformer(net, x, ref_out, err_emul, tag, **kw):
    (a_out, a_log, a_lq), (h_out, h_log, h_lq) = _both(net, x, **kw)
    assert torch.equal(h_log, a_log) and torch.equal(h_lq, a_lq), f'{tag}: logits / lq_feat must not depend on the precision'
    assert torch.equal(h_log.argmax(2), a_log.argmax(2))
    sub = h_out if ref_out.shape[-1] == 512 else h_out[..., ::4, ::4]
    err = maxabs(sub.cpu(), ref_out)
    print(f'{tag}: fp16 out vs reference max-abs {err:.3e}, emulation {err_emul:.3e}; fp32 mode '
          f'{maxabs((a_out if ref_out.shape[-1] == 512 else a_out[..., ::4, ::4]).cpu(), ref_out):.3e}')
    assert err <= 2 * err_emul + 1e-4
    assert not torch.equal(h_out, a_out)
    return a_out, h_out


def test_codeformer_fp16_main_config_vs_reference_golden(net_main, emul):
    g = golden('codeformer_main.npz')
    x = faces_input(slice(0, 1)).cuda()
    _, h = _check_codeformer(net_main, x, g['out'], float(emul['main_err']), 'main', w=0.5, adain=True)
    assert np.array_equal(net_main.set_precision('fp16')(x, w=0.5, adain=True)[1].argmax(2).cpu().numpy(), g['top_idx'])
    net_main.set_precision('fp32')


def test_codeformer_fp16_variants_vs_reference_golden(net_main, emul):
    g = golden('codeformer_variants.npz')
    x = faces_input(slice(1, 2)).cuda()
    _check_codeformer(net_main, x, g['w0_out'], float(emul['w0_err']), 'w0', w=0, adain=True)      # fusion skipped
    net3 = cb.CodeFormer(connect_list=['32', '64', '128']).cuda().eval()
    net3.load_state_dict(S.random_state_dict(S.codeformer_spec(connect_list=('32', '64', '128')), 3))
    _check_codeformer(net3, x, g['c3_out'], float(emul['c3_err']), 'c3', w=0.7, adain=True)


def test_vqautoencoder_fp16_vs_reference_golden(emul):
    g = golden('vqae.npz')
    v = cb.VQAutoEncoder(512, 64, [1, 2, 2, 4, 4, 8], 'nearest', 2, [16], 1024).cuda().eval()
    v.load_state_dict(S.random_state_dict(S.vqae_spec(), 2), strict=True)
    x = faces_input(slice(0, 1)).cuda()
    a_out, a_loss, a_st = v(x)
    a_out = a_out.clone()
    assert v.set_precision('fp16') is v and v.precision == 'fp16'
    h_out, h_loss, h_st = v(x)
    torch.cuda.synchronize()
    cb.check_async_status()
    assert torch.equal(h_st['min_encoding_indices'], a_st['min_encoding_indices']) and float(h_loss) == float(a_loss)
    assert np.array_equal(h_st['min_encoding_indices'].cpu().numpy(), g['idx'])
    err, err_emul = maxabs(h_out[..., ::4, ::4].cpu(), g['out']), float(emul['vqae_err'])
    print(f'vqae: fp16 out vs reference max-abs {err:.3e}, emulation {err_emul:.3e}')
    assert err <= 2 * err_emul + 1e-4 and not torch.equal(h_out, a_out)


def test_fp16_batch_invariance_and_determinism(net_main):
    g = torch.Generator().manual_seed(5)
    x = torch.randn(32, 3, 512, 512, generator=g).clamp_(-1, 1)
    x[:4] = faces_input(slice(0, 4))
    xd = x.cuda()
    net_main.set_precision('fp16')
    try:
        o1, l1, q1 = [t.clone() for t in net_main(xd, w=0.5, adain=True)]
        o2, l2, q2 = net_main(xd, w=0.5, adain=True)
        assert torch.equal(o1, o2) and torch.equal(l1, l2) and torch.equal(q1, q2), 'deterministic'
        o_single = net_main(xd[:1], w=0.5, adain=True)[0]            # one face: the CUDA-graph path
        assert torch.equal(o_single[0], o1[0]), 'the face at B=32 equals the single face'
        o5 = net_main(xd[:5], w=0.5, adain=True)[0]                  # eager path
        assert torch.equal(o5, o1[:5])
        assert bool(torch.isfinite(o1).all())
    finally:
        net_main.set_precision('fp32')


def test_fp16_restore_faces_matches_forward_and_the_emulation(net_main, emul):
    """restore_faces in fp16 mode: the fused uint8 plumbing around the fp16 forward (equal to the forward's own output through
    the reference plumbing up to rounding ties), and as far from the emulated fp16 face as the emulation is from the fp32
    reference face.  The two fp16 results are not equal within one level everywhere: where an fp32 operand lies within its
    rounding error of an fp16 rounding boundary the kernel and the float64 emulation round it apart, and some 60 convs carry
    those one-ulp differences into the image."""
    from oracle import plumbing_oracle as P
    bgr = np.ascontiguousarray(golden('faces.npz')['faces'][:1][..., ::-1])
    net_main.set_precision('fp16')
    try:
        got = net_main.restore_faces([bgr[0]], w=0.5, adain=True, on_error='raise')[0]
        fwd = net_main(torch.from_numpy(P.face_to_input(bgr)).cuda(), w=0.5, adain=True)[0]
    finally:
        net_main.set_precision('fp32')
    d_fwd = np.abs(got.astype(np.int32) - P.output_to_face(fwd.cpu().numpy())[0].astype(np.int32))
    assert d_fwd.max() <= 1 and (d_fwd > 0).mean() < 1e-4
    emu = emul['u8_face0'][0].astype(np.int32)
    ref = P.output_to_face(golden('codeformer_main.npz')['out'])[0].astype(np.int32)
    d, d_emu = np.abs(got.astype(np.int32) - emu), np.abs(emu - ref)
    print(f'restore_faces fp16 vs emulation: {(d > 0).mean():.3%} differ, {(d > 1).mean():.3%} by more than one level, max '
          f'{d.max()}; emulation vs fp32 reference: {(d_emu > 0).mean():.3%} differ, max {d_emu.max()}')
    assert got.shape == emu.shape and d.max() <= d_emu.max() + 1 and (d > 1).mean() < 1e-2
    assert (d > 0).mean() <= 1.5 * (d_emu > 0).mean()
    fp32 = net_main.restore_faces([bgr[0]], w=0.5, adain=True, on_error='raise')[0]
    assert not np.array_equal(fp32, got)


def test_precision_switching_restores_fp32_bits_on_every_path(net_main):
    """fp32 -> fp16 -> fp32 on the CUDA-graph path (B <= 4), the eager path, forward_u8 and forward_host."""
    x1 = faces_input(slice(0, 1)).cuda()
    x5 = faces_input(slice(0, 4)).repeat(2, 1, 1, 1)[:5].contiguous().cuda()
    u8 = torch.from_numpy(np.ascontiguousarray(golden('faces.npz')['faces'][:2][..., ::-1])).cuda()
    assert net_main.precision == 'fp32'
    runs = lambda: [net_main(x1, w=0.5, adain=True)[0].clone(), net_main(x5, w=0.5, adain=True)[0].clone(),   # noqa: E731
                    net_main.forward_u8(u8, w=0.5, adain=True).clone(), net_main.forward_host(x1.cpu(), w=0.5, adain=True)[0]]
    a = runs()
    net_main.set_precision('fp16')
    h = runs()
    net_main.set_precision('fp32')
    b = runs()
    for i, (ai, hi, bi) in enumerate(zip(a, h, b)):
        assert torch.equal(ai.cpu(), bi.cpu()), f'path {i}: fp32 bits must come back after fp16'
        assert not torch.equal(ai.cpu(), hi.cpu()), f'path {i}: fp16 must take effect'
    assert torch.equal(h[0][0].cpu(), h[1][0].cpu()), 'graph and eager paths agree in fp16 too'
    assert torch.equal(h[3][0], h[0][0].cpu())


def test_precision_survives_load_state_dict_and_to():
    sd = S.random_state_dict(S.codeformer_spec(), 1)
    net = cb.CodeFormer().cuda().eval()
    net.load_state_dict(sd)
    x = faces_input(slice(2, 3)).cuda()
    h = net.set_precision('fp16')(x, w=0.5, adain=True)[0].clone()
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 7))
    net.load_state_dict(sd)                                           # re-prepared twice
    net = net.to('cuda')
    assert net.precision == 'fp16' and torch.equal(net(x, w=0.5, adain=True)[0], h)


def test_precision_errors(net_main):
    with pytest.raises(ValueError):
        net_main.set_precision('bf16')
    with pytest.raises(ValueError):
        net_main.set_precision(1)
    assert net_main.precision == 'fp32'
    lib = _lib.load()
    net_main(faces_input(slice(0, 1)).cuda(), w=0.5, adain=True)      # the handle exists
    with pytest.raises(RuntimeError, match='precision'):
        _lib.check(lib.cfb_net_set_precision(net_main._net, 2), 'cfb_net_set_precision')
    net = cb.CodeFormer().cuda().eval()
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1))
    net.set_engine('f32')
    net.set_precision('fp16')
    for b in (1, 5):                                                  # CUDA-graph path and eager path
        with pytest.raises(RuntimeError, match='fp16'):
            net(faces_input(slice(0, 1)).repeat(b, 1, 1, 1).cuda(), w=0.5, adain=True)
    cb.check_async_status()
