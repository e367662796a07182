"""-m gpu: the Transformer stage of CodeFormer -- LayerNorm in both forms, both attention cores and the code lookup -- against
float64, at the rows where such kernels go wrong: large row means (r = |mean| / std up to 1e4), a massive channel,
near-constant and constant rows, peaked / flat / tied / offset softmax rows, probabilities below fp16's normal range, v with a
DC offset, NaN / -inf logits; and the stage end to end on both engines with DC-offset tokens and peaked attention.

Bars follow tests/test_gpu_groupnorm_range.py: the kernel's error against float64 is at most k x the error of float32 torch
(on the CPU) against float64, plus a floor.  Errors are in units of |gamma| (LayerNorm outputs), of the float64 standard
deviation of v per image and head (attention outputs) or of the float64 per-row standard deviation (token rows), never
relative to a maximum, which a DC offset would inflate.  tests/test_transformer_numerics_cpu.py shows that the LayerNorm bar
accepts the kernel's arithmetic and rejects a one-pass variance, a wrong eps and a lost float4 by at least 4x.  The wgmma
attention core is held to the split-fp16 error model of tests/test_gpu_split_error_model.py instead."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import codeformer_b200 as cb
from codeformer_b200 import _lib
from codeformer_b200 import spec as S
from tests import gpu_util as G
from tests import layernorm_emul as L
from tests import split_emul as SE
from tests.test_gpu_split_error_model import TAU, _attention_ref, plane_bytes

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

C = L.C
T = 3 * 256                     # three images of 256 tokens: every image's position rows are checked
POS_ROWS = 256


def _planes(buf, n):
    """uint8 plane buffer (hi | lo, each plane_bytes(n)) -> (hi, lo) fp16 numpy arrays of n values"""
    a = buf.cpu().numpy()
    nb = plane_bytes(n)
    return a[:nb].view(np.float16)[:n], a[nb:2 * nb].view(np.float16)[:n]


def _layer_norm(x, gamma, beta, pos, planes, want_y=True, want_y2=True):
    """one call of cfb_layer_norm (planes False) or cfb_debug_layer_norm_planes -> (y, y2): fp32 [T, C] numpy arrays, or
    (hi, lo) pairs of fp16 arrays; None where not requested"""
    lib = _lib.load()
    rows = x.shape[0]
    xd, gd, bd, pd = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, gamma, beta, pos))
    if planes:
        mk = lambda: torch.zeros(2 * plane_bytes(rows * C), dtype=torch.uint8, device='cuda')   # noqa: E731
    else:
        mk = lambda: torch.full((rows, C), float('nan'), device='cuda')                          # noqa: E731
    y = mk() if want_y else None
    y2 = mk() if want_y2 else None
    fn = lib.cfb_debug_layer_norm_planes if planes else lib.cfb_layer_norm
    _lib.check(fn(_lib.ptr(xd), _lib.ptr(gd), _lib.ptr(bd), _lib.ptr(y), _lib.ptr(y2), _lib.ptr(pd), POS_ROWS, rows, C,
                  G.stream()), 'layer_norm')
    torch.cuda.synchronize()
    if planes:
        return tuple(None if t is None else _planes(t, rows * C) for t in (y, y2))
    return tuple(None if t is None else t.cpu().numpy() for t in (y, y2))


def _pos(seed):
    return (0.5 * np.random.default_rng(seed).standard_normal((POS_ROWS, C))).astype(np.float32)


# ---- a. LayerNorm, both forms ----------------------------------------------------------------------------------------------------
def test_layer_norm_both_forms_vs_float64():
    """fp32 form (cfb_layer_norm, the f32 engine's) and operand-plane form (the forward's on the wgmma engine) on the row
    classes of tests/layernorm_emul.py; y2 = y + pos[t % 256].  Planes: hi == fp16(y) of the fp32 form and lo == fp16(y - hi),
    bit for bit, so the planes carry the fp32 form's accuracy to 2^-21 relative."""
    x, classes = L.row_classes(T, 1)
    gamma, beta = L.affine(2)
    pos = _pos(3)
    pos_t = np.tile(pos, (T // POS_ROWS, 1))
    y64, y32 = L.reference(x, gamma, beta)
    y2_64, y2_32 = y64 + pos_t.astype(np.float64), y32 + pos_t          # float32 torch adds pos in fp32
    cb.check_async_status()
    y, y2 = _layer_norm(x, gamma, beta, pos, planes=False)
    cb.check_async_status()                                            # the fp32 form never reports
    failures = []
    for n, (ek, et) in L.class_errors(y, y64, y32, gamma, classes).items():
        L.judge(f'fp32 form y   {n}', ek, et, failures)
    for n, (ek, et) in L.class_errors(y2, y2_64, y2_32, gamma, classes).items():
        L.judge(f'fp32 form y2  {n}', ek, et, failures)
    (hi, lo), (hi2, lo2) = _layer_norm(x, gamma, beta, pos, planes=True)
    cb.check_async_status()                                            # |y| < 65504: nothing to report
    for name, h, l, ref in (('y', hi, lo, y), ('y2', hi2, lo2, y2)):
        r = ref.reshape(-1)
        h16 = r.astype(np.float16)
        assert np.array_equal(h.view(np.uint16), h16.view(np.uint16)), f'{name}: hi plane != fp16 of the fp32 form'
        assert np.array_equal(l.view(np.uint16), (r - h16.astype(np.float32)).astype(np.float16).view(np.uint16)), \
            f'{name}: lo plane != fp16(y - hi)'
        err = np.abs(h.astype(np.float64) + l.astype(np.float64) - r)
        assert (err <= 2.0 ** -21 * np.abs(r) + 2.0 ** -24).all(), f'{name}: hi + lo off y by {err.max():.3e}'
        sel = np.zeros(T, bool)
        sel[classes['dc r=10000']] = True
        print(f'planes {name}: bit-exact hi / lo over {r.size} values ({int(sel.sum())} rows at r = 1e4)')
    assert not failures, '\n'.join(failures)


# ---- b. the fp16 range of the LayerNorm planes --------------------------------------------------------------------------------------
def test_layer_norm_planes_fp16_range_guard():
    """A LayerNorm output past 65504 cannot be an fp16 operand: the planes form reports it through the status word (an error
    that names fp16), for y and for y2 = y + pos alike; the fp32 form has no fp16 operand and does not report.  The report is
    cleared once raised."""
    x, _ = L.row_classes(T, 4)
    x = x[np.arange(T) % 8 == 0]                                       # benign rows only
    rows = x.shape[0]
    gamma, beta = L.affine(5)
    big = gamma.copy()
    big[37] = 4e4                                                      # |y| > 65504 where |normalised x| > 1.64
    y64, _ = L.reference(x, big, beta)
    assert 0 < (np.abs(y64) > 65504).any(1).sum() < rows
    pos = np.zeros((POS_ROWS, C), np.float32)
    cb.check_async_status()
    _layer_norm(x, big, beta, pos, planes=False)
    cb.check_async_status()
    _layer_norm(x, big, beta, pos, planes=True, want_y2=False)
    with pytest.raises(RuntimeError, match='fp16'):
        cb.check_async_status()
    cb.check_async_status()                                            # reported once, then cleared
    # y2 alone: |y| < 10 everywhere, pos moves channel 5 so that y2 straddles 65504 (about half of the rows above it)
    y64, _ = L.reference(x, gamma, beta)
    pos[:, 5] = np.float32(65504.0 - np.median(y64[:, 5]))
    y2 = y64[:, 5] + pos[0, 5]
    assert (y2 > 65504.1).any() and (y2 < 65503.9).any() and np.abs(y64).max() < 10
    _layer_norm(x, gamma, beta, pos, planes=True, want_y=False)
    with pytest.raises(RuntimeError, match='fp16'):
        cb.check_async_status()
    pos[:, 5] = 65000.0                                                # control: inside the range, no report
    _layer_norm(x, gamma, beta, pos, planes=True)
    cb.check_async_status()


IDX_GAIN = 6e4


def test_net_reports_layer_norm_overflow():
    """idx_pred_layer's LayerNorm weight x IDX_GAIN: its output (an fp16 operand of the logits linear on the wgmma engine)
    leaves the fp16 range.  The tc engine must raise an error naming fp16; the f32 engine has no fp16 operand there and must
    still pick the float64 oracle's codes (the gain scales the logits, not their order)."""
    from oracle import codeformer_oracle as O
    from tests.util import faces_input
    sd = S.random_state_dict(S.codeformer_spec(), 1)
    sd['idx_pred_layer.0.weight'] = sd['idx_pred_layer.0.weight'] * IDX_GAIN
    x = faces_input(slice(0, 1))
    col = {}
    l64, _ = O.codeformer_forward({k: v.double() for k, v in sd.items()}, x.double(), code_only=True, collect=col)
    n64 = F.layer_norm(col['ft.8'], (512,), sd['idx_pred_layer.0.weight'].double(), sd['idx_pred_layer.0.bias'].double())
    print(f'idx_norm output max {float(n64.abs().max()):.3e}')
    assert float(n64.abs().max()) > 2 * 65504
    net = cb.CodeFormer().cuda().eval()
    net.load_state_dict(sd)
    net.set_engine('tc')
    cb.check_async_status()
    raised = None
    try:
        net(x.cuda(), w=0.5, adain=False)
        torch.cuda.synchronize()
        cb.check_async_status()
    except RuntimeError as e:
        raised = str(e)
    if raised and 'not supported by the wgmma engine' in raised:
        pytest.skip('tc-only mode: some shapes are not on the tensor-core engine')
    print(f'tc: {raised}')
    assert raised is not None and 'fp16' in raised, 'a LayerNorm output past 65504 went into the fp16 planes silently'
    net.set_engine('f32')
    _, logits, _ = net(x.cuda(), w=0.5, adain=False)
    torch.cuda.synchronize()
    cb.check_async_status()
    e = float((logits.cpu().double() - l64).abs().max())
    top2 = l64.topk(2, dim=2).values
    sure = (top2[..., 0] - top2[..., 1]) > 100 * e
    same = logits.argmax(2).cpu() == l64.argmax(2)
    print(f'f32: logits err {e:.3e} (logits max {float(l64.abs().max()):.3e}); {int(sure.sum())} tokens compared')
    assert int(sure.sum()) > 128 and bool(same[sure].all())


# ---- c. both attention cores -------------------------------------------------------------------------------------------------------
N_IMG = 3
REGIMES = ('random', 'flat', 'peaked', 'tie', 'offset', 'dc_v', 'subnormal_p')


def attention_inputs(regime, heads, d, seed):
    """q, k, v [N_IMG, 256, heads * d] fp32 for one regime (per head):
    random: N(0, 1);  flat: q = 0 (out = mean of v);  peaked: each query is a multiple of one key, scores in about +-60 with
    a top-1 gap >= 20;  tie: the same with keys in identical pairs (each query's top score is an exact tie of two keys with
    different v);  offset: every score 500 + N(0, 5^2);  dc_v: v = 1e3 + N(0, 1);  subnormal_p: scores N(0, 4^2), so most
    probabilities of a row lie below 2^-14, the smallest normal fp16."""
    g = torch.Generator().manual_seed(seed)
    E = heads * d
    rn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)     # noqa: E731
    q, k, v = rn(N_IMG, 256, heads, d), rn(N_IMG, 256, heads, d), rn(N_IMG, 256, heads, d)
    if regime == 'flat':
        q.zero_()
    elif regime in ('peaked', 'tie'):
        k = k / k.norm(dim=-1, keepdim=True) * math.sqrt(d)                  # |k| = sqrt(d): score of its own query = alpha sqrt(d)
        if regime == 'tie':
            k[:, 1::2] = k[:, 0::2]
        alpha = 7.0 if d == 64 else 2.5
        pick = torch.stack([torch.randperm(256, generator=g) for _ in range(N_IMG * heads)]).view(N_IMG, heads, 256)
        if regime == 'tie':
            pick = pick // 2 * 2
        q = alpha * torch.gather(k, 1, pick.transpose(1, 2)[..., None].expand(-1, -1, -1, d))
    elif regime == 'offset':
        a = math.sqrt(500 * math.sqrt(d))
        q = 5.0 * q * math.sqrt(d / (d - 1))
        q[..., 0] = a
        k[..., 0] = a
    elif regime == 'dc_v':
        v = v + 1e3
    elif regime == 'subnormal_p':
        q, k = 2 * q, 2 * k
    return tuple(t.reshape(N_IMG, 256, E).float() for t in (q, k, v))


def _scores64(q, k, heads):
    n, t, E = q.shape
    d = E // heads
    qh, kh = (z.double().view(n, t, heads, d).transpose(1, 2) for z in (q, k))
    return qh @ kh.transpose(-1, -2) / math.sqrt(d)


def _check_regime(regime, q, k, heads):
    """the regime is what it claims, in float64"""
    s = _scores64(q, k, heads)
    p = torch.softmax(s, -1)
    top2 = s.topk(2, -1).values
    if regime == 'peaked':
        assert float((top2[..., 0] - top2[..., 1]).min()) >= 20 and float(s.abs().max()) <= 75
    elif regime == 'tie':
        assert bool((top2[..., 0] == top2[..., 1]).all()) and float(p.amax(-1).min()) > 0.49
    elif regime == 'offset':
        assert 480 < float(s.mean()) < 520 and 4 < float(s.std()) < 6
    elif regime == 'subnormal_p':
        assert float((p < 2.0 ** -14).double().mean()) > 0.5
    elif regime == 'flat':
        assert bool((s == 0).all())


def _v_unit(v, heads):
    """float64 standard deviation of v per image and head, broadcast to [n, 256, E]"""
    n, t, E = v.shape
    d = E // heads
    s = v.double().view(n, t, heads, d).std(dim=(1, 3), unbiased=False)
    return s[:, None, :, None].expand(n, t, heads, d).reshape(n, t, E)


def _torch32(q, k, v, heads):
    """float32 torch on the CPU (the reference's math backend): softmax(q k^T d^-1/2) v"""
    n, t, E = q.shape
    d = E // heads
    qh, kh, vh = (z.view(n, t, heads, d).transpose(1, 2) for z in (q, k, v))
    o = F.softmax(qh @ kh.transpose(-1, -2) * d ** -0.5, dim=-1) @ vh
    return o.transpose(1, 2).reshape(n, t, E)


# The CUDA-core core against float32 torch: it sums the 256 products of P v one after another with FMAs where torch's CPU GEMM
# blocks them, and computes exp with expf; ATT_K = 8 leaves that a 2x margin over the worst ratio measured on an H100 (see
# DESIGN.md section 4); ATT_FLOOR (in units of v's spread) covers the flat and tied rows, where torch is nearly exact.
ATT_K = 8.0
ATT_FLOOR = 4e-6
ATT_SHAPES = [(8, 64), (1, 512)]


@pytest.mark.parametrize('heads,d', ATT_SHAPES, ids=['transformer-8x64', 'attnblock-1x512'])
def test_attention_cores_in_hard_regimes(heads, d):
    """cfb_attention (f32 engine) and cfb_debug_bmm_tc (wgmma engine) in every regime of attention_inputs"""
    lib = _lib.load()
    E = heads * d
    failures = []
    for ri, regime in enumerate(REGIMES):
        q, k, v = attention_inputs(regime, heads, d, 100 + 10 * ri + heads)
        _check_regime(regime, q, k, heads)
        qd, kd, vd = q.cuda(), k.cuda(), v.cuda()
        ref, bound, floor = _attention_ref(qd, kd, vd, heads)
        unit = _v_unit(v, heads)
        e32 = float(((_torch32(q, k, v, heads).double() - ref.cpu()).abs() / unit).max())
        # CUDA-core core
        out = torch.full((N_IMG, 256, E), float('nan'), device='cuda')
        _lib.check(lib.cfb_attention(_lib.ptr(qd), _lib.ptr(kd), _lib.ptr(vd), _lib.ptr(out), N_IMG, 256, heads, d, E, E, E, E,
                                     d ** -0.5, G.stream()), 'cfb_attention')
        torch.cuda.synchronize()
        eg = float(((out.cpu().double() - ref.cpu()).abs() / unit).nan_to_num(float('inf')).max())
        L.judge(f'simt {heads}x{d} {regime}', eg, e32, failures, ATT_K, ATT_FLOOR)
        # wgmma core: the split-fp16 error model, and its output planes
        out = torch.full((N_IMG, 256, E), float('nan'), device='cuda')
        pl = torch.zeros(2 * plane_bytes(out.numel()), dtype=torch.uint8, device='cuda')
        wsb = lib.cfb_debug_bmm_tc_workspace_bytes(N_IMG, heads, d)
        ws = torch.empty(int(wsb), dtype=torch.uint8, device='cuda')
        _lib.check(lib.cfb_debug_bmm_tc(_lib.ptr(qd), _lib.ptr(kd), _lib.ptr(vd), _lib.ptr(out), _lib.ptr(pl), N_IMG, heads, d,
                                        _lib.ptr(ws), wsb, G.stream()), 'cfb_debug_bmm_tc')
        torch.cuda.synchronize()
        bar = SE.split_bar(out.double(), ref, bound, floor, TAU['random'])
        et = float(((out.double() - ref).abs() / unit.cuda()).nan_to_num(float('inf')).max())
        print(f'{"wgmma " + str(heads) + "x" + str(d) + " " + regime:44s} kernel {et:.3e}  torch32 {e32:.3e}  {bar}')
        if not bar.ok:
            failures.append(f'wgmma {regime}: {bar}')
        o = out.reshape(-1).cpu().numpy()
        hi, lo = _planes(pl, o.size)
        if not np.array_equal(hi.view(np.uint16), o.astype(np.float16).view(np.uint16)):
            failures.append(f'wgmma {regime}: hi plane != fp16(out)')
        if not (np.abs(hi.astype(np.float64) + lo.astype(np.float64) - o) <= 2.0 ** -21 * np.abs(o) + 2.0 ** -24).all():
            failures.append(f'wgmma {regime}: hi + lo != out to 2^-21')
    cb.check_async_status()
    assert not failures, '\n'.join(failures)


# ---- d. the code lookup ----------------------------------------------------------------------------------------------------------
LOOKUP_T = 8 * 3 + 5             # ragged: the last CTA has 5 of its 8 warps' tokens
LOOKUP_D = 256


def lookup_logits(K, seed):
    """[LOOKUP_T, K] logits: random rows, and rows 8..15 special -- exact ties inside one lane's stride (columns j, j + 32, read
    by one lane) and across lanes (first maximum in a higher lane than a later one, and in the last column), all -inf, all
    NaN, NaN at the maximum and elsewhere, NaN with -inf, +inf"""
    g = torch.Generator().manual_seed(seed)
    lg = torch.randn(LOOKUP_T, K, generator=g)
    nan, inf = float('nan'), float('inf')
    lg[8, [45, 45 + 32, 45 + 96]] = 9.0                      # one lane
    lg[9, [37, 70]] = 9.0                                     # lanes 5 and 6
    lg[10, [70, 101]] = 9.0                                   # lane 6 before lane 5
    lg[11, [K - 1, 3]] = 9.0                                  # the last column and an early one
    lg[12] = -inf
    lg[13] = nan
    m = int(lg[14].argmax())
    lg[14, [m, 0, K // 2]] = nan                              # NaN where the maximum was
    lg[15, ::2] = nan
    lg[15, 1::2] = -inf
    lg[16, K // 3] = inf
    return lg


@pytest.mark.parametrize('K', [1024, 512, 1000])
def test_code_lookup(K):
    """cfb_debug_code_lookup: idx = the first maximum of each row (torch.argmax) and quant = E[idx] bit for bit; NaN logits
    are skipped (a row's NaNs never win, unlike torch.argmax, which returns a NaN's position), a row with nothing but NaN and
    -inf gives index 0, always inside [0, K).  Nothing is written past row T."""
    lib = _lib.load()
    lg = lookup_logits(K, K)
    E = torch.randn(K, LOOKUP_D, generator=torch.Generator().manual_seed(K + 1))
    lgd, Ed = lg.cuda(), E.cuda()
    idx = torch.full((LOOKUP_T + 3,), -7, dtype=torch.int64, device='cuda')
    quant = torch.full((LOOKUP_T + 3, LOOKUP_D), -3.0, device='cuda')
    _lib.check(lib.cfb_debug_code_lookup(_lib.ptr(lgd), _lib.ptr(Ed), _lib.ptr(idx), _lib.ptr(quant), LOOKUP_T, K, LOOKUP_D,
                                         G.stream()), 'cfb_debug_code_lookup')
    torch.cuda.synchronize()
    idx, quant = idx.cpu(), quant.cpu()
    assert (idx[LOOKUP_T:] == -7).all() and (quant[LOOKUP_T:] == -3.0).all(), 'written past row T'
    idx, quant = idx[:LOOKUP_T], quant[:LOOKUP_T]
    assert int(idx.min()) >= 0 and int(idx.max()) < K
    assert torch.equal(quant, E[idx])
    expect = torch.where(torch.isnan(lg), torch.full_like(lg, -float('inf')), lg).argmax(1)   # first maximum, NaN skipped
    assert torch.equal(idx, expect), (idx, expect)
    clean = ~torch.isnan(lg).any(1)
    assert torch.equal(idx[clean], lg[clean].argmax(1))
    assert idx[8] == 45 and idx[9] == 37 and idx[10] == 70 and idx[11] == 3
    assert idx[12] == 0 and idx[13] == 0 and idx[15] == 0 and idx[16] == K // 3
    # only idx, only quant
    q2 = torch.zeros(LOOKUP_T, LOOKUP_D, device='cuda')
    _lib.check(lib.cfb_debug_code_lookup(_lib.ptr(lgd), _lib.ptr(Ed), None, _lib.ptr(q2), LOOKUP_T, K, LOOKUP_D, G.stream()),
               'cfb_debug_code_lookup')
    torch.cuda.synchronize()
    assert torch.equal(q2.cpu(), quant)


# ---- e. the stage end to end ---------------------------------------------------------------------------------------------------
DC_TOKENS = 300.0                # feat_emb.bias + DC_TOKENS (every channel): token rows at r ~ 200 .. 1600 at every LayerNorm
QK_GAIN, QK_LAYERS = 16.0, (0, 2, 4, 6, 8)    # q and k rows of in_proj_weight x QK_GAIN: scores x 256, peaked rows


def offset_state_dict():
    sd = S.random_state_dict(S.codeformer_spec(), 1)
    sd['feat_emb.bias'] = (sd['feat_emb.bias'] + DC_TOKENS).contiguous()
    for l in QK_LAYERS:
        w = sd[f'ft_layers.{l}.self_attn.in_proj_weight'].clone()
        w[:2 * C] *= QK_GAIN
        sd[f'ft_layers.{l}.self_attn.in_proj_weight'] = w
    return sd


def _token_rows(t):
    """oracle [256, B, E] -> [B * 256, E] (the net's token order)"""
    return t.permute(1, 0, 2).reshape(-1, t.shape[-1])


@pytest.fixture(scope='module')
def stage_oracles():
    from oracle import codeformer_oracle as O
    from tests.util import faces_input
    sd = offset_state_dict()
    x = faces_input(slice(0, 3))
    c64, c32 = {}, {}
    l64, lq64 = O.codeformer_forward({k: v.double() for k, v in sd.items()}, x.double(), code_only=True, collect=c64)
    l32, _ = O.codeformer_forward(sd, x, code_only=True, collect=c32)
    # the r of every LayerNorm input, and how peaked the attention rows are, in float64
    sd64 = {k: v.double() for k, v in sd.items()}
    B = x.shape[0]
    pos = sd64['position_emb'].unsqueeze(1).repeat(1, B, 1)
    q0 = F.linear(lq64.flatten(2).permute(2, 0, 1), sd64['feat_emb.weight'], sd64['feat_emb.bias'])
    ins = [q0] + [c64[f'ft.{l}'] for l in range(9)]
    rs, peaked = [], []
    for l, t in enumerate(ins):
        rs.append(float((t.mean(-1).abs() / t.std(-1, unbiased=False)).min()))
        if l < 9:
            p = f'ft_layers.{l}'
            t2 = F.layer_norm(t, (C,), sd64[p + '.norm1.weight'], sd64[p + '.norm1.bias']) + pos
            W, b = sd64[p + '.self_attn.in_proj_weight'], sd64[p + '.self_attn.in_proj_bias']
            q = F.linear(t2, W[:C], b[:C]).view(256, B * 8, 64).transpose(0, 1)
            k = F.linear(t2, W[C:2 * C], b[C:2 * C]).view(256, B * 8, 64).transpose(0, 1)
            peaked.append(float((torch.softmax(q @ k.transpose(1, 2) / 8, -1).amax(-1) >= 0.99).double().mean()))
    print('norm1 / idx_norm inputs, min r over tokens: ' + ' '.join(f'{r:.0f}' for r in rs))
    print('attention rows with max P >= 0.99: ' + ' '.join(f'{p:.2f}' for p in peaked))
    assert min(rs) >= 100, 'every LayerNorm input must have r >= 100'
    assert min(peaked[l] for l in QK_LAYERS) >= 0.5, 'most rows of the scaled layers must be peaked'
    return sd, x, c64, c32, l64, l32


# Stage bars: STAGE_FACTOR[engine] x the fp32 oracle's error + STAGE_FLOOR, in units of the float64 per-row standard deviation.
# f32: fp32 arithmetic in another order through 9 layers (4x), with a 2x margin.  tc: the split-fp16 operands carry ~21 bits
# against fp32's 24 (8x), and the peaked softmax rows amplify score errors alike in both (x1), with a 2x margin.  Both are
# set from that model; on an H100 80GB HBM3 (700 W) the worst stage was 1.1x the fp32 oracle's error (tc) and 0.9x (f32).
STAGE_FACTOR = {'f32': 8, 'tc': 16}
STAGE_FLOOR = 2e-5
# Codes of the offset stage: at most CODE_FACTOR x the float32 oracle's misses + CODE_SLACK tokens.
CODE_FACTOR, CODE_SLACK = 2, 8


@pytest.mark.parametrize('engine', ['tc', 'f32'])
def test_transformer_stage_vs_float64_oracle(stage_oracles, engine):
    """B = 3 (every image's position rows), DC-offset token rows and peaked attention: ft.0 .. ft.8 within the stage bar;
    quant (adain off) == E[argmax of the net's own logits] bit for bit; codes that differ from the float64 oracle's no more
    often than the float32 oracle's do (CODE_FACTOR, CODE_SLACK)."""
    sd, x, c64, c32, l64, l32 = stage_oracles
    net = cb.CodeFormer().cuda().eval()
    net.load_state_dict(sd)
    net.set_engine(engine)
    try:
        net(x.cuda(), w=0.5, adain=False)
    except RuntimeError as e:
        if engine == 'tc' and 'not supported by the wgmma engine' in str(e):
            pytest.skip('tc-only mode: some shapes are not on the tensor-core engine')
        raise
    keys = [f'ft.{l}' for l in range(9)]
    bufs = {k: torch.empty(x.shape[0] * 256 * C, device='cuda') for k in keys}
    bufs['quant'] = torch.empty(x.shape[0] * 256 * 256, device='cuda')
    for k, b in bufs.items():
        net.capture(k, b)
    _, logits, _ = net(x.cuda(), w=0.5, adain=False)
    torch.cuda.synchronize()
    for k in bufs:
        net.capture(k, None)
    cb.check_async_status()
    failures = []
    print(f'[{engine}] token rows, errors in units of the per-row standard deviation (gpu / fp32 oracle / bar):')
    for k in keys:
        ref = _token_rows(c64[k])
        unit = ref.std(-1, unbiased=False, keepdim=True)
        eg = float(((bufs[k].cpu().double().view_as(ref) - ref).abs() / unit).max())
        e32 = float(((_token_rows(c32[k]).double() - ref).abs() / unit).max())
        bar = STAGE_FACTOR[engine] * e32 + STAGE_FLOOR
        print(f'   {k:6s} {eg:.3e} {e32:.3e} {bar:.3e}' + ('' if eg <= bar else '  FAIL'))
        if not eg <= bar:
            failures.append(f'{k}: {eg:.3e} > {STAGE_FACTOR[engine]} x {e32:.3e} + {STAGE_FLOOR}')
    idx = logits.argmax(2).cpu()
    E = sd['quantize.embedding.weight']
    assert torch.equal(bufs['quant'].cpu().view(-1, 256), E[idx.view(-1)]), 'quant != E[argmax of the logits]'
    # The peaked rows amplify every rounding (fp32's included) into logits errors of ~5e-2 against top-2 gaps of ~0.2, so
    # hardly a token clears the 100 x error margin of test_code_indices_vs_float64_oracle; here the net must pick the float64
    # oracle's code about as often as the float32 oracle does.
    ref_idx = l64.argmax(2)
    e_log, e_log32 = float((logits.cpu().double() - l64).abs().max()), float((l32.double() - l64).abs().max())
    miss, miss32 = int((idx != ref_idx).sum()), int((l32.argmax(2) != ref_idx).sum())
    print(f'[{engine}] logits err {e_log:.3e} (fp32 oracle {e_log32:.3e}); codes differing from the float64 oracle: '
          f'{miss} of {idx.numel()} (fp32 oracle {miss32}; bar {CODE_FACTOR * miss32 + CODE_SLACK})')
    assert miss <= CODE_FACTOR * miss32 + CODE_SLACK, 'the net misses the float64 codes much more often than fp32 does'
    assert not failures, '\n'.join(failures)


@pytest.fixture(scope='module')
def clean_oracle():
    from oracle import codeformer_oracle as O
    from tests.util import faces_input
    sd = S.random_state_dict(S.codeformer_spec(), 1)
    x = faces_input(slice(0, 3))
    l64, _ = O.codeformer_forward({k: v.double() for k, v in sd.items()}, x.double(), code_only=True)
    return sd, x, l64


@pytest.mark.parametrize('engine', ['tc', 'f32'])
def test_code_indices_vs_float64_oracle(clean_oracle, engine):
    """B = 3 with the seeded weights: quant (adain off) == E[argmax of the net's own logits] bit for bit, and that argmax ==
    the float64 oracle's on every token whose float64 top-2 gap exceeds 100 x the measured logits error (near-ties counted
    and printed); at least 90 % of the tokens must clear that margin."""
    sd, x, l64 = clean_oracle
    net = cb.CodeFormer().cuda().eval()
    net.load_state_dict(sd)
    net.set_engine(engine)
    try:
        net(x.cuda(), w=0.5, adain=False)
    except RuntimeError as e:
        if engine == 'tc' and 'not supported by the wgmma engine' in str(e):
            pytest.skip('tc-only mode: some shapes are not on the tensor-core engine')
        raise
    quant = torch.empty(x.shape[0] * 256 * 256, device='cuda')
    net.capture('quant', quant)
    _, logits, _ = net(x.cuda(), w=0.5, adain=False)
    torch.cuda.synchronize()
    net.capture('quant', None)
    cb.check_async_status()
    idx = logits.argmax(2).cpu()
    E = sd['quantize.embedding.weight']
    assert torch.equal(quant.cpu().view(-1, 256), E[idx.view(-1)]), 'quant != E[argmax of the logits]'
    e_log = float((logits.cpu().double() - l64).abs().max())
    top2 = l64.topk(2, dim=2).values
    sure = (top2[..., 0] - top2[..., 1]) > 100 * e_log
    same = idx == l64.argmax(2)
    print(f'[{engine}] logits err {e_log:.3e}; tokens compared {int(sure.sum())}, near-ties skipped {int((~sure).sum())}, '
          f'differing codes among the compared {int((~same & sure).sum())}')
    assert bool(same[sure].all()), 'code indices must equal the float64 oracle where its top-2 gap exceeds 100 x the error'
    assert int(sure.sum()) >= 0.9 * idx.numel(), 'too few tokens clear the margin: the logits error is too large'
