"""-m gpu: every split-fp16 tensor-core form, through its entry point, against float64 at the error model of tests/split_emul.py.

Each output must satisfy |out - ref| <= TAU * B + floor: B = conv(|x|, |w|) of the operand the MMAs read (after the fused
transform and the padding), floor the term of subnormal lo (split_emul.bounds), plus the fp32 rounding of the epilogue.
tests/test_split_bar_cpu.py shows on the same CASES that this bar accepts the float64 emulation of the split (exact and with a
truncating accumulator) and rejects each way of losing lo products by at least 4x; mutants cannot be built on the GPU.

Every case runs with random unit-scale operands and, where the test controls the value that is split (raw split, operand
planes, GEN, per-tap), with sign-aligned operands (split_emul.aligned_operands), under which a lost lo product shows at full
size.  Tile kinds of the halo engine (cfb_debug_conv_tc_prec reports them): 128 and -64 (channel-major) by default, 64 with
CFB_TC_BN=64, which is read once per process, so the halo cases run in one subprocess per setting.  Each kind has a case of
more than 2 x 132 tiles, and images differ in scale, shift, residual and SFT weight, so consecutive tiles of one CTA belong to
different images (per-image SFT weights are built for raw-input convs only).  Also: the attention core on the engine (cfb_debug_bmm_tc) against float64 attention, and the magnitude
properties of the split (exact weight scaling, small activations, per-channel weight scales)."""
import collections
import ctypes
import math
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from codeformer_b200 import _lib
from tests import split_emul as S

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Measured on one H100 80GB HBM3 (700 W), DESIGN.md section 4: worst err / B 8.0e-7 with random operands, 1.2e-5 with
# sign-aligned ones, where every truncation of the fp32 accumulator (partial sums of 8 k-blocks) errs the same way.  The
# aligned bar is therefore too loose to see one lost 64-channel k-block of lo at Cin >= 256; the random bar sees it.
TAU = {'random': 1.5e-6, 'aligned': 2.2e-5}
EPI = 2.0 ** -22                     # fp32 rounding of the epilogue (bias, residual, SFT), relative to the terms it adds

Case = collections.namedtuple('Case', 'name entry g N H W Cin Cout operand cin1 resid sft planes extra')


def case(name, entry, g, N, H, W, Cin, Cout, operand='raw', cin1=0, resid=False, sft=False, planes=False, **extra):
    return Case(name, entry, g, N, H, W, Cin, Cout, operand, cin1, resid, sft, planes, extra)


# operand: 'raw' (the fp32 value is split as it is), 'gnsilu' (fused GroupNorm-affine + SiLU), 'affine' (affine only)
CASES = [
    # cfb_conv2d_nhwc, engine 2
    case('conv-k3', 'conv2d', S.SAME3, 1, 16, 16, 256, 128),
    case('conv-k3-gnsilu', 'conv2d', S.SAME3, 2, 16, 16, 512, 128, 'gnsilu'),
    case('conv-k1', 'conv2d', S.SAME1, 1, 16, 16, 512, 128),
    case('conv-down', 'conv2d', S.DOWN, 1, 32, 32, 128, 128),
    case('conv-up', 'conv2d', S.UP, 1, 16, 16, 256, 128),
    # cfb_debug_conv_tc_prec / _wv, precision 0 (halo engine; tile kinds)
    case('halo-big128-gnsilu', 'halo', S.SAME3, 3, 128, 128, 128, 128, 'gnsilu', resid=True),
    case('halo-bigcm-planes', 'halo', S.SAME3, 3, 128, 128, 64, 64, resid=True, sft=True),
    case('halo-split-512', 'halo', S.SAME3, 1, 16, 16, 512, 256, resid=True, planes=True, xform=1),
    case('halo-split-cat', 'halo', S.SAME3, 1, 16, 16, 256, 128, cin1=128, xform=1),
    case('halo-planes-512', 'halo', S.SAME3, 1, 16, 16, 512, 512, sft=True),
    case('halo-planes-cm', 'halo', S.SAME3, 2, 16, 16, 256, 64, planes=True),
    case('halo-up-planes', 'halo', S.UP, 1, 16, 16, 128, 128, planes=True),
    case('halo-up-planes-cm', 'halo', S.UP, 1, 16, 16, 256, 64, resid=True),
    case('halo-k1', 'halo', S.SAME1, 1, 16, 16, 512, 256, ksize=1),
    # cfb_conv2d_gen_nhwc
    case('gen-zero-ragged', 'gen', S.SAME3, 2, 21, 27, 64, 64, in_pitch=96, out_pitch=128, out_c0=32),
    case('gen-reflect', 'gen', S.Geometry(pad_mode=1), 1, 20, 20, 128, 64),
    case('gen-replicate-up', 'gen', S.Geometry(pad_mode=2, up=True), 1, 13, 17, 64, 64),
    case('gen-sub', 'gen', S.Geometry(sub=True), 1, 22, 26, 192, 64),
    # cfb_conv2d_pertap_nhwc / _slice_nhwc
    case('pertap-k1', 'pertap', S.SAME1, 2, 21, 27, 128, 64),
    case('pertap-k1-s2', 'pertap', S.Geometry(ksize=1, stride=2, pad=(0, 0, 0, 0)), 2, 21, 27, 64, 128),
    case('pertap-k3', 'pertap', S.SAME3, 1, 19, 23, 64, 64),
    case('pertap-k3-s2', 'pertap', S.Geometry(stride=2), 2, 21, 27, 128, 64),
    case('pertap-slice-k1', 'pertap_slice', S.SAME1, 1, 21, 27, 128, 64, out_pitch=192, out_c0=64),
    # cfb_debug_arcface_conv: the affine-only transform (zero padding outside the image)
    case('arcface-affine', 'arcface', S.SAME3, 2, 28, 28, 64, 64, 'affine'),
]
KINDS = ('random', 'aligned')


def kinds(c):
    return KINDS if c.operand == 'raw' else ('random',)


def _seed(c, kind):
    return 1000 * [x.name for x in CASES].index(c.name) + 7 * KINDS.index(kind)


def case_inputs(c, kind, H=None, W=None, N=None):
    """-> x (NCHW, the conv's input), w (OIHW), bias, per-(n, cin) scale / shift or None, residual (NCHW) or None,
    SFT dec / scale (NCHW) or None, per-image SFT weights or None.  H, W, N: a smaller spatial size (the CPU test)."""
    N, H, W = N or c.N, H or c.H, W or c.W
    s = _seed(c, kind)
    k = c.g.ksize
    if kind == 'aligned':
        x, w = S.aligned_operands((N, c.Cin, H, W), (c.Cout, c.Cin, k, k), s, 1.0, 1.0 / math.sqrt(c.Cin * k * k))
    else:
        x = S.random_operand((N, c.Cin, H, W), s) * (2 if c.operand != 'raw' else 1)
        w = S.random_operand((c.Cout, c.Cin, k, k), s + 1, 1.0 / math.sqrt(c.Cin * k * k))
    b = S.random_operand((c.Cout,), s + 2, 0.1)
    sc = sh = None
    if c.operand != 'raw':
        sc = 1 + 0.2 * S.random_operand((N, c.Cin), s + 3)
        sh = 0.3 * S.random_operand((N, c.Cin), s + 4)
    Ho, Wo = out_size(c, H, W)
    r = S.random_operand((N, c.Cout, Ho, Wo), s + 5) * torch.arange(1, N + 1).view(-1, 1, 1, 1) if c.resid else None
    dec = S.random_operand((N, c.Cout, Ho, Wo), s + 6) if c.sft else None
    scl = 0.5 * S.random_operand((N, c.Cout, Ho, Wo), s + 7) if c.sft else None
    wv = torch.linspace(0.25, 1.0, N) if c.sft else None
    return x, w, b, sc, sh, r, dec, scl, wv


def operand(c, x, sc, sh):
    """The fp32 operand the MMAs split (before padding): the raw input, or its fused transform."""
    if c.operand == 'raw':
        return x
    y = x.double() * sc.double()[:, :, None, None] + sh.double()[:, :, None, None]
    return (F.silu(y) if c.operand == 'gnsilu' else y).float()


def out_size(c, H, W):
    g = c.g
    if g.up:
        return 2 * H, 2 * W
    if g.sub:
        return H // 2, W // 2
    if g.stride == 2:
        return (H + g.pad[2] + g.pad[3] - g.ksize) // 2 + 1, (W + g.pad[0] + g.pad[1] - g.ksize) // 2 + 1
    return H, W


def expected(c, inputs, dev):
    """-> (ref, B, floor) of the case's output (NCHW, float64 on dev): the conv's bounds carried through the epilogue."""
    x, w, b, sc, sh, r, dec, scl, wv = [None if t is None else t.to(dev) for t in inputs]
    ref, B, floor = S.bounds(operand(c, x, sc, sh), w, c.g)
    ref = ref + b.double().view(1, -1, 1, 1)
    mag = ref.abs() + b.double().abs().view(1, -1, 1, 1)
    if r is not None:
        ref = ref + r.double()
        mag = mag + r.double().abs()
    if dec is not None:
        wvd = wv.double().view(-1, 1, 1, 1)
        d, s = dec.double(), scl.double()
        ref = d + wvd * (d * s + ref)
        B, floor = wvd * B, wvd * floor
        mag = d.abs() + wvd * (d * s).abs() + wvd * mag
    return ref, B, floor + EPI * mag


def plane_bytes(n):
    return (n * 2 + 1023) // 1024 * 1024


def tiles_launched(c, tile):
    Ho, Wo = out_size(c, c.H, c.W)
    return c.N * -(-Ho * Wo // 128) * (c.Cout // abs(tile))


# ---- the entry points ----

def _ws(nbytes):
    return torch.empty(int(nbytes), dtype=torch.uint8, device='cuda')


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _d(t, nhwc=False):
    if t is None:
        return None
    return (t.permute(0, 2, 3, 1) if nhwc else t).contiguous().cuda()


def run(c, inputs):
    """-> (out NCHW cuda, tile kind or None, out planes (uint8) or None)"""
    lib = _lib.load()
    x, w, b, sc, sh, r, dec, scl, wv = inputs
    N, Cin, H, W = x.shape
    Ho, Wo = out_size(c, H, W)
    k = c.g.ksize
    wd, bd, scd, shd, rd = _d(w), _d(b), _d(sc), _d(sh), _d(r, True)
    st = _stream()
    tile, pl = None, None
    if c.entry == 'conv2d':
        mode = 2 if c.g.up else (1 if c.g.stride == 2 else 0)
        xd = _d(x, True)
        out = torch.empty(N, Ho, Wo, c.Cout, device='cuda')
        wsb = lib.cfb_conv2d_workspace_bytes(N, H, W, Cin, c.Cout, k, mode)
        ws = _ws(wsb)
        _lib.check(lib.cfb_conv2d_nhwc(_lib.ptr(xd), _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(out), N, H, W, Cin, c.Cout, k, mode,
                                       _lib.ptr(scd), _lib.ptr(shd), 1 if c.operand == 'gnsilu' else 0, _lib.ptr(rd), 0, 2,
                                       _lib.ptr(ws), wsb, st), 'cfb_conv2d_nhwc')
    elif c.entry == 'halo':
        mode = 2 if c.g.up else 0
        xd = _d(x, True)
        x0 = xd[..., :c.cin1].contiguous() if c.cin1 else xd
        x1 = xd[..., c.cin1:].contiguous() if c.cin1 else None
        out = torch.empty(N, Ho, Wo, c.Cout, device='cuda')
        pl = torch.zeros(2 * plane_bytes(out.numel()), dtype=torch.uint8, device='cuda') if c.planes else None
        xform = 1 if c.operand == 'gnsilu' else c.extra.get('xform', 0)
        wsb = lib.cfb_conv2d_workspace_bytes(N, H, W, Cin, c.Cout, k, mode)
        ws = _ws(wsb)
        tn = ctypes.c_int32(0)
        decd, scld, wvd = _d(dec, True), _d(scl, True), _d(wv)
        _lib.check(lib.cfb_debug_conv_tc_prec_wv(
            _lib.ptr(x0), _lib.ptr(x1), c.cin1, _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(out), N, H, W, Cin, c.Cout, mode, xform,
            _lib.ptr(scd), _lib.ptr(shd), 1 if c.operand == 'gnsilu' else 0, _lib.ptr(rd), _lib.ptr(decd), _lib.ptr(scld),
            _lib.ptr(wvd), _lib.ptr(pl), None, _lib.ptr(ws), wsb, st, ctypes.byref(tn), k, 0, 0), 'cfb_debug_conv_tc_prec_wv')
        tile = tn.value
    elif c.entry == 'gen':
        ip, op, c0 = c.extra.get('in_pitch', Cin), c.extra.get('out_pitch', c.Cout), c.extra.get('out_c0', 0)
        xin = torch.full((N, H, W, ip), 7.25, device='cuda')
        xin[..., :Cin] = _d(x, True)
        buf = torch.full((N, Ho, Wo, op), -3.0, device='cuda')
        wsb = lib.cfb_conv2d_gen_workspace_bytes(Cin, c.Cout)
        ws = _ws(wsb)
        _lib.check(lib.cfb_conv2d_gen_nhwc(_lib.ptr(xin), ip, _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(buf), op, c0, N, H, W, Cin, c.Cout,
                                           int(c.g.up), c.g.pad_mode, int(c.g.sub), 0, None, c.Cout, None, c.Cout, 1.0,
                                           _lib.ptr(ws), wsb, st), 'cfb_conv2d_gen_nhwc')
        keep = torch.ones(op, dtype=torch.bool)
        keep[c0:c0 + c.Cout] = False
        torch.cuda.synchronize()
        assert bool((buf[..., keep.cuda()] == -3.0).all()), 'channels outside the destination slice changed'
        out = buf[..., c0:c0 + c.Cout]
    elif c.entry in ('pertap', 'pertap_slice'):
        xd = _d(x, True)
        stride = c.g.stride
        wsb = lib.cfb_conv2d_pertap_workspace_bytes(N, H, W, Cin, c.Cout, k, stride)
        ws = _ws(wsb)
        if c.entry == 'pertap':
            out = torch.empty(N, Ho, Wo, c.Cout, device='cuda')
            _lib.check(lib.cfb_conv2d_pertap_nhwc(_lib.ptr(xd), _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(out), N, H, W, Cin, c.Cout, k,
                                                  stride, 0, _lib.ptr(rd), _lib.ptr(ws), wsb, st), 'cfb_conv2d_pertap_nhwc')
        else:
            op, c0 = c.extra['out_pitch'], c.extra['out_c0']
            buf = torch.full((N, Ho, Wo, op), -3.0, device='cuda')
            _lib.check(lib.cfb_conv2d_pertap_slice_nhwc(_lib.ptr(xd), _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(buf), N, H, W, Cin, c.Cout,
                                                        k, stride, 0, op, c0, _lib.ptr(ws), wsb, st), 'cfb_conv2d_pertap_slice_nhwc')
            out = buf[..., c0:c0 + c.Cout]
    elif c.entry == 'arcface':
        xd = _d(x, True)
        out = torch.empty(N, Ho, Wo, c.Cout, device='cuda')
        wsb = lib.cfb_conv2d_gen_workspace_bytes(Cin, c.Cout)
        ws = _ws(wsb)
        _lib.check(lib.cfb_debug_arcface_conv(_lib.ptr(xd), _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(out), N, H, W, Cin, c.Cout, k, 1,
                                              _lib.ptr(scd), _lib.ptr(shd), 0, 0.0, None, _lib.ptr(ws), wsb, st),
                   'cfb_debug_arcface_conv')
    else:
        raise ValueError(c.entry)
    torch.cuda.synchronize()
    return out.permute(0, 3, 1, 2), tile, pl


HALO_CHILD = r'''
import sys
import numpy as np, torch
sys.path.insert(0, %(root)r)
from tests.test_gpu_split_error_model import CASES, case_inputs, kinds, run
res = {}
for c in CASES:
    if c.entry != 'halo':
        continue
    for kind in kinds(c):
        out, tile, pl = run(c, case_inputs(c, kind))
        res[c.name + '/' + kind] = out.cpu().numpy()              # NCHW
        res[c.name + '/' + kind + '/tile'] = np.array(tile)
        if pl is not None:
            res[c.name + '/' + kind + '/planes'] = pl.cpu().numpy()
np.savez(sys.argv[1], **res)
''' % {'root': ROOT}


@pytest.fixture(scope='module')
def halo_results():
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for bn in (None, '64'):
            e = dict(os.environ)
            e.pop('CFB_TC_BN', None)
            if bn:
                e['CFB_TC_BN'] = bn
            path = os.path.join(d, f'halo{bn}.npz')
            p = subprocess.run([sys.executable, '-c', HALO_CHILD, path], cwd=ROOT, env=e, capture_output=True, text=True,
                               timeout=900)
            assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
            out[bn] = dict(np.load(path))
    return out


def _check(c, kind, out, tile, planes=None):
    inputs = case_inputs(c, kind)
    ref, B, floor = expected(c, inputs, 'cuda')
    out = torch.as_tensor(out).cuda().double()
    bar = S.split_bar(out.permute(0, 2, 3, 1), ref.permute(0, 2, 3, 1), B.permute(0, 2, 3, 1), floor.permute(0, 2, 3, 1),
                      TAU[kind], tile)
    norm = float(((out - ref).abs() / (B + floor / TAU[kind])).max())
    print(f'{c.name:22s} {kind:8s} tile {str(tile):4s} tiles {tiles_launched(c, tile or 64):5d}  worst err/B {norm:.3g}  {bar}')
    assert bar.ok, f'{c.name} {kind}: {bar}'
    if planes is not None:
        o = out.float().permute(0, 2, 3, 1).reshape(-1).cpu().numpy()
        nb = plane_bytes(o.size)
        hi = planes[:nb].view(np.float16)[:o.size].astype(np.float64)
        lo = planes[nb:].view(np.float16)[:o.size].astype(np.float64)
        assert np.array_equal(hi, o.astype(np.float16).astype(np.float64)), 'hi plane != fp16(out)'
        assert (np.abs(hi + lo - o) <= 2.0 ** -21 * np.abs(o) + 2.0 ** -24).all(), 'hi + lo planes do not carry out'


HALO = [(c, k) for c in CASES if c.entry == 'halo' for k in kinds(c)]
OTHER = [(c, k) for c in CASES if c.entry != 'halo' for k in kinds(c)]


@pytest.mark.parametrize('bn', [None, '64'], ids=['default-tiles', 'bn64'])
@pytest.mark.parametrize('c,kind', HALO, ids=[f'{c.name}-{k}' for c, k in HALO])
def test_halo_tiles_hold_the_split_bar(halo_results, bn, c, kind):
    r = halo_results[bn]
    tile = int(r[c.name + '/' + kind + '/tile'])
    if c.g.ksize == 1:
        assert tile == 64
    elif bn == '64':
        assert tile == 64
    else:
        assert tile == (128 if c.Cout % 128 == 0 else -64)
    _check(c, kind, torch.from_numpy(r[c.name + '/' + kind]), tile, r.get(c.name + '/' + kind + '/planes'))


def test_every_tile_kind_has_a_case_beyond_two_waves(halo_results):
    most = collections.defaultdict(int)
    for bn in (None, '64'):
        for c, kind in HALO:
            t = int(halo_results[bn][c.name + '/' + kind + '/tile'])
            most[t] = max(most[t], tiles_launched(c, t))
    print('largest launch per tile kind:', dict(most))
    assert set(most) == {128, 64, -64} and min(most.values()) > 2 * 132


@pytest.mark.parametrize('c,kind', OTHER, ids=[f'{c.name}-{k}' for c, k in OTHER])
def test_form_holds_the_split_bar(c, kind):
    out, tile, _ = run(c, case_inputs(c, kind))
    _check(c, kind, out, tile)


# ---- magnitude properties (GEN: raw operand, no transform) ----

def _gen(x, w, g=S.SAME3):
    c = case('mag', 'gen', g, x.shape[0], x.shape[2], x.shape[3], x.shape[1], w.shape[0])
    b = torch.zeros(w.shape[0])
    out, _, _ = run(c, (x, w, b, None, None, None, None, None, None))
    return out.double(), c


def test_weight_scale_by_powers_of_two_is_exact():
    x, w = S.aligned_operands((1, 128, 16, 20), (64, 128, 3, 3), 5, 1.0, 1 / 34)
    base, _ = _gen(x, w)
    for k in range(-20, 5):
        out, _ = _gen(x, w * 2.0 ** k)
        assert torch.equal(out, base * 2.0 ** k), f'weights x 2^{k}: output is not the output x 2^{k}'


@pytest.mark.parametrize('kind', KINDS)
def test_small_and_large_activations_hold_the_model_with_its_floor(kind):
    worst = {}
    for k in range(-14, 13, 2):
        if kind == 'aligned':
            x, w = S.aligned_operands((1, 256, 16, 16), (128, 256, 3, 3), 11, 2.0 ** k, 1 / 48)
        else:
            x = S.random_operand((1, 256, 16, 16), 11, 2.0 ** k)
            w = S.random_operand((128, 256, 3, 3), 12, 1 / 48)
        assert float(x.abs().max()) < 65504
        out, _ = _gen(x, w)
        ref, B, floor = S.bounds(x.cuda(), w.cuda())
        bar = S.split_bar(out, ref, B, floor, TAU[kind])
        worst[k] = bar.worst
        assert bar.ok, f'activations x 2^{k}: {bar}'
    print(kind, 'worst err/(tau*B+floor) per activation exponent:', {k: f'{v:.2g}' for k, v in worst.items()})


def test_per_channel_weight_scales_hold_each_channel_bound():
    """Folded BatchNorm: output channel co scaled by 2^-16..1; each channel against its own B (one weight exponent per conv)."""
    x, w = S.aligned_operands((1, 128, 16, 16), (64, 128, 3, 3), 21, 1.0, 1 / 34)
    w = w * 2.0 ** -torch.linspace(0, 16, 64).view(-1, 1, 1, 1)
    out, _ = _gen(x, w)
    ref, B, floor = S.bounds(x.cuda(), w.cuda())
    bar = S.split_bar(out, ref, B, floor, TAU['aligned'])
    assert bar.ok, bar


# ---- the attention core (cfb_debug_bmm_tc) ----

def _attention_ref(q, k, v, heads):
    """float64 softmax(q k^T d^-1/2) v per head; -> (out, bound, floor) [n, 256, heads*d]"""
    n, t, E = q.shape
    d = E // heads
    qh, kh, vh = (z.double().view(n, t, heads, d).transpose(1, 2) for z in (q, k, v))
    s = qh @ kh.transpose(-1, -2) / math.sqrt(d)
    p = torch.softmax(s, -1)
    o = p @ vh
    sb = (qh.abs() @ kh.abs().transpose(-1, -2) / math.sqrt(d)).amax(-1, keepdim=True)   # score bound of the row
    # B of P v, plus the score error (tau * sb at most) carried through the softmax: sum_j p_j |v_j - o|
    bound = p @ vh.abs() + sb * torch.einsum('nhij,nhijc->nhic', p, (vh[:, :, None] - o[:, :, :, None]).abs())
    floor = 2.0 ** -25 * vh.abs().sum(-2, keepdim=True) + 2.0 ** -21 * (p @ vh.abs())
    back = lambda z: z.transpose(1, 2).reshape(n, t, E)                                   # noqa: E731
    return back(o), back(bound), back(floor.expand_as(o))


@pytest.mark.parametrize('n,heads,d', [(2, 8, 64), (1, 1, 512)], ids=['transformer-8x64', 'attnblock-512'])
def test_bmm_tc_attention_core(n, heads, d):
    lib = _lib.load()
    E = heads * d
    q, k, v = (S.random_operand((n, 256, E), 90 + i, s) for i, s in enumerate((1.0, 1.0, 1.0)))
    qd, kd, vd = q.cuda(), k.cuda(), v.cuda()
    out = torch.empty(n, 256, E, device='cuda')
    pl = torch.zeros(2 * plane_bytes(out.numel()), dtype=torch.uint8, device='cuda')
    wsb = lib.cfb_debug_bmm_tc_workspace_bytes(n, heads, d)
    ws = _ws(wsb)
    _lib.check(lib.cfb_debug_bmm_tc(_lib.ptr(qd), _lib.ptr(kd), _lib.ptr(vd), _lib.ptr(out), _lib.ptr(pl), n, heads, d,
                                    _lib.ptr(ws), wsb, _stream()), 'cfb_debug_bmm_tc')
    torch.cuda.synchronize()
    ref, bound, floor = _attention_ref(qd, kd, vd, heads)
    bar = S.split_bar(out.double(), ref, bound, floor, TAU['random'])
    print(f'bmm heads {heads} d {d}: worst err/bound {float(((out.double() - ref).abs() / bound).max()):.3g}  {bar}')
    assert bar.ok, bar
    o = out.reshape(-1).cpu().numpy()
    nb = plane_bytes(o.size)
    plc = pl.cpu().numpy()
    hi = plc[:nb].view(np.float16)[:o.size].astype(np.float64)
    lo = plc[nb:].view(np.float16)[:o.size].astype(np.float64)
    assert np.array_equal(hi, o.astype(np.float16).astype(np.float64)), 'hi plane != fp16(out)'
    assert (np.abs(hi + lo - o) <= 2.0 ** -21 * np.abs(o) + 2.0 ** -24).all()
