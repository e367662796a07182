"""-m gpu: GroupNorm statistics at large mean-to-spread ratios r = |group mean| / group standard deviation.

Every GroupNorm of CodeFormer / VQAutoEncoder takes its statistics from one of three producers -- the standalone kernel of
cfb_group_norm_coef, the per-slot partials of the tensor-core conv epilogue and of conv_first (finalized by the kernel behind
cfb_debug_gn_coef_from_partials), and the merge of two sources' partials for Fuse_sft_block's concatenation.  Each check
compares y = x * scale + shift with float64 F.group_norm of the same fp32 x, and measures torch's own fp32 CPU group_norm on
that input against float64 as well:

    max|y_gpu - y_f64| <= 4 * max|y_torch32 - y_f64| + 2e-6

torch fp32's error grows like r * 2^-24 (the rounding of the mean), so the bar follows r as the reference arithmetic does.  The
factor 4 leaves room for another summation order and for scale and shift being rounded to fp32 separately; 2e-6 covers r = 0,
where torch is off by a few fp32 ulps of |y| < 5.  Sums of squares in fp32 miss the bar from r ~ 100 on: their error grows like
r^2 * 2^-24.  Inputs are x = offset_g + spread_c + z with z ~ N(0, 1): offsets of r standard deviations (another offset for the
second image of the batch), a per-channel spread inside each group or none, and three special groups -- the constant 2 (exact
in binary), the constant 0.1 (not exact) and a group of standard deviation 1e-4 = 0.1 sqrt(eps), where eps dominates."""
import ctypes
import json
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from codeformer_b200 import _lib
from tests import gpu_util as G

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 1e-6
R_VALUES = (0, 10, 100, 1000, 10000)


def _affine(C, seed):
    g = torch.Generator().manual_seed(seed)
    return 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)


def group_offsets(r, N=2):
    """[N, 32] group offsets of r (unit standard deviations): signs alternating in pairs of groups (so that the two groups one
    group of a concatenation takes from a source share theirs), 1..1.5 r, the second image at -0.6x"""
    g = torch.arange(32, dtype=torch.float64)
    off = r * torch.where((g // 2) % 2 == 0, 1.0, -1.0) * (1 + g / 64)
    return torch.stack([off, -0.6 * off])[:N]


def special_groups(x, cpg, tiny):
    """groups 29..31 of x [..., C]: standard deviation 1e-4 around 0.5 (tiny = the unit-variance values), constant 2, 0.1"""
    x[..., 29 * cpg:30 * cpg] = 0.5 + 1e-4 * tiny[..., 29 * cpg:30 * cpg]
    x[..., 30 * cpg:31 * cpg] = 2.0
    x[..., 31 * cpg:] = 0.1
    return x


def group_input(N, C, HW, r, spread, seed):
    """x [N, HW, C] fp32 = offset_g + spread_c + z, groups 29..31 special"""
    g = torch.Generator().manual_seed(seed)
    cpg = C // 32
    z = torch.randn(N, HW, C, generator=g, dtype=torch.float64)
    sp = spread * torch.randn(C, generator=g, dtype=torch.float64)
    x = z + sp + math.sqrt(1 + spread ** 2) * group_offsets(r, N).repeat_interleave(cpg, dim=1)[:, None, :]
    return special_groups(x, cpg, z).float()


def y_errors(x, scale, shift, gamma, beta):
    """x [N, HW, C] fp32 (cpu), scale / shift [N, C] of the GPU -> (max|y_gpu - y_f64|, max|y_torch32 - y_f64|)"""
    xc = x.permute(0, 2, 1)
    y64 = F.group_norm(xc.double(), 32, gamma.double(), beta.double(), eps=EPS)
    e32 = float((F.group_norm(xc, 32, gamma, beta, eps=EPS).double() - y64).abs().max())
    yg = xc.double() * scale.cpu().double()[:, :, None] + shift.cpu().double()[:, :, None]
    return float((yg - y64).abs().max()), e32


def _judge(what, err, e32, failures):
    bar = 4 * e32 + 2e-6
    print(f'{what:48s} gpu {err:.3e}  torch32 {e32:.3e}  bar {bar:.3e}' + ('' if err <= bar else '  FAIL'))
    if not err <= bar:
        failures.append(f'{what}: {err:.3e} > {bar:.3e} (torch fp32 {e32:.3e})')


# ---- a. the standalone statistics kernel (cfb_group_norm_coef): per-thread sums of 16 (C 64, HW 256) to 1024 pixels ------------
@pytest.mark.parametrize('HW', [256, 4096, 65536])
@pytest.mark.parametrize('C', [64, 128, 256, 512])
def test_group_norm_coef_large_mean(C, HW):
    lib = _lib.load()
    gamma, beta = _affine(C, 1)
    spread = 0.5 if C in (64, 256) else 0.0
    wsb = lib.cfb_gn_workspace_bytes(2, HW, C)
    ws = torch.empty(int(wsb), dtype=torch.uint8, device='cuda')
    g_d, b_d = gamma.cuda(), beta.cuda()
    failures = []
    for r in R_VALUES:
        x = group_input(2, C, HW, r, spread, seed=C + HW)
        xd = x.cuda()
        scale, shift = torch.empty(2, C, device='cuda'), torch.empty(2, C, device='cuda')
        _lib.check(lib.cfb_group_norm_coef(_lib.ptr(xd), _lib.ptr(g_d), _lib.ptr(b_d), _lib.ptr(scale), _lib.ptr(shift), 2, HW, C,
                                           32, EPS, _lib.ptr(ws), wsb, G.stream()), 'cfb_group_norm_coef')
        torch.cuda.synchronize()
        _judge(f'standalone C {C} HW {HW} r {r}', *y_errors(x, scale, shift, gamma, beta), failures)
        del x, xd
    assert not failures, '\n'.join(failures)


# ---- b. epilogue partials -> finalize, and the concatenation merge ---------------------------------------------------------------
# (N, H): 32 slots per image (one finalize CTA), 512 (two CTAs + ticket), 8192 (16 CTAs)
EPI_SIZES = [(2, 32), (2, 128)]
EPI_SIZES_64 = EPI_SIZES + [(1, 512)]


def conv_with_offsets(lib, N, H, Cout, r, sign, seed, gp):
    """3x3 conv (Cin 64) on the wgmma engine, bias = the group offsets (the same for every channel of a group); groups 29..31
    special (weights x1e-4 around bias 0.5, zero weights with bias 2 and 0.1).  gn_part -> gp.  Returns (out, tile)."""
    g = torch.Generator().manual_seed(seed)
    cpg = Cout // 32
    x = torch.randn(N, H, H, 64, generator=g).cuda()
    w = torch.randn(Cout, 64, 3, 3, generator=g) / 24.0
    w[29 * cpg:30 * cpg] *= 1e-4
    w[30 * cpg:] = 0
    b = (sign * group_offsets(r, 1)[0]).repeat_interleave(cpg).float()
    b[29 * cpg:30 * cpg], b[30 * cpg:31 * cpg], b[31 * cpg:] = 0.5, 2.0, 0.1
    w, b = w.cuda(), b.cuda()
    out = torch.empty(N, H, H, Cout, device='cuda')
    wsb = lib.cfb_conv2d_workspace_bytes(N, H, H, 64, Cout, 3, 0)
    ws = torch.empty(int(wsb), dtype=torch.uint8, device='cuda')
    tn = ctypes.c_int32(0)
    _lib.check(lib.cfb_debug_conv_tc(_lib.ptr(x), None, 0, _lib.ptr(w), _lib.ptr(b), _lib.ptr(out), N, H, H, 64, Cout, 0, 0,
                                     None, None, 0, None, None, None, 0.0, None, _lib.ptr(gp), _lib.ptr(ws), wsb, G.stream(),
                                     ctypes.byref(tn)), 'cfb_debug_conv_tc')
    return out, tn.value


def finalize(lib, gp, N, HW, C, gamma, beta):
    slots = HW // 32
    wsb = lib.cfb_debug_gn_partials_workspace_bytes(N, slots)
    ws = torch.empty(int(wsb), dtype=torch.uint8, device='cuda')
    scale, shift = torch.empty(N, C, device='cuda'), torch.empty(N, C, device='cuda')
    g_d, b_d = gamma.cuda(), beta.cuda()
    _lib.check(lib.cfb_debug_gn_coef_from_partials(_lib.ptr(gp), slots, _lib.ptr(g_d), _lib.ptr(b_d), _lib.ptr(scale),
                                                   _lib.ptr(shift), N, HW, C, EPS, _lib.ptr(ws), wsb, G.stream()),
               'cfb_debug_gn_coef_from_partials')
    torch.cuda.synchronize()
    return scale, shift


def epilogue_failures(Cout, expect_tile):
    """every size x r for one Cout: statistics of one conv output and of the concatenation of two.  The reference is float64
    GroupNorm of the GPU's own fp32 outputs, so conv rounding does not enter."""
    lib = _lib.load()
    failures = []
    for N, H in (EPI_SIZES_64 if Cout == 64 else EPI_SIZES):
        HW = H * H
        slots = HW // 32
        gamma, beta = _affine(Cout, 2)
        gamma2, beta2 = _affine(2 * Cout, 3)
        for r in R_VALUES:
            ga = torch.zeros(N * slots * 64, device='cuda')
            gb = torch.zeros(N * slots * 64, device='cuda')
            a, tile = conv_with_offsets(lib, N, H, Cout, r, 1.0, 5, ga)
            assert tile == expect_tile, f'Cout {Cout}: tile {tile}, expected {expect_tile}'
            b, _ = conv_with_offsets(lib, N, H, Cout, r, -0.7, 6, gb)
            gc = torch.zeros(N * slots * 64, device='cuda')
            _lib.check(lib.cfb_debug_gn_cat_partials(_lib.ptr(ga), _lib.ptr(gb), _lib.ptr(gc), N * slots, Cout, G.stream()),
                       'cfb_debug_gn_cat_partials')
            sa, ha = finalize(lib, ga, N, HW, Cout, gamma, beta)
            sc, hc = finalize(lib, gc, N, HW, 2 * Cout, gamma2, beta2)
            ac, bc = a.view(N, HW, Cout).cpu(), b.view(N, HW, Cout).cpu()
            _judge(f'epilogue Cout {Cout} tile {tile} {N}x{H}^2 r {r}', *y_errors(ac, sa, ha, gamma, beta), failures)
            _judge(f'concat 2x{Cout} {N}x{H}^2 r {r}', *y_errors(torch.cat([ac, bc], -1), sc, hc, gamma2, beta2), failures)
    return failures


@pytest.mark.parametrize('Cout', [64, 128, 256, 512])
def test_epilogue_partials_large_mean(Cout):
    """default tiles: channel-major 128 x 64 (Cout 64, 2 channels per group), 128 x 128 (4 / 8 / 16 channels per group)"""
    failures = epilogue_failures(Cout, -64 if Cout == 64 else 128)
    assert not failures, '\n'.join(failures)


CHILD = r'''
import json, sys
sys.path.insert(0, %(root)r)
from tests.test_gpu_groupnorm_range import epilogue_failures
print('RESULT ' + json.dumps(epilogue_failures(64, 64)))
''' % {'root': ROOT}


def test_epilogue_partials_large_mean_pixel_major():
    """Cout 64 on pixel-major 128 x 64 tiles (CFB_TC_BN=64 is read once per process: its own subprocess)"""
    e = dict(os.environ, CFB_TC_BN='64')
    p = subprocess.run([sys.executable, '-c', CHILD], cwd=ROOT, env=e, capture_output=True, text=True, timeout=900)
    print(p.stdout[-6000:])
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    failures = json.loads(re.findall(r'^RESULT (.*)$', p.stdout, re.M)[-1])
    assert not failures, '\n'.join(failures)


# ---- c. the forward with DC offsets ------------------------------------------------------------------------------------------------
DC_ENC, DC_GEN, DC_GEN_LAST = 10.0, 30.0, 7


def offset_state_dict():
    """random_state_dict(seed 1) whose conv_first bias and ResBlock conv2 biases carry a per-group DC offset: DC_ENC in the
    encoder, DC_GEN in the 16 x 16 generator blocks (0..DC_GEN_LAST).  The residual streams accumulate it: r >= 100 at several
    norms while |activations| stay < 1e4 (the SFT blocks multiply the two streams, so the larger generator blocks get none)."""
    from codeformer_b200 import spec as S
    sd = S.random_state_dict(S.codeformer_spec(), 1)
    for k in list(sd):
        m = re.match(r'(encoder|generator)\.blocks\.(\d+)\.(conv2\.)?bias$', k)
        if not m or not (m.group(3) or k == 'encoder.blocks.0.bias'):
            continue
        if m.group(1) == 'generator' and int(m.group(2)) > DC_GEN_LAST:
            continue
        c = sd[k].numel()
        g = torch.arange(c) // (c // 32)
        dc = DC_ENC if m.group(1) == 'encoder' else DC_GEN
        sd[k] = (sd[k] + dc * torch.where(g % 2 == 0, 1.0, -0.5) * (1 + g / 32.0)).contiguous()
    return sd


def _oracle(sd, x, dtype):
    """codeformer_oracle in `dtype` with every block output collected and the r of every GroupNorm input recorded"""
    from oracle import codeformer_oracle as O
    col, rs = {}, []
    gn = O.group_norm

    def rec(sd_, p, t):
        v = t.double().reshape(t.shape[0], 32, -1)
        rs.append((p, float((v.mean(-1).abs() / v.std(-1, unbiased=False).clamp_min(1e-30)).max()), float(t.abs().max())))
        return gn(sd_, p, t)
    O.group_norm = rec
    try:
        res = O.codeformer_forward({k: v.to(dtype) for k, v in sd.items()}, x.to(dtype), w=0.5, adain_on=True, collect=col)
    finally:
        O.group_norm = gn
    return res, col, rs


@pytest.fixture(scope='module')
def offset_oracles():
    from tests.util import faces_input
    sd = offset_state_dict()
    x = faces_input(slice(0, 1))
    (o64, l64, q64), c64, rs = _oracle(sd, x, torch.float64)
    (o32, _, _), c32, _ = _oracle(sd, x, torch.float32)
    print('GroupNorm inputs of the float64 oracle (r = max over images and groups of |mean| / std):')
    for p, r, m in rs:
        print(f'   {p:42s} r {r:9.1f}  max|x| {m:8.1f}')
    assert sum(r >= 100 for _, r, _ in rs) >= 5, 'the offsets must give r >= 100 at several norms'
    assert max(m for _, _, m in rs) < 1e4, 'activations must stay well inside the fp16 operand range'
    return sd, x, o64, l64, c64, o32, c32


# Stage bars: STAGE_FACTOR[engine] x the fp32 oracle's error + STAGE_FLOOR, both in units of the group's standard deviation.
# f32: 8x for fp32 rounding in another order through ~50 layers, 2x margin.  tc: the split-fp16 operands carry ~21 bits against
# fp32's 24 (8x), compounded through the SFT products of the 256 / 512 generator stages: 23x measured at fuse.256 on an H100
# (where r ~ 1, the same before and after the (mean, M2) slots), so 32x; the slots themselves are checked at their own
# bar by the epilogue tests above.
STAGE_FACTOR = {'f32': 16, 'tc': 32}
STAGE_FLOOR = 2e-5


@pytest.mark.parametrize('engine', ['tc', 'f32'])
def test_forward_large_mean_vs_float64_oracle(offset_oracles, engine):
    """tc: statistics from the conv epilogue's and conv_first's partials and the concatenation merge; f32: the standalone
    kernel everywhere.  Stage errors are measured in units of the float64 reference's per-group standard deviation (a DC
    offset would inflate a max-relative bar and hide them) and must stay within STAGE_FACTOR[engine] x the fp32 oracle's +
    STAGE_FLOOR."""
    import codeformer_b200 as cb
    sd, x, o64, l64, c64, o32, c32 = offset_oracles
    net = cb.CodeFormer().cuda().eval()
    net.load_state_dict(sd)
    net.set_engine(engine)
    try:
        net(x.cuda(), w=0.5, adain=True)
    except RuntimeError as e:
        if engine == 'tc' and 'not supported by the wgmma engine' in str(e):
            pytest.skip('tc-only mode: some shapes are not on the tensor-core engine')
        raise
    keys = [k for k, v in c64.items() if v.dim() == 4 and k not in ('enc.23', 'gen.23', 'gen.24')]
    bufs = {k: torch.empty(c64[k].numel(), device='cuda') for k in keys}
    for k in keys:
        net.capture(k, bufs[k])
    out, logits, _ = net(x.cuda(), w=0.5, adain=True)
    torch.cuda.synchronize()
    for k in keys:
        net.capture(k, None)
    failures = []
    print(f'[{engine}] stage errors in units of the per-group standard deviation (gpu / fp32 oracle):')
    for k in keys:
        ref = c64[k].permute(0, 2, 3, 1)                          # NHWC float64
        N, H, W, C = ref.shape
        std = ref.reshape(N, H * W, 32, C // 32).std(dim=(1, 3), unbiased=False).clamp_min(1e-12)   # [N, 32]
        unit = std.repeat_interleave(C // 32, dim=1)[:, None, None, :]
        eg = float(((bufs[k].cpu().double().view(N, H, W, C) - ref).abs() / unit).max())
        e32 = float(((c32[k].permute(0, 2, 3, 1).double() - ref).abs() / unit).max())
        bad = eg > STAGE_FACTOR[engine] * e32 + STAGE_FLOOR
        print(f'   {k:10s} {eg:.3e} {e32:.3e}' + ('  FAIL' if bad else ''))
        if bad:
            failures.append(f'{k}: {eg:.3e} > {STAGE_FACTOR[engine]} x {e32:.3e} + {STAGE_FLOOR}')
    top2 = l64.topk(2, dim=2).values
    sure = (top2[..., 0] - top2[..., 1]) > 1e-3
    same = logits.argmax(2).cpu() == l64.argmax(2)
    e_out = float((out.cpu().double() - o64).abs().max())
    print(f'[{engine}] out {e_out:.3e} (fp32 oracle {float((o32.double() - o64).abs().max()):.3e}); '
          f'code indices differing where the margin > 1e-3: {int((~same & sure).sum())}')
    assert bool(same[sure].all()), 'code indices must equal the float64 oracle where its top-1/top-2 margin exceeds 1e-3'
    assert e_out < 1e-3
    assert not failures, '\n'.join(failures)
