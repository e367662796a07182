"""-m gpu: 128-output-channel tiles of the halo engine give the same results as 64-wide tiles, bit for bit.

CFB_TC_BN is read once per process, so every side runs in its own subprocess and writes its results to a temporary .npz:
  default          3x3 / Upsample halo convs with Cout % 128 == 0 on 128 x 128 tiles (two MMA warpgroups)
  CFB_TC_BN=64     every conv on 128 x 64 tiles
Kernel cases go through cfb_debug_conv_tc, which reports the tile width it launched (so a case cannot pass by running the same
kernel on both sides): Cout in {128, 256, 512}, Cin in {64, 128, 256, 512} (one to five partial sums per tile); fused transform
with GroupNorm-affine + SiLU and as a raw split, the two-source concatenation, raw operand planes, Upsample; residual, SFT and
operand-plane epilogues and GroupNorm partials.  Outputs, planes and partials must agree bitwise, the output must match a
float64 torch conv at the bar of test_conv_matches_torch.  Forward: config 1 at batch 32 bitwise between the two, and the
default against the golden vectors (batch 1 and 6 rows identical)."""
import math
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.util import golden, maxabs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (N, Cin, Cout, H, mode, operand, cin1, residual, sft, out planes, GroupNorm partials)
# operand: 'gnsilu' / 'split' = fused transform with GroupNorm-affine + SiLU / raw hi-lo split; 'planes' = raw operand planes;
# cin1 > 0: channels [cin1, Cin) come from a second tensor (Fuse_sft_block's torch.cat)
CASES = [
    (2, 64, 128, 32, 0, 'gnsilu', 0, True, False, False, True),
    (2, 128, 128, 32, 0, 'gnsilu', 0, False, False, False, True),
    (1, 512, 512, 16, 0, 'gnsilu', 0, True, False, False, True),
    (1, 128, 256, 32, 0, 'gnsilu', 0, False, False, True, True),
    (1, 256, 256, 16, 0, 'split', 0, True, False, False, True),
    (1, 512, 256, 32, 0, 'gnsilu', 256, False, True, False, False),
    (1, 256, 128, 32, 0, 'split', 128, False, False, False, True),
    (2, 128, 128, 16, 0, 'planes', 0, True, False, True, False),
    (1, 512, 512, 16, 0, 'planes', 0, False, True, False, True),
    (1, 128, 128, 16, 2, 'planes', 0, False, False, True, True),
    (1, 256, 256, 16, 2, 'planes', 0, True, False, False, False),
    (1, 512, 256, 16, 2, 'planes', 0, False, False, False, True),
]
SFT_W = 0.5

KERNEL_CHILD = r'''
import ctypes, sys
import numpy as np, torch
sys.path.insert(0, %(root)r)
from codeformer_b200 import _lib
from tests.test_gpu_wide_tiles import CASES, SFT_W, case_inputs, plane_bytes
lib = _lib.load()
st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
res = {}
for i, case in enumerate(CASES):
    N, Cin, Cout, H, mode, operand, cin1, resid, sft, planes, gn = case
    x, w, b, sc, sh, r, dec, scl = [None if t is None else t.cuda() for t in case_inputs(case)]
    Ho = 2 * H if mode == 2 else H
    x0 = x[..., :cin1].contiguous() if cin1 else x
    x1 = x[..., cin1:].contiguous() if cin1 else None
    out = torch.empty(N, Ho, Ho, Cout, device='cuda')
    pl = torch.zeros(2 * plane_bytes(N, Ho, Cout), dtype=torch.uint8, device='cuda') if planes else None
    gp = torch.zeros(N * Ho * Ho // 128 * 4 * 64, device='cuda') if gn else None
    wsb = lib.cfb_conv2d_workspace_bytes(N, H, H, Cin, Cout, 3, mode)
    ws = torch.empty(int(wsb), dtype=torch.uint8, device='cuda')
    tn = ctypes.c_int32(0)
    _lib.check(lib.cfb_debug_conv_tc(_lib.ptr(x0), _lib.ptr(x1), cin1, _lib.ptr(w), _lib.ptr(b), _lib.ptr(out), N, H, H, Cin, Cout,
                                     mode, 0 if operand == 'planes' else 1, _lib.ptr(sc), _lib.ptr(sh), 1 if operand == 'gnsilu' else 0,
                                     _lib.ptr(r), _lib.ptr(dec), _lib.ptr(scl), SFT_W, _lib.ptr(pl), _lib.ptr(gp), _lib.ptr(ws), wsb,
                                     st, ctypes.byref(tn)), 'cfb_debug_conv_tc')
    torch.cuda.synchronize()
    res['out%%d' %% i] = out.cpu().numpy()
    res['tile%%d' %% i] = np.array(tn.value)
    if planes:
        res['planes%%d' %% i] = pl.cpu().numpy()
    if gn:
        res['gn%%d' %% i] = gp.cpu().numpy()
np.savez(sys.argv[1], **res)
''' % {'root': ROOT}

FORWARD_CHILD = r'''
import sys
import numpy as np, torch
sys.path.insert(0, %(root)r)
import codeformer_b200 as cb
from codeformer_b200 import spec as S
from tests.util import faces_input
torch.set_grad_enabled(False)
net = cb.CodeFormer().cuda().eval()
net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1))
x = faces_input().cuda()
x = x.repeat((32 + x.shape[0] - 1) // x.shape[0], 1, 1, 1)[:32].contiguous()
out, logits, lq = net(x, w=0.5, adain=True)
res = dict(out=out.cpu().numpy(), logits=logits.cpu().numpy(), lq=lq.cpu().numpy())
x1 = faces_input(slice(0, 1)).cuda()
for tag, batch in (('b1', 1), ('b6', 6)):
    o, lg, l = net(x1.expand(batch, -1, -1, -1).contiguous(), w=0.5, adain=True)
    res[tag + '_out'] = o.cpu().numpy(); res[tag + '_logits'] = lg.cpu().numpy(); res[tag + '_lq'] = l.cpu().numpy()
np.savez(sys.argv[1], **res)
''' % {'root': ROOT}


def _rand(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def plane_bytes(N, Ho, Cout):
    return (N * Ho * Ho * Cout * 2 + 1023) // 1024 * 1024


def case_inputs(case):
    """NHWC x, OIHW w, bias, per-(n, cin) scale / shift, NHWC residual, SFT dec / scale (None where the case has none)."""
    N, Cin, Cout, H, mode, operand, cin1, resid, sft, planes, gn = case
    Ho = 2 * H if mode == 2 else H
    x = _rand(N, H, H, Cin, seed=11) * 2 + 0.5
    w = _rand(Cout, Cin, 3, 3, seed=12, scale=1.0 / math.sqrt(Cin * 9))
    b = _rand(Cout, seed=13, scale=0.1)
    sc = 1 + 0.1 * _rand(N, Cin, seed=14) if operand == 'gnsilu' else None
    sh = 0.1 * _rand(N, Cin, seed=15) if operand == 'gnsilu' else None
    r = _rand(N, Ho, Ho, Cout, seed=16) if resid else None
    dec = _rand(N, Ho, Ho, Cout, seed=17) if sft else None
    scl = 0.5 * _rand(N, Ho, Ho, Cout, seed=18) if sft else None
    return x, w, b, sc, sh, r, dec, scl


def reference(case):
    """float64 torch: NHWC output of the case"""
    N, Cin, Cout, H, mode, operand, cin1, resid, sft, planes, gn = case
    x, w, b, sc, sh, r, dec, scl = [None if t is None else t.double() for t in case_inputs(case)]
    if operand == 'gnsilu':
        x = F.silu(x * sc[:, None, None, :] + sh[:, None, None, :])
    x = x.permute(0, 3, 1, 2)
    if mode == 2:
        x = F.interpolate(x, scale_factor=2.0, mode='nearest')
    v = F.conv2d(x, w, b, padding=1).permute(0, 2, 3, 1)
    if resid:
        v = v + r
    if sft:
        v = dec + SFT_W * (dec * scl + v)
    return v


def _run(child, bn, path):
    e = dict(os.environ)
    e.pop('CFB_TC_BN', None)
    if bn:
        e['CFB_TC_BN'] = bn
    p = subprocess.run([sys.executable, '-c', child, path], cwd=ROOT, env=e, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    return np.load(path)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


@pytest.fixture(scope='module')
def kernel_results():
    with tempfile.TemporaryDirectory() as d:
        yield {bn: dict(_run(KERNEL_CHILD, bn, os.path.join(d, f'k{bn}.npz'))) for bn in ('64', None)}


def _case_id(c):
    N, Cin, Cout, H, mode, operand, cin1, resid, sft, planes, gn = c
    return '-'.join([('up' if mode == 2 else 'same'), f'cin{Cin}', f'cout{Cout}', operand] + (['cat'] if cin1 else []) +
                    (['res'] if resid else []) + (['sft'] if sft else []) + (['pl'] if planes else []) + (['gn'] if gn else []))


@pytest.mark.parametrize('i', range(len(CASES)), ids=[_case_id(c) for c in CASES])
def test_wide_tiles_equal_narrow_tiles_torch_and_gn_moments(kernel_results, i):
    N, Cin, Cout, H, mode, operand, cin1, resid, sft, planes, gn = CASES[i]
    wide, narrow = kernel_results[None], kernel_results['64']
    assert int(wide[f'tile{i}']) == 128 and int(narrow[f'tile{i}']) == 64, 'the two sides must run 128- and 64-wide tiles'
    ow, on = wide[f'out{i}'], narrow[f'out{i}']
    assert np.array_equal(_bits(ow), _bits(on)), f'128-wide tiles differ from 64-wide tiles by {np.abs(ow - on).max()}'
    ref = reference(CASES[i])
    assert maxabs(torch.from_numpy(ow).double(), ref) < 6e-5 * max(1.0, float(ref.abs().max()))
    if planes:
        pw = wide[f'planes{i}']
        assert np.array_equal(pw, narrow[f'planes{i}']), 'operand planes differ'
        nb = plane_bytes(N, ow.shape[1], Cout)
        hi = pw[:nb].view(np.float16)[:ow.size].astype(np.float32)
        lo = pw[nb:].view(np.float16)[:ow.size].astype(np.float32)
        assert np.array_equal(hi, ow.reshape(-1).astype(np.float16).astype(np.float32))
        assert np.abs(hi + lo - ow.reshape(-1)).max() <= 2.0 ** -20 * max(1.0, float(np.abs(ow).max()))
    if gn:
        gw = wide[f'gn{i}']
        assert np.array_equal(_bits(gw), _bits(narrow[f'gn{i}'])), 'GroupNorm partials differ'
        assert_gn_partials(gw, ow, N, Cout)


def assert_gn_partials(part, out, N, Cout):
    """GroupNorm partials [N * slots][32 groups][mean, M2] (M2: squared deviations from the slot mean, 32 pixels x Cout/32
    channels per slot) merged in float64 against the per-image group mean and M2 of the output"""
    p = part.reshape(N, -1, 32, 2).astype(np.float64)
    mk, m2k = p[..., 0], p[..., 1]
    mean = mk.mean(1)
    m2 = m2k.sum(1) + Cout * ((mk - mean[:, None]) ** 2).sum(1)
    grp = out.reshape(N, -1, 32, Cout // 32).astype(np.float64)
    gmean = grp.mean((1, 3))
    gm2 = ((grp - gmean[:, None, :, None]) ** 2).sum((1, 3))
    assert np.abs(mean - gmean).max() < 1e-5 * np.abs(grp).max()
    assert np.abs(m2 - gm2).max() < 1e-4 * gm2.max()


def test_forward_wide_tiles_bitwise_and_golden():
    with tempfile.TemporaryDirectory() as d:
        wide = _run(FORWARD_CHILD, None, os.path.join(d, 'wide.npz'))
        narrow = _run(FORWARD_CHILD, '64', os.path.join(d, 'narrow.npz'))
        for k in ('out', 'logits', 'lq'):
            assert np.array_equal(_bits(wide[k]), _bits(narrow[k])), \
                f'batch 32 {k}: 128-wide tiles differ from 64-wide tiles by {np.abs(wide[k] - narrow[k]).max()}'
        g = golden('codeformer_main.npz')
        for tag in ('b1', 'b6'):
            out, logits, lq = wide[tag + '_out'], wide[tag + '_logits'], wide[tag + '_lq']
            assert np.array_equal(logits[:1].argmax(2), g['top_idx']), f'{tag}: code indices must be bit-exact'
            assert maxabs(out[:1], g['out']) < 1e-3 and maxabs(logits[:1], g['logits']) < 2e-4 and \
                maxabs(lq[:1], g['lq_feat']) < 2e-4, tag
            assert np.array_equal(out[:1], out[-1:]), f'{tag}: identical faces in one batch must give identical outputs'
