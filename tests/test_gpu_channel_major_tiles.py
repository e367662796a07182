"""-m gpu: channel-major 128 x 64 tiles of the halo engine give the same results as pixel-major 128 x 64 tiles, bit for bit.

The 3x3 / Upsample halo convs with Cout % 128 == 64 run on tiles computed transposed (weights as the wgmma A operand, one
m64n128k16 per product and k-step).  CFB_TC_BN is read once per process, so every side runs in its own subprocess:
  default          channel-major tiles (cfb_debug_conv_tc reports -64)
  CFB_TC_BN=64     every conv on pixel-major 128 x 64 tiles (reports 64)
Cases at Cout = 64: Cin 64 (one partial sum of 9 k-blocks), 128 (8 + 8 + 2) and 256; fused transform with GroupNorm-affine +
SiLU, as a raw split and as the two-source concatenation, raw operand planes, Upsample; residual, SFT and operand-plane epilogues
and GroupNorm partials (2 channels per group); one case at 512^2 with N = 2, so every CTA runs many tiles and the slot and
patch phases wrap.  Outputs, planes and partials must agree bitwise, the output must match a float64 torch conv."""
import os
import tempfile

import numpy as np
import pytest
import torch

from tests.test_gpu_wide_tiles import ROOT, _bits, _case_id, _run, assert_gn_partials, plane_bytes, reference
from tests.util import maxabs

pytestmark = pytest.mark.gpu

# (N, Cin, Cout, H, mode, operand, cin1, residual, sft, out planes, GroupNorm partials): as in test_gpu_wide_tiles
CASES = [
    (2, 64, 64, 32, 0, 'gnsilu', 0, True, False, False, True),
    (2, 128, 64, 32, 0, 'gnsilu', 0, False, False, True, True),
    (1, 256, 64, 32, 0, 'split', 0, True, False, False, True),
    (1, 128, 64, 32, 0, 'gnsilu', 64, False, True, False, True),
    (2, 64, 64, 16, 0, 'planes', 0, True, False, True, True),
    (1, 128, 64, 16, 0, 'planes', 0, False, True, False, False),
    (1, 128, 64, 16, 2, 'planes', 0, True, False, True, True),
    (2, 64, 64, 512, 0, 'gnsilu', 0, True, False, False, True),
]

KERNEL_CHILD = r'''
import ctypes, sys
import numpy as np, torch
sys.path.insert(0, %(root)r)
from codeformer_b200 import _lib
from tests.test_gpu_channel_major_tiles import CASES
from tests.test_gpu_wide_tiles import SFT_W, case_inputs, plane_bytes
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


@pytest.fixture(scope='module')
def kernel_results():
    with tempfile.TemporaryDirectory() as d:
        yield {bn: dict(_run(KERNEL_CHILD, bn, os.path.join(d, f'k{bn}.npz'))) for bn in ('64', None)}


@pytest.mark.parametrize('i', range(len(CASES)), ids=[_case_id(c) for c in CASES])
def test_channel_major_tiles_equal_pixel_major_tiles_torch_and_gn_moments(kernel_results, i):
    N, Cin, Cout, H, mode, operand, cin1, resid, sft, planes, gn = CASES[i]
    cm, pm = kernel_results[None], kernel_results['64']
    assert int(cm[f'tile{i}']) == -64 and int(pm[f'tile{i}']) == 64, 'the two sides must run channel- and pixel-major tiles'
    oc, op = cm[f'out{i}'], pm[f'out{i}']
    assert np.array_equal(_bits(oc), _bits(op)), f'channel-major tiles differ from pixel-major tiles by {np.abs(oc - op).max()}'
    ref = reference(CASES[i])
    assert maxabs(torch.from_numpy(oc).double(), ref) < 6e-5 * max(1.0, float(ref.abs().max()))
    if planes:
        pc = cm[f'planes{i}']
        assert np.array_equal(pc, pm[f'planes{i}']), 'operand planes differ'
        nb = plane_bytes(N, oc.shape[1], Cout)
        hi = pc[:nb].view(np.float16)[:oc.size].astype(np.float32)
        lo = pc[nb:].view(np.float16)[:oc.size].astype(np.float32)
        assert np.array_equal(hi, oc.reshape(-1).astype(np.float16).astype(np.float32))
        assert np.abs(hi + lo - oc.reshape(-1)).max() <= 2.0 ** -20 * max(1.0, float(np.abs(oc).max()))
    if gn:
        gc = cm[f'gn{i}']
        assert np.array_equal(_bits(gc), _bits(pm[f'gn{i}'])), 'GroupNorm partials differ'
        assert_gn_partials(gc, oc, N, Cout)
