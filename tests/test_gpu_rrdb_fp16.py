"""-m gpu: the single-pass fp16 precision of the generalised conv engine (RRDBNet / RealESRGANer ``precision='fp16'``).
Unit convs are compared with the float64 emulation of tests/fp16_emul.py (operands rounded as the kernel rounds them, so only
the accumulation order differs), whole networks with the reference golden vectors and the CPU oracle, against twice the error
the emulation itself makes there."""
import ctypes
import math

import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import _lib
from codeformer_b200 import spec as S
from tests import fp16_emul as E
from tests.util import golden, maxabs

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

FILL = -3.0


def _rand(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def _gen_conv(x_nchw, w, b, precision=None, up=0, pad_mode=0, sub=0, act=0, res=None, res2=None, post=1.0, in_pitch=None,
              out_pitch=None, out_c0=0):
    """One generalised conv on host tensors: cfb_conv2d_gen_nhwc_prec (precision 0 / 1), or cfb_conv2d_gen_nhwc when
    precision is None.  Returns the NCHW [out_c0, out_c0 + cout) slice and checks that the rest of the destination kept
    its fill."""
    lib = _lib.load()
    N, Cin, H, W = x_nchw.shape
    Cout = w.shape[0]
    in_pitch = in_pitch or Cin
    xin = torch.full((N, H, W, in_pitch), 7.25)                     # channels beyond cin hold finite junk (they meet zero weights)
    xin[..., :Cin] = x_nchw.permute(0, 2, 3, 1)
    xin = xin.cuda()
    Ho, Wo = (2 * H, 2 * W) if up else ((H // 2, W // 2) if sub else (H, W))
    out_pitch = out_pitch or Cout
    out = torch.full((N, Ho, Wo, out_pitch), FILL, device='cuda')
    wd, bd = w.contiguous().cuda(), (None if b is None else b.contiguous().cuda())
    rd = None if res is None else res.permute(0, 2, 3, 1).contiguous().cuda()
    r2d = None if res2 is None else res2.permute(0, 2, 3, 1).contiguous().cuda()
    wsb = lib.cfb_conv2d_gen_workspace_bytes(Cin, Cout)
    ws = torch.empty(int(wsb), dtype=torch.uint8, device='cuda')
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = (_lib.ptr(xin), in_pitch, _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(out), out_pitch, out_c0, N, H, W, Cin, Cout, up, pad_mode,
            sub, act, _lib.ptr(rd), Cout, _lib.ptr(r2d), Cout, post, _lib.ptr(ws), wsb, st)
    if precision is None:
        _lib.check(lib.cfb_conv2d_gen_nhwc(*args), 'cfb_conv2d_gen_nhwc')
    else:
        _lib.check(lib.cfb_conv2d_gen_nhwc_prec(*args, precision), 'cfb_conv2d_gen_nhwc_prec')
    torch.cuda.synchronize()
    cb.check_async_status()
    full = out.cpu()
    if out_pitch != Cout:
        mask = torch.ones(out_pitch, dtype=torch.bool)
        mask[out_c0:out_c0 + Cout] = False
        assert bool((full[..., mask] == FILL).all()), 'channels outside the destination slice were written'
    return full[..., out_c0:out_c0 + Cout].permute(0, 3, 1, 2).contiguous()


def _check_modes(x, w, b, **kw):
    """fp16 mode against the emulation (<= 2e-5 max|ref|); fp32 mode of the _prec entry point == cfb_conv2d_gen_nhwc bit for
    bit; and the two modes differ."""
    ekw = {k: v for k, v in kw.items() if k in ('pad_mode', 'act', 'res', 'res2', 'post')}
    ref = E.conv_layer(x, w, b, up=bool(kw.get('up', 0)), sub=bool(kw.get('sub', 0)), **ekw)
    got = _gen_conv(x, w, b, precision=1, **kw)
    err = maxabs(got, ref)
    print(f'fp16 vs emulation: max-abs {err:.3e} (|ref|max {float(ref.abs().max()):.3f})')
    assert got.shape == ref.shape and err <= 2e-5 * float(ref.abs().max())
    split = _gen_conv(x, w, b, precision=0, **kw)
    assert torch.equal(split, _gen_conv(x, w, b, **kw)), 'precision 0 is the existing entry point'
    assert not torch.equal(got, split), 'fp16 mode must take effect'


# (N, Cin, Cout, H, W, pad_mode): the shapes of test_gpu_aux.GEN_CASES (ragged tiles, dense-block windows, both paddings)
GEN_CASES = [(1, 64, 32, 20, 28, 0), (2, 96, 32, 17, 23, 0), (1, 160, 32, 40, 9, 0), (1, 192, 64, 33, 31, 0),
             (1, 64, 64, 24, 40, 1), (2, 128, 128, 19, 21, 1), (1, 256, 128, 16, 16, 1), (1, 64, 64, 50, 7, 2)]


@pytest.mark.parametrize('case', GEN_CASES)
def test_fp16_gen_conv_matches_emulation(case):
    """3x3 stride-1 conv, LeakyReLU, into a channel slice of a wider buffer (the dense-block placement)."""
    N, Cin, Cout, H, W, pm = case
    x = _rand(N, Cin, H, W, seed=1)
    w = _rand(Cout, Cin, 3, 3, seed=2, scale=1 / math.sqrt(9 * Cin))
    b = _rand(Cout, seed=3, scale=0.1)
    in_pitch = (Cin + 63) // 64 * 64 + (64 if Cin % 64 else 0)
    _check_modes(x, w, b, pad_mode=pm, act=1, in_pitch=in_pitch, out_pitch=Cout + 32, out_c0=16)


@pytest.mark.parametrize('pm', [0, 1])
def test_fp16_gen_conv_stride2_upsample_and_residuals(pm):
    N, C, H, W = 1, 64, 26, 18
    x = _rand(N, C, H, W, seed=4)
    w = _rand(128, C, 3, 3, seed=5, scale=1 / math.sqrt(9 * C))
    b = _rand(128, seed=6, scale=0.1)
    _check_modes(x, w, b, pad_mode=pm, sub=1)                                     # stride 2: even positions
    _check_modes(x, w, b, pad_mode=2 if pm == 1 else 0, up=1, act=1)             # nearest x2 + conv (four parity convs)
    w2 = _rand(64, C, 3, 3, seed=7, scale=1 / math.sqrt(9 * C))
    b2 = _rand(64, seed=8, scale=0.1)
    r1, r2 = _rand(N, 64, H, W, seed=9), _rand(N, 64, H, W, seed=10)
    _check_modes(x, w2, b2, pad_mode=pm, res=r1, res2=r2, post=0.2)              # (conv + b + r1) * 0.2 + r2


def _net(scale, num_block, sd, precision=None):
    net = cb.RRDBNet(3, 3, scale=scale, num_feat=64, num_block=num_block, num_grow_ch=32).cuda().eval()
    net.load_state_dict(sd, strict=True)
    if precision:
        net.set_precision(precision)
    return net


@pytest.mark.parametrize('case', ['s2', 's4'])
def test_rrdbnet_fp16_vs_reference_golden(case):
    """RRDBNet x2 / x4 (23 RRDBs) in fp16 mode against the reference's fp32 output: error <= 2x that of the float64 emulation
    of the whole network in single-pass fp16, + 1e-4."""
    from oracle import gen_golden as GG
    scale, sd, x = GG.rrdb_inputs(case)
    net = _net(scale, 23, sd, 'fp16')
    out = net(x.cuda())
    torch.cuda.synchronize()
    cb.check_async_status()
    ref = golden('rrdbnet.npz')[case + '_out']
    err = maxabs(out.cpu(), ref)
    err_emul = maxabs(E.rrdbnet_forward(sd, x, scale=scale, num_block=23), ref)
    print(f'rrdbnet {case} fp16: max-abs {err:.3e}, emulation {err_emul:.3e} (|out|max {float(np.abs(ref).max()):.2f})')
    assert out.shape == ref.shape and err <= 2 * err_emul + 1e-4
    assert torch.equal(net(x.cuda()), out), 'deterministic'


def test_rrdbnet_fp16_odd_sizes_batch_invariance_and_empty_batch():
    from oracle import rrdbnet_oracle as RO
    sd = S.random_state_dict(S.rrdbnet_spec(3, 3, 4, 64, 3, 32), 9)
    net = _net(4, 3, sd, 'fp16')
    x = torch.rand(3, 3, 37, 53, generator=torch.Generator().manual_seed(1))
    out = net(x.cuda())
    torch.cuda.synchronize()
    cb.check_async_status()
    ref = RO.rrdbnet_forward(sd, x, scale=4, num_block=3)
    err, err_emul = maxabs(out.cpu(), ref), maxabs(E.rrdbnet_forward(sd, x, scale=4, num_block=3), ref)
    print(f'rrdbnet 37x53 fp16: max-abs {err:.3e}, emulation {err_emul:.3e}')
    assert err <= 2 * err_emul + 1e-4
    assert torch.equal(net(x.cuda()), out), 'deterministic'
    assert torch.equal(net(x[1:2].cuda())[0], out[1]), 'images must not interact'
    e = net(torch.empty(0, 3, 8, 8, device='cuda'))
    assert e.shape == (0, 3, 32, 32)


def test_precision_switching_keeps_fp32_bits():
    sd = S.random_state_dict(S.rrdbnet_spec(3, 3, 2, 64, 2, 32), 5)
    x = torch.rand(2, 3, 34, 46, generator=torch.Generator().manual_seed(2)).cuda()
    net = _net(2, 2, sd)
    assert net.precision == 'fp32'
    a = net(x)
    assert net.set_precision('fp16') is net and net.precision == 'fp16'
    h = net(x)
    net.set_precision('fp32')
    b = net(x)
    assert torch.equal(a, b), 'fp32 -> fp16 -> fp32 must give the fp32 bits back'
    assert torch.equal(a, _net(2, 2, sd)(x)), 'a switched module equals a fresh fp32 module'
    assert torch.equal(h, _net(2, 2, sd, 'fp16')(x)), 'a fresh fp16 module equals a switched one'
    assert not torch.equal(a, h)
    # the setting survives load_state_dict (re-prepare) and .to()
    net.set_precision('fp16')
    net.load_state_dict(sd)
    net = net.to('cuda')
    assert net.precision == 'fp16' and torch.equal(net(x), h)


def test_realesrganer_fp16_tiles_equal_the_emulated_pipeline():
    """enhance(tile=32, tile_pad=8) with precision='fp16' against the same front-end around the float64 fp16 emulation: uint8
    values equal up to one LSB at rounding boundaries.  precision=None leaves the model (and the result) as it is."""
    sd = S.random_state_dict(S.rrdbnet_spec(3, 3, 2, 64, 2, 32), 11)
    img = np.random.default_rng(3).integers(0, 256, (75, 61, 3), dtype=np.uint8)

    class Emulated(torch.nn.Module):
        def forward(self, x):
            return E.rrdbnet_forward(sd, x, scale=2, num_block=2).float()

    def enhance(model, **kw):
        return cb.RealESRGANer(scale=2, model=model, tile=32, tile_pad=8, pre_pad=0, device=kw.pop('device', 'cuda'),
                               **kw).enhance(img, outscale=2)[0]
    net = _net(2, 2, sd).cpu()
    a = enhance(net, precision='fp16')
    assert net.precision == 'fp16'
    b = enhance(Emulated(), device='cpu')
    d = np.abs(a.astype(np.int32) - b.astype(np.int32))
    print(f'RealESRGANer fp16: {(d > 0).sum()} of {d.size} values differ by one')
    assert a.shape == (150, 122, 3) and d.max() <= 1 and (d > 0).mean() < 1e-3
    assert np.array_equal(enhance(net, precision=None), a) and net.precision == 'fp16', 'None keeps the model as it is'
    plain = _net(2, 2, sd)
    today = enhance(plain)
    assert np.array_equal(enhance(plain, precision=None), today) and plain.precision == 'fp32'
    assert np.array_equal(enhance(_net(2, 2, sd), precision='fp32'), today)


def test_precision_errors():
    net = _net(2, 1, S.random_state_dict(S.rrdbnet_spec(3, 3, 2, 64, 1, 32), 1))
    with pytest.raises(ValueError):
        net.set_precision('bf16')
    with pytest.raises(ValueError):
        net.set_precision(1)
    assert net.precision == 'fp32'
    with pytest.raises(ValueError):
        cb.RealESRGANer(scale=2, model=net, precision='half', device='cuda')
    lib = _lib.load()
    net(torch.rand(1, 3, 8, 8, device='cuda'))                  # creates the handle
    with pytest.raises(RuntimeError, match='precision'):
        _lib.check(lib.cfb_rrdb_set_precision(net._net, 2), 'cfb_rrdb_set_precision')
    x = _rand(1, 64, 12, 12, seed=1)
    w = _rand(64, 64, 3, 3, seed=2, scale=1 / 24)
    with pytest.raises(RuntimeError, match='precision'):
        _gen_conv(x, w, None, precision=2)
    with pytest.raises(RuntimeError, match='SiLU|single-pass'):
        _gen_conv(x, w, None, precision=1, act=4)


@pytest.mark.parametrize('precision', [0, 1])
def test_fp16_range_guard_reports_through_the_status_word(precision):
    """An activation beyond the fp16 range is reported as an error (the status word), in both modes; the context stays usable."""
    x = _rand(1, 64, 12, 12, seed=1)
    w = _rand(64, 64, 3, 3, seed=2, scale=1 / 24)
    ok = _gen_conv(x, w, None, precision=precision)
    big = x.clone()
    big[0, 5, 3, 4] = 1e5
    with pytest.raises(RuntimeError, match='fp16'):
        _gen_conv(big, w, None, precision=precision)
    cb.check_async_status()                                    # reported once, then cleared
    assert torch.equal(_gen_conv(x, w, None, precision=precision), ok)
