"""CPU checks of tests/fp16_emul.py, the float64 model of the single-pass fp16 GEN conv that the GPU tests compare against:
its weight rounding is the hi plane of the split scheme, its Upsample form is the pre-summed parity conv rounded after the
sum, and its error against the exact conv stays inside the analytic fp16 bound."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import fp16_emul as E

U = 2.0 ** -11          # unit roundoff of fp16 round-to-nearest


def _rand(*shape, seed, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


@pytest.mark.parametrize('scale', [0.02, 3.0, 1e-5])
def test_weight_rounding_is_the_hi_plane_of_the_split(scale):
    w = _rand(64, 96, 3, 3, seed=1, scale=scale)
    wn = w.numpy()
    e = int(np.frexp(np.abs(wn).max())[1])
    s = np.float32(2.0 ** (14 - e))
    hi = (wn * s).astype(np.float16)
    lo = (wn * s - hi.astype(np.float32)).astype(np.float16)
    assert 2.0 ** 13 <= np.abs(wn * s).max() < 2.0 ** 14
    got = E.weight_hi(w).numpy()
    assert np.array_equal(got, hi.astype(np.float64) * 2.0 ** (e - 14))
    # the split path reads hi + lo of the same planes: the single pass drops lo only
    assert np.abs(hi.astype(np.float64) + lo.astype(np.float64) - wn.astype(np.float64) * s).max() <= 2.0 ** -8
    assert not np.array_equal(got, wn.astype(np.float64))


def test_upsample_form_is_the_presummed_parity_conv_rounded_after_summing():
    # on fp16-exact operands the parity form equals nearest x2 + zero-padded 3x3 conv bit for bit
    x = torch.randint(-8, 9, (2, 5, 6, 7), generator=torch.Generator().manual_seed(2)).double() / 4
    w = torch.randint(-8, 9, (4, 5, 3, 3), generator=torch.Generator().manual_seed(3)).double() / 64
    ref = F.conv2d(F.interpolate(x, scale_factor=2, mode='nearest'), w, padding=1)
    assert torch.equal(E.conv3x3(x, w, up=True), ref)
    # reflect padding after the upsample is replicate padding before it
    ref = F.conv2d(F.pad(F.interpolate(x, scale_factor=2, mode='nearest'), (1, 1, 1, 1), mode='reflect'), w)
    assert torch.equal(E.conv3x3(x, w, pad_mode=2, up=True), ref)
    # general weights: the 16 parity taps are summed in fp32 first, then rounded with one exponent over all of them
    w = _rand(8, 16, 3, 3, seed=4, scale=0.05)
    wu = E.up4_weights(w)
    assert torch.equal(wu[0, 0, :, :, 1, 1], ((w[:, :, 1, 1] + w[:, :, 1, 2]) + w[:, :, 2, 1]) + w[:, :, 2, 2])
    assert torch.equal(wu[1, 0, :, :, 0, 1], (w[:, :, 0, 1] + w[:, :, 0, 2]) + w[:, :, 1, 1] + w[:, :, 1, 2])
    assert torch.equal(E.up4_weights_hi(w), E.weight_hi(wu))
    # rounding the 3x3 weights before summing is a different model
    hw = E.weight_hi(w)
    pre = hw[:, :, 1, 1] + hw[:, :, 1, 2] + hw[:, :, 2, 1] + hw[:, :, 2, 2]
    assert not torch.equal(pre, E.up4_weights_hi(w)[0, 0, :, :, 1, 1])


@pytest.mark.parametrize('form', ['same_zero', 'same_reflect', 'sub', 'up'])
def test_error_within_the_analytic_fp16_bound(form):
    """|single pass - exact| <= 2 * 2^-11 * sum |w| |x| (each operand rounded once, products and sums exact)."""
    N, Cin, Cout, H, W = 2, 96, 32, 13, 18
    x = _rand(N, Cin, H, W, seed=5, scale=2.0).double()
    w = _rand(Cout, Cin, 3, 3, seed=6, scale=1 / math.sqrt(9 * Cin)).double()
    pm = 1 if form == 'same_reflect' else 0
    up, sub = form == 'up', form == 'sub'
    got = E.conv3x3(x, w, pad_mode=pm, up=up, sub=sub)
    xi = F.interpolate(x, scale_factor=2, mode='nearest') if up else x
    xp = F.pad(xi, (1, 1, 1, 1), mode=E.PADS[pm])
    exact, mag = F.conv2d(xp, w), F.conv2d(xp.abs(), w.abs())
    if sub:
        exact, mag = exact[..., ::2, ::2], mag[..., ::2, ::2]
    err = (got - exact).abs()
    assert got.shape == exact.shape
    assert bool((err <= 2 * U * mag).all())
    assert float(err.max()) > 1e-2 * U * float(mag.max())          # and the rounding did take place
