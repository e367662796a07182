"""Float64 model of the split-fp16 tensor-core arithmetic of the conv engine (DESIGN.md section 4), the error bar the GPU
tests hold every split form to, and the faults that bar has to catch.

Every operand is an fp16 pair x = hi + lo:
  * weights: hi + lo of w * 2^(14-e), one e = frexp(max|w|) per conv (fp16_emul.weight_exponent); Upsample convs split the
    fp32 parity sums of fp16_emul.up4_weights, one e over all 16 parity taps;
  * activations: hi + lo of the fp32 operand the MMAs read -- after the fused transform and the padding -- unscaled, so below
    |x| ~ 0.25 lo is an fp16 subnormal and the pair keeps fewer than 21 bits;
  * the products hi*hi + hi*lo + lo*hi; lo*lo is dropped.
``model`` returns that emulated conv with exact accumulation, the float64 reference conv(x, w), the per-output bound
B = conv(|x|, |w|) and the floor of subnormal lo: each operand is exact only to about 2^-25 * u (u = 1 for activations,
2^(e-14) for weights), so floor = 2^-25 * (conv(x != 0, |w|) + 2^(e-14) * conv(|x|, 1)).

``trunc=True``: a pessimistic model of the tensor core's accumulation at a sample of outputs.  Within a partial sum of
CHUNK = 8 k-blocks (64 input channels of one tap; channel block outer, tap inner, as the halo engine walks them) every k16
product group is added into an fp32 accumulator truncated toward zero, per k-step in the kernel's order lo*hi, hi*lo,
hi*hi; the partial sums are folded with round-to-nearest fp32 adds.  Convs of at most 12 k-blocks run as one partial sum.

``mutant`` drops part of the lo arithmetic as a fault in one code path of the kernels would (MUTANTS; CPU only, the kernels
have no such switch).  ``split_bar`` is the check: |out - ref| <= tau * B + floor at every output.
"""
import dataclasses

import numpy as np
import torch
import torch.nn.functional as F

from tests.fp16_emul import PADS, fp16_round, up4_weights, weight_exponent, weight_hi

CHUNK = 8
EPS = 2.0 ** -25
# no_lo: every lo product dropped;  tap / kblock: lo of one tap (Upsample: one of the 16 parity taps) / of the last 64-channel
# k-block of that tap;  cat: activation lo of the second concat source;  edge: activation lo of the image's outermost rows and
# columns (the border and the last, possibly ragged, tile row and column);  upper64: every lo product of output channels
# 64..127 of each 128-channel tile;  w_lo: the weight lo plane;  single_pass: fp16(x) * hi of the weights (fp16_emul's product)
MUTANTS = ('no_lo', 'tap', 'kblock', 'cat', 'edge', 'upper64', 'w_lo', 'single_pass')


@dataclasses.dataclass(frozen=True)
class Geometry:
    """How a conv reads its operand: ksize x ksize taps at ``stride`` on the operand padded by ``pad`` = (left, right, top,
    bottom) in ``pad_mode`` (0 zero / 1 reflect / 2 replicate); ``up``: nearest x2 first, run as four 2x2 parity convs on the
    low-resolution operand padded by 1; ``sub``: the even outputs of the stride-1 conv."""
    ksize: int = 3
    stride: int = 1
    pad: tuple = (1, 1, 1, 1)
    pad_mode: int = 0
    up: bool = False
    sub: bool = False


SAME3 = Geometry()
SAME1 = Geometry(ksize=1, pad=(0, 0, 0, 0))
DOWN = Geometry(stride=2, pad=(0, 1, 0, 1))          # Downsample: pad right / bottom 1, 3x3 stride 2
UP = Geometry(up=True)


def split(x):
    """fp32 values -> (hi, lo) as float64: hi = fp16(x), lo = fp16(x - hi) (round to nearest even, subnormals kept)."""
    x = x.float()
    hi = x.half()
    return hi.double(), (x - hi.float()).half().double()


def split_weights(w, up=False):
    """-> (hi, lo, e): the weight pair as unscaled float64 values, OIHW (up: [2, 2, Cout, Cin, 2, 2] parity weights)."""
    wf = up4_weights(w) if up else w.float()
    e = weight_exponent(wf)
    hi, lo = split(wf * 2.0 ** (14 - e))
    return hi * 2.0 ** (e - 14), lo * 2.0 ** (e - 14), e


def pad(x, g):
    """The padded operand (exact copies of fp32 values), NCHW."""
    x = x.float()
    if not any(g.pad):
        return x
    return F.pad(x, g.pad, mode=PADS[g.pad_mode]) if g.pad_mode else F.pad(x, g.pad)


def _conv(xp, w, g):
    """The conv the kernel computes on a padded operand, float64: parity convs for ``up``."""
    if g.up:
        N, _, Hp, Wp = xp.shape
        H, W = Hp - 2, Wp - 2
        y = xp.new_zeros(N, w.shape[2], 2 * H, 2 * W)
        for py in range(2):
            for px in range(2):
                y[:, :, py::2, px::2] = F.conv2d(xp[:, :, py:py + H + 1, px:px + W + 1], w[py, px])
        return y
    y = F.conv2d(xp, w, stride=g.stride)
    return y[..., ::2, ::2] if g.sub else y


def _ref_conv(xp, w, g):
    """The reference: nearest x2 of the padded low-resolution operand less its outer pixel, then the 3x3 conv, for ``up``."""
    if g.up:
        xp = xp.repeat_interleave(2, 2).repeat_interleave(2, 3)[..., 1:-1, 1:-1]
        return F.conv2d(xp, w)
    y = F.conv2d(xp, w, stride=g.stride)
    return y[..., ::2, ::2] if g.sub else y


def bounds(x, w, g=SAME3):
    """-> (ref, B, floor), NCHW float64: the float64 conv of the operand x (NCHW fp32 values; low resolution for ``up``) with
    w (OIHW, no bias), B = conv(|x|, |w|) and the floor of subnormal lo."""
    xp = pad(x, g).double()
    wd = w.double()
    e = weight_exponent(up4_weights(w.cpu()) if g.up else w)
    ref = _ref_conv(xp, wd, g)
    B = _ref_conv(xp.abs(), wd.abs(), g)
    floor = EPS * (_ref_conv((xp != 0).double(), wd.abs(), g) + 2.0 ** (e - 14) * _ref_conv(xp.abs(), torch.ones_like(wd), g))
    return ref, B, floor


def _trunc32(v):
    """float64 -> the fp32 value next to it toward zero, as float64."""
    f = v.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(v)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f.astype(np.float64)


def _classes(xp, w, g):
    """(patches [M, taps, Cin], weights [Cout, taps, Cin], output (y, x) slices, spatial shape) per output parity class."""
    N, C = xp.shape[:2]
    Co = w.shape[-4]
    if g.up:
        H, W = xp.shape[2] - 2, xp.shape[3] - 2
        for py in range(2):
            for px in range(2):
                pt = xp[:, :, py:py + H + 1, px:px + W + 1].unfold(2, 2, 1).unfold(3, 2, 1)
                yield (pt.permute(0, 2, 3, 4, 5, 1).reshape(-1, 4, C), w[py, px].reshape(Co, C, 4).permute(0, 2, 1),
                       (slice(py, None, 2), slice(px, None, 2)), (N, H, W))
        return
    k, s = g.ksize, 1 if g.sub else g.stride
    pt = xp.unfold(2, k, s).unfold(3, k, s)
    if g.sub:
        pt = pt[:, :, ::2, ::2]
    shape = (N, pt.shape[2], pt.shape[3])
    yield (pt.permute(0, 2, 3, 4, 5, 1).reshape(-1, k * k, C), w.reshape(Co, C, k * k).permute(0, 2, 1),
           (slice(None), slice(None)), shape)


def _truncating(out, xh, xl, wh, wx, wl, e, g, samples):
    """Overwrite ``samples`` outputs of each parity class of ``out`` with the truncating accumulation model."""
    s = 2.0 ** (14 - e)
    for (ph, wh_t, sl, shape), (pl_, wx_t, _, _), (_, wl_t, _, _) in zip(_classes(xh, wh, g), _classes(xl, wx, g),
                                                                         _classes(xh, wl, g)):
        M, T, C = ph.shape
        idx = np.unique(np.r_[np.linspace(0, M - 1, min(M, samples)).astype(np.int64), M - 1])
        Cp = (C + 63) // 64 * 64
        def prep(t, scale=1.0):                                          # noqa: E306
            t = t.numpy() * scale
            return np.pad(t, [(0, 0)] * (t.ndim - 1) + [(0, Cp - C)])
        a_hi, a_lo = prep(ph[idx]), prep(pl_[idx])
        b_hi, b_x, b_lo = prep(wh_t, s), prep(wx_t, s), prep(wl_t, s)
        nit = T * (Cp // 64)
        chunk = nit if nit <= 12 else CHUNK
        run = np.zeros((len(idx), b_hi.shape[0]))
        part = None
        for it in range(nit):
            kb, t = divmod(it, T)
            if it % chunk == 0:
                part = np.zeros_like(run)
            for k in range(4):
                c = slice(kb * 64 + 16 * k, kb * 64 + 16 * k + 16)
                for a, b in ((a_lo, b_x), (a_hi, b_lo), (a_hi, b_hi)):
                    part = _trunc32(part + a[:, t, c] @ b[:, t, c].T)
            if it % chunk == chunk - 1 or it == nit - 1:
                run = (run + part).astype(np.float32).astype(np.float64)
        n, y, x = np.unravel_index(idx, shape)
        view = out[:, :, sl[0], sl[1]]
        view[n, :, y, x] = torch.from_numpy(run / s)


def model(x, w, g=SAME3, mutant=None, cin1=0, trunc=False, samples=96):
    """The emulated conv of the operand x (NCHW fp32 values, low resolution for ``up``) with w (OIHW, no bias), float64 NCHW,
    with the lo arithmetic of ``mutant`` dropped; ``trunc``: the truncating accumulation at ``samples`` outputs per parity
    class (exact accumulation elsewhere).  ``cin1``: first channel of the second concat source."""
    xp = pad(x, g)
    if mutant == 'single_pass':
        return _conv(fp16_round(xp), weight_hi(up4_weights(w) if g.up else w), g)
    xh, xl = split(xp)
    wh, wl, e = split_weights(w, g.up)
    wx = wh                                              # the weights the activation lo multiplies
    if mutant == 'no_lo':
        xl, wl = torch.zeros_like(xl), torch.zeros_like(wl)
    elif mutant == 'w_lo':
        wl = torch.zeros_like(wl)
    elif mutant in ('tap', 'kblock'):
        C = w.shape[1]
        c = slice(None) if mutant == 'tap' else slice((C - 1) // 64 * 64, C)
        m = torch.ones_like(wh)
        k = wh.shape[-1]
        if g.up:
            m[0, 0, :, c, 1, 1] = 0
        else:
            m[:, c, k // 2, k // 2] = 0
        wx, wl = wh * m, wl * m
    elif mutant == 'cat':
        xl = xl.clone()
        xl[:, cin1:] = 0
    elif mutant == 'edge':
        xl = xl.clone()
        t, l = g.pad[2], g.pad[0]
        H, W = x.shape[2], x.shape[3]
        xl[:, :, [t, t + H - 1], :] = 0
        xl[:, :, :, [l, l + W - 1]] = 0
    elif mutant not in (None, 'upper64'):
        raise ValueError(mutant)
    out = _conv(xh, wh, g) + _conv(xl, wx, g) + _conv(xh, wl, g)
    if trunc:
        _truncating(out, xh, xl, wh, wx, wl, e, g, samples)
    if mutant == 'upper64':
        hi_only = _conv(xh, wh, g)
        ch = (torch.arange(out.shape[1]) % 128) >= 64
        out[:, ch] = hi_only[:, ch]
    return out


@dataclasses.dataclass
class Bar:
    """Outcome of split_bar: the worst err / (tau * B + floor), its position (n, y, x, c of an NHWC output) and the tile."""
    worst: float
    where: tuple
    tile: object = None

    @property
    def ok(self):
        return self.worst <= 1.0

    def __str__(self):
        return f'worst err/(tau*B+floor) {self.worst:.3g} at (n, y, x, c) = {self.where}, tile {self.tile}'


def split_bar(out, ref, B, floor, tau, tile=None):
    """|out - ref| <= tau * B + floor at every output (arrays of one shape; NaN fails).  -> Bar; ``.ok`` is the verdict."""
    out, ref, B, floor = (t.double() if torch.is_tensor(t) else torch.as_tensor(np.asarray(t)).double()
                          for t in (out, ref, B, floor))
    r = (out - ref).abs() / (tau * B + floor)
    r = torch.where(torch.isnan(r), torch.full_like(r, float('inf')), r)
    i = int(r.argmax())
    return Bar(float(r.reshape(-1)[i]), tuple(int(v) for v in np.unravel_index(i, tuple(r.shape))), tile)


# ---- operands ----

def random_operand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def push_lo(mag, sign, seed):
    """|values| -> sign * values whose lo is at least 0.3 ulp of their hi with the sign of ``sign`` (fp32)."""
    g = torch.Generator().manual_seed(seed)
    hi = mag.float().half().float()
    ulp = torch.where(hi >= 2.0 ** -14, 2.0 ** (torch.floor(torch.log2(hi.clamp_min(2.0 ** -14))) - 10), torch.full_like(hi, 2.0 ** -24))
    u = 0.3 + 0.19 * torch.rand(hi.shape, generator=g)
    return sign * (hi + u * ulp)


def aligned_operands(x_shape, w_shape, seed, x_scale=1.0, w_scale=1.0):
    """Sign-aligned x (NCHW) and w (OIHW): every product x[ci] * w[:, ci] and every lo product has the sign sigma[ci] *
    sigma[ci] = +1, and every lo is >= 0.3 ulp, so a lost lo product shows at full size."""
    g = torch.Generator().manual_seed(seed)
    sigma = torch.where(torch.rand(x_shape[1], generator=g) < 0.5, -1.0, 1.0)
    x = push_lo(torch.randn(*x_shape, generator=g).abs() * x_scale, sigma.view(1, -1, 1, 1), seed + 1)
    w = torch.randn(*w_shape, generator=g).abs() * w_scale
    e = weight_exponent(w)
    w = push_lo(w * 2.0 ** (14 - e), sigma.view(1, -1, 1, 1), seed + 2) * 2.0 ** (e - 14)
    return x.float(), w.float()
