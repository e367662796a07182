"""CPU emulation of the single-pass fp16 precision of the generalised conv engine (RRDBNet ``precision='fp16'``, DESIGN.md
section 4): every operand rounded as the kernel rounds it, products and sums in float64.  What it leaves out is only the
kernel's fp32 accumulation order.  Pinned by tests/test_fp16_single_pass_cpu.py; the GPU tests compare against it.

  * weights: the hi plane of the split, fp16(w * 2^(14-e)) * 2^(e-14) with e from frexp(max|w|) of the whole (padded) conv;
  * Upsample convs (nearest x2 + 3x3) run as four 2x2 parity convs whose weights are the 3x3 taps pre-summed in fp32, so the
    rounding applies to those sums (and e to their maximum);
  * activations: fp16(x) of the conv input, after the padding (reflect / replicate copy rounded values, zero stays zero).
"""
import math

import torch
import torch.nn.functional as F

PADS = {0: 'constant', 1: 'reflect', 2: 'replicate'}


def fp16_round(x):
    return x.float().half().double()


def weight_exponent(w):
    """e = frexp(max|w|) of the whole conv (tc_split_weights): the split scales the weights by 2^(14-e)."""
    amax = float(w.float().abs().max()) if w.numel() else 0.0
    return math.frexp(amax)[1] if amax > 0 and math.isfinite(amax) else 0


def weight_hi(w):
    """Hi plane of the split weights as float64 values: fp16(w * 2^(14-e)) * 2^(e-14), e = frexp(max|w|) (tc_split_weights)."""
    e = weight_exponent(w)
    return (w.float() * 2.0 ** (14 - e)).half().double() * 2.0 ** (e - 14)


# rows (columns) of the 3x3 kernel a 2x2 parity tap d sums for output parity 0 / 1 (up4_range in conv_tc.cu)
_UP4 = {0: ((0, 0), (1, 2)), 1: ((0, 1), (2, 2))}


def up4_weights(w):
    """[2, 2, Cout, Cin, 2, 2] fp32 parity weights W'[py][px][:, :, dy, dx]: the 3x3 taps reading the same low-resolution
    pixel, summed in fp32 in the kernel's order (rows outer, columns inner, from 0)."""
    w = w.float()
    out = torch.zeros(2, 2, w.shape[0], w.shape[1], 2, 2, dtype=torch.float32)
    for py in range(2):
        for px in range(2):
            for dy in range(2):
                for dx in range(2):
                    r0, r1 = _UP4[py][dy]
                    s0, s1 = _UP4[px][dx]
                    v = torch.zeros(w.shape[:2], dtype=torch.float32)
                    for r in range(r0, r1 + 1):
                        for q in range(s0, s1 + 1):
                            v = v + w[:, :, r, q]
                    out[py, px, :, :, dy, dx] = v
    return out


def up4_weights_hi(w):
    """up4_weights rounded like tc_split_weights_up4: one exponent over all 16 parity taps, rounded after summing."""
    return weight_hi(up4_weights(w))


def conv3x3(x, w, pad_mode=0, up=False, sub=False):
    """The conv alone (no bias) as the single-pass kernel computes it, in float64.  x [N, Cin, H, W] (low resolution when
    ``up``), w [Cout, Cin, 3, 3].  ``up``: nearest x2 then the conv, padding ``pad_mode`` of the low-resolution tensor;
    ``sub``: the even output positions (stride 2)."""
    xp = fp16_round(F.pad(x.float(), (1, 1, 1, 1), mode=PADS[pad_mode]))
    if not up:
        y = F.conv2d(xp, weight_hi(w))
        return y[..., ::2, ::2] if sub else y
    N, _, H, W = x.shape
    wu = up4_weights_hi(w)
    y = torch.empty(N, w.shape[0], 2 * H, 2 * W, dtype=torch.float64)
    for py in range(2):
        for px in range(2):
            y[:, :, py::2, px::2] = F.conv2d(xp[:, :, py:py + H + 1, px:px + W + 1], wu[py, px])
    return y


def conv_layer(x, w, b, pad_mode=0, up=False, sub=False, act=0, res=None, res2=None, post=1.0):
    """One generalised conv: act(conv + bias + res) * post + res2 (act 0 none / 1 LeakyReLU(0.2) / 3 ReLU), float64."""
    y = conv3x3(x, w, pad_mode, up, sub)
    if b is not None:
        y = y + b.double().view(1, -1, 1, 1)
    if res is not None:
        y = y + res.double()
    if act == 1:
        y = F.leaky_relu(y, 0.2)
    elif act == 3:
        y = F.relu(y)
    if res2 is not None:
        y = y * post + res2.double()
    return y


def _pixel_unshuffle(x, s):
    b, c, hh, hw = x.shape
    return x.view(b, c, hh // s, s, hw // s, s).permute(0, 1, 3, 5, 2, 4).reshape(b, c * s * s, hh // s, hw // s)


def rrdbnet_forward(sd, x, scale=4, num_block=23):
    """RRDBNet.forward (oracle/rrdbnet_oracle.py) with every GEN conv emulated in single-pass fp16; conv_first and conv_last
    stay exact (the kernel keeps them fp32).  float64 throughout."""
    sd = {k: v.double() for k, v in sd.items()}
    x = x.double()
    conv = lambda n, t, **kw: conv_layer(t, sd[n + '.weight'], sd[n + '.bias'], **kw)    # noqa: E731
    exact = lambda n, t: F.conv2d(t, sd[n + '.weight'], sd[n + '.bias'], padding=1)      # noqa: E731
    feat = _pixel_unshuffle(x, 2) if scale == 2 else (_pixel_unshuffle(x, 4) if scale == 1 else x)
    feat = exact('conv_first', feat)
    body = feat
    for b in range(num_block):
        out = body
        for r in range(1, 4):
            p, t = f'body.{b}.rdb{r}', out
            xs = [t]
            for k in range(1, 5):
                xs.append(conv(f'{p}.conv{k}', torch.cat(xs, 1), act=1))
            out = conv(f'{p}.conv5', torch.cat(xs, 1)) * 0.2 + t
        body = out * 0.2 + body
    feat = feat + conv('conv_body', body)
    feat = conv('conv_up1', feat, up=True, act=1)
    feat = conv('conv_up2', feat, up=True, act=1)
    return exact('conv_last', conv('conv_hr', feat, act=1))
