"""Float64 emulation of ParseNet in its fp16 precision (``ParseNet.set_precision('fp16')``), composed from tests/fp16_emul.py:
every GEN conv (shortcut, conv1, conv2 of the encoder, body and decoder blocks) has its operands rounded as the single-pass
kernel rounds them; encoder.0 and the heads stay exact, as the kernel keeps them fp32.  Eval-mode BatchNorm is folded into the
conv in fp32 first, as ``fold_bn_kernel`` does at prepare, and the folded weights are what the weight split rounds.  Runs on
the device of ``x`` (float64 convs), so the 512 configuration is cheap on a GPU.  ``rounding=False`` gives the same forms with
exact float64 convs: that is the reference network, which tests/test_parsenet_fp16_emul_cpu.py pins against the oracle.
"""
import torch
import torch.nn.functional as F

from tests import fp16_emul as E


def fold_bn(sd, p, eps=1e-5):
    """fold_bn_kernel in fp32: s = gamma / sqrt(var + eps), w' = w * s, b' = beta - mean * s."""
    q = p + '.norm.norm.'
    w = sd[p + '.conv2d.weight'].float()
    s = sd[q + 'weight'].float() / torch.sqrt(sd[q + 'running_var'].float() + eps)
    return w * s.view(-1, 1, 1, 1), sd[q + 'bias'].float() - sd[q + 'running_mean'].float() * s


def conv3x3(x, w, pad_mode=0, up=False, sub=False, rounding=True):
    """fp16_emul.conv3x3 on the device of x (the weights are rounded on the host, then moved).  rounding=False: the exact
    float64 conv of the same form (nearest x2 before the padding when ``up``)."""
    dev = x.device
    if not rounding:
        xi = F.interpolate(x.double(), scale_factor=2, mode='nearest') if up else x.double()
        y = F.conv2d(F.pad(xi, (1, 1, 1, 1), mode=E.PADS[1 if up and pad_mode == 2 else pad_mode]), w.double().to(dev))
        return y[..., ::2, ::2] if sub else y
    xp = E.fp16_round(F.pad(x.float(), (1, 1, 1, 1), mode=E.PADS[pad_mode]))
    if not up:
        y = F.conv2d(xp, E.weight_hi(w.cpu()).to(dev))
        return y[..., ::2, ::2] if sub else y
    N, _, H, W = x.shape
    wu = E.up4_weights_hi(w.cpu()).to(dev)
    y = torch.empty(N, w.shape[0], 2 * H, 2 * W, dtype=torch.float64, device=dev)
    for py in range(2):
        for px in range(2):
            y[:, :, py::2, px::2] = F.conv2d(xp[:, :, py:py + H + 1, px:px + W + 1], wu[py, px])
    return y


def conv_layer(x, w, b, pad_mode=0, up=False, sub=False, act=0, res=None, res2=None, post=1.0, rounding=True):
    """fp16_emul.conv_layer with ``conv3x3`` above: act(conv + bias + res) * post + res2, float64."""
    y = conv3x3(x, w, pad_mode, up, sub, rounding)
    if b is not None:
        y = y + b.double().to(x.device).view(1, -1, 1, 1)
    if res is not None:
        y = y + res.double()
    if act == 1:
        y = F.leaky_relu(y, 0.2)
    if res2 is not None:
        y = y * post + res2.double()
    return y


def _exact(sd, p, x):
    """encoder.0 / the heads: ReflectionPad2d(1) + 3x3 conv, exact (fp32 SIMT in the kernel)."""
    dev = x.device
    return F.conv2d(F.pad(x, (1, 1, 1, 1), mode='reflect'), sd[p + '.conv2d.weight'].double().to(dev),
                    sd[p + '.conv2d.bias'].double().to(dev))


def parsenet_forward(sd, x, plan, rounding=True, return_img=False):
    """ParseNet.forward (oracle/parsenet_oracle.py) with the GEN convs as the fp16 precision computes them, in the kernel's
    forms: 'down' = stride-1 conv then the even positions, 'up' = parity convs with replicate padding of the low-resolution
    tensor, the residual sums as epilogue terms.  plan: codeformer_b200.parsing.parsenet_plan(...)[0].  -> logits [, img]."""
    x = x.double()
    n_body = sum(1 for p, *_ in plan if p.startswith('body'))
    seen_body = 0

    def gen(p, t, bn, **kw):
        w, b = fold_bn(sd, p) if bn else (sd[p + '.conv2d.weight'].float(), sd[p + '.conv2d.bias'].float())
        return conv_layer(t, w, b, rounding=rounding, **kw)

    t = _exact(sd, 'encoder.0', x)
    feat = None
    for p, kind, cin, cout in plan:
        if p.startswith('body') and feat is None:
            feat = t
        if kind == 'down':
            s = gen(p + '.shortcut_func', t, False, pad_mode=1, sub=True)
            c1 = gen(p + '.conv1', t, True, pad_mode=1, act=1)
            t = gen(p + '.conv2', c1, True, pad_mode=1, sub=True, res=s)
        elif kind == 'up':
            s = gen(p + '.shortcut_func', t, False, pad_mode=2, up=True)
            c1 = gen(p + '.conv1', t, True, pad_mode=2, up=True, act=1)
            t = gen(p + '.conv2', c1, True, pad_mode=1, res=s)
        else:
            seen_body += 1
            last = seen_body == n_body
            c1 = gen(p + '.conv1', t, True, pad_mode=1, act=1)
            t = gen(p + '.conv2', c1, True, pad_mode=1, res=t, res2=feat if last else None)
    logits = _exact(sd, 'out_mask_conv', t)
    return (logits, _exact(sd, 'out_img_conv', t)) if return_img else logits
