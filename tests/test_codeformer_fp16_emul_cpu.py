"""CPU checks of tests/codeformer_fp16_emul.py, the float64 model of CodeFormer's fp16 mode that the GPU tests compare
against: at a small configuration its generator (with a fusion block) equals a direct restatement and stays close to the exact
float64 generator; at the real size its logits, lq_feat and code indices are the fp32 oracle's bit for bit, and its error
against the reference golden is the one stored in tests/golden/codeformer_fp16.npz."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from codeformer_b200 import spec as S
from oracle import codeformer_oracle as O
from tests import codeformer_fp16_emul as CE
from tests import fp16_emul as E
from tests.util import faces_input, golden, maxabs

torch.set_grad_enabled(False)

# a small generator: conv_in, ResBlocks with and without conv_out, AttnBlocks, an Upsample, the final norm + conv
SMALL = dict(nf=32, ch_mult=(1, 2), res_blocks=1, resolution=32, attn_resolutions=(16,), emb_dim=32)
FUSE_AT, FUSE_C = 7, 32                       # a Fuse_sft_block after block 7 (the 32-channel ResBlock at 32 x 32)


def _small_sd():
    spec = S.vqae_spec(img_size=32, nf=32, ch_mult=(1, 2), res_blocks=1, attn_resolutions=(16,), codebook_size=16, emb_dim=32)
    sd = {k: v for k, v in S.random_state_dict(spec, 5).items() if k.startswith('generator.')}
    g = torch.Generator().manual_seed(6)
    p = 'fuse_convs_dict.t'
    shapes = {'.encode_enc.norm1': (2 * FUSE_C,), '.encode_enc.norm2': (FUSE_C,)}
    for n in ('.encode_enc.conv1', '.encode_enc.conv2', '.encode_enc.conv_out', '.scale.0', '.scale.2', '.shift.0', '.shift.2'):
        cin = 2 * FUSE_C if n in ('.encode_enc.conv1', '.encode_enc.conv_out') else FUSE_C
        k = 1 if n.endswith('conv_out') else 3
        sd[p + n + '.weight'] = torch.randn(FUSE_C, cin, k, k, generator=g) / math.sqrt(cin * k * k)
        sd[p + n + '.bias'] = 0.1 * torch.randn(FUSE_C, generator=g)
    for n, shp in shapes.items():
        sd[p + n + '.weight'] = 1 + 0.1 * torch.randn(shp, generator=g)
        sd[p + n + '.bias'] = 0.1 * torch.randn(shp, generator=g)
    return CE.decoder_sd(sd)


def _direct(sd, x, enc, w):
    """The fp16 mode restated op by op: every decoder conv except the AttnBlocks' and the last one reads fp16(input) and the
    hi weight plane fp16(w * 2^(14-e)) * 2^(e-14); the Upsample conv runs as its four 2x2 parity convs."""
    def hi(t):
        e = math.frexp(float(t.float().abs().max()))[1]
        return (t.float() * 2.0 ** (14 - e)).half().double() * 2.0 ** (e - 14)

    def r16(t):
        return t.float().half().double()

    def conv(p, t, pad=1):
        return F.conv2d(r16(t), hi(sd[p + '.weight']), sd[p + '.bias'], padding=pad)

    def gn_silu(p, t):
        return F.silu(F.group_norm(t, 32, sd[p + '.weight'], sd[p + '.bias'], eps=1e-6))

    def res(p, t):
        h = conv(p + '.conv2', gn_silu(p + '.norm2', conv(p + '.conv1', gn_silu(p + '.norm1', t))))
        return h + (conv(p + '.conv_out', t, 0) if p + '.conv_out.weight' in sd else t)

    def up(p, t):
        wu = E.up4_weights_hi(sd[p + '.conv.weight'])
        tp = r16(F.pad(t, (1, 1, 1, 1)))
        N, _, H, W = t.shape
        y = torch.zeros(N, wu.shape[2], 2 * H, 2 * W, dtype=torch.float64)
        for py in range(2):
            for px in range(2):
                for dy in range(2):
                    for dx in range(2):
                        win = tp[:, :, py + dy:py + dy + H, px + dx:px + dx + W]
                        y[:, :, py::2, px::2] += torch.einsum('nchw,oc->nohw', win, wu[py, px, :, :, dy, dx])
        return y + sd[p + '.conv.bias'].view(1, -1, 1, 1)

    g = 'generator.blocks.'
    x = conv(g + '0', x)
    x = res(g + '1', x)
    x = O.attnblock(sd, g + '2', x)
    x = res(g + '3', x)
    x = res(g + '4', x)
    x = O.attnblock(sd, g + '5', x)
    x = up(g + '6', x)
    x = res(g + '7', x)
    f = 'fuse_convs_dict.t'
    e = res(f + '.encode_enc', torch.cat([enc, x], 1))
    scale = conv(f + '.scale.2', F.leaky_relu(conv(f + '.scale.0', e), 0.2))
    shift = conv(f + '.shift.2', F.leaky_relu(conv(f + '.shift.0', e), 0.2))
    x = x + w * (x * scale + shift)
    x = F.group_norm(x, 32, sd[g + '8.weight'], sd[g + '8.bias'], eps=1e-6)
    return F.conv2d(x, sd[g + '9.weight'], sd[g + '9.bias'], padding=1)


def test_small_generator_equals_a_direct_restatement_and_stays_near_the_exact_one():
    sd = _small_sd()
    plan = O.generator_plan(**SMALL)
    assert [k for k, _, _ in plan] == ['conv', 'res', 'attn', 'res', 'res', 'attn', 'up', 'res', 'norm', 'conv']
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, 32, 16, 16, generator=g)
    enc = torch.randn(2, FUSE_C, 32, 32, generator=g).double()
    got = CE.generator_forward(sd, x, plan=plan, fuse={FUSE_AT: ('fuse_convs_dict.t', enc)}, w=0.5)
    ref = _direct(sd, x.double(), enc, 0.5)
    assert got.shape == (2, 3, 32, 32)
    assert maxabs(got, ref) <= 1e-12 * float(ref.abs().max())
    # the exact float64 generator + fusion: the fp16 operands move the output, by about the fp16 unit roundoff
    xe = x.double()
    for i, (kind, _, _) in enumerate(plan):
        xe = O.run_block(sd, f'generator.blocks.{i}', kind, xe)
        if i == FUSE_AT:
            xe = O.fuse_sft(sd, 'fuse_convs_dict.t', enc, xe, 0.5)
    rel = maxabs(got, xe) / float(xe.abs().max())
    print(f'small generator: fp16 emulation vs exact float64, max-abs relative {rel:.2e}')
    assert 1e-6 < rel < 2e-2
    # without the fusion (w = 0) the fusion parameters are not read
    assert torch.equal(CE.generator_forward(sd, x, plan=plan, fuse={FUSE_AT: ('fuse_convs_dict.t', enc)}, w=0.0),
                       CE.generator_forward(sd, x, plan=plan))


def test_full_size_codes_are_the_fp32_oracles_and_the_error_is_the_stored_one():
    sd = S.random_state_dict(S.codeformer_spec(), 1)
    x = faces_input(slice(0, 1))
    out, logits, lq, idx = CE.codeformer_forward(sd, x, w=0.5, adain_on=True)
    ol, oq = O.codeformer_forward(sd, x, w=0.5, adain_on=True, code_only=True)
    assert torch.equal(logits, ol) and torch.equal(lq, oq), 'encoder and Transformer are the fp32 oracle'
    g = golden('codeformer_main.npz')
    assert np.array_equal(idx[..., 0].numpy(), g['top_idx']) and torch.equal(idx[..., 0], ol.argmax(2))
    err, stored = maxabs(out, g['out']), float(golden('codeformer_fp16.npz')['main_err'])
    print(f'main config: emulated fp16 out vs reference golden max-abs {err:.4e} (stored {stored:.4e})')
    assert abs(err - stored) <= 1e-6 * stored
    assert out.dtype == torch.float64 and out.shape == (1, 3, 512, 512)
