"""CPU emulation of CodeFormer / VQAutoEncoder with ``set_precision('fp16')`` (DESIGN.md section 4), built on the fp32
oracle (oracle/codeformer_oracle.py) and the operand rounding of tests/fp16_emul.py.  Pinned by
tests/test_codeformer_fp16_emul_cpu.py; tools/gen_codeformer_fp16_golden.py stores what the GPU tests compare against.

  * encoder, Transformer, code lookup / quantizer and AdaIN: the fp32 oracle itself.  The library keeps them on the split
    path in both precisions, so logits, lq_feat and the code indices are those of the fp32 mode;
  * every conv of the generator blocks and of the Fuse_sft_blocks except the AttnBlocks' q, k, v, proj_out and the last conv:
    the single-pass kernel's operands -- fp16(x) of the conv input (after GroupNorm + SiLU where the block has them), the hi
    weight plane ``weight_hi`` (Upsample: the four 2x2 parity convs with ``up4_weights_hi``) -- with products and sums in
    float64;
  * the rest of the decoder (GroupNorm, SiLU, AttnBlocks, residual adds, LeakyReLU, SFT, the last conv) exact in float64.
What it leaves out is the kernel's fp32 accumulation order and its fp32 GroupNorm / SiLU / activation storage.
"""
import torch
import torch.nn.functional as F

from oracle import codeformer_oracle as O
from tests.fp16_emul import conv3x3, fp16_round, weight_hi

DECODER = ('generator.', 'fuse_convs_dict.')


def decoder_sd(sd):
    """The generator and fusion parameters in float64 (the emulation's working copy)."""
    return {k: v.double() for k, v in sd.items() if k.startswith(DECODER)}


def conv(sd, p, x, padding=1):
    """A single-pass conv (3x3, or 1x1 with padding 0): fp16(x) * weight_hi(w) + bias, float64."""
    return F.conv2d(fp16_round(x), weight_hi(sd[p + '.weight']), sd[p + '.bias'], padding=padding)


def upsample(sd, p, x):
    """Upsample (nearest x2 + 3x3) as the kernel runs it: four 2x2 parity convs on fp16(x) with the pre-summed weights."""
    return conv3x3(x, sd[p + '.conv.weight'], up=True) + sd[p + '.conv.bias'].view(1, -1, 1, 1)


def resblock(sd, p, x_in):
    """ResBlock.forward (vqgan_arch.py:153-164) with single-pass convs."""
    x = conv(sd, p + '.conv1', O.swish(O.group_norm(sd, p + '.norm1', x_in)))
    x = conv(sd, p + '.conv2', O.swish(O.group_norm(sd, p + '.norm2', x)))
    if (p + '.conv_out.weight') in sd:
        x_in = conv(sd, p + '.conv_out', x_in, padding=0)
    return x + x_in


def fuse_sft(sd, p, enc_feat, dec_feat, w):
    """Fuse_sft_block.forward (codeformer_arch.py:151-157) with single-pass convs."""
    enc = resblock(sd, p + '.encode_enc', torch.cat([enc_feat, dec_feat], dim=1))
    scale = conv(sd, p + '.scale.2', F.leaky_relu(conv(sd, p + '.scale.0', enc), 0.2))
    shift = conv(sd, p + '.shift.2', F.leaky_relu(conv(sd, p + '.shift.0', enc), 0.2))
    return dec_feat + w * (dec_feat * scale + shift)


def generator_forward(sd, x, plan=None, fuse=None, w=0.0):
    """Generator.forward (+ the SFT fusion of codeformer_arch.py:272-277) in fp16 mode, float64.  ``sd``: decoder_sd();
    ``plan``: O.generator_plan() by default; ``fuse``: {block index: (Fuse_sft_block prefix, encoder feature)}, applied
    after that block when w > 0."""
    plan = O.generator_plan() if plan is None else plan
    x = x.double()
    for i, (kind, _, _) in enumerate(plan):
        p = f'generator.blocks.{i}'
        if kind == 'res':
            x = resblock(sd, p, x)
        elif kind == 'attn':
            x = O.attnblock(sd, p, x)                     # q, k, v, proj_out and the attention core stay split (exact here)
        elif kind == 'up':
            x = upsample(sd, p, x)
        elif kind == 'norm':
            x = O.group_norm(sd, p, x)
        elif kind == 'conv':
            x = conv(sd, p, x) if i + 1 < len(plan) else O.conv(sd, p, x)    # the last conv is the fp32 SIMT conv
        else:
            raise ValueError(kind)
        if fuse and i in fuse and w > 0:
            fp, feat = fuse[i]
            x = fuse_sft(sd, fp, feat.double(), x, w)
    return x


def codeformer_forward(sd, x, w=0.0, adain_on=False, connect_list=('32', '64', '128', '256'), n_head=8):
    """CodeFormer.forward (codeformer_arch.py:223-280) in fp16 mode -> (out float64, logits, lq_feat, top_idx); logits,
    lq_feat and top_idx are the fp32 oracle's (encoder and Transformer as in O.codeformer_forward)."""
    lq_feat, enc_feats = O.encoder_forward(sd, x, [O.FUSE_ENCODER_BLOCK[s] for s in connect_list])
    B = x.shape[0]
    pos = sd['position_emb'].unsqueeze(1).repeat(1, B, 1)
    q = F.linear(lq_feat.flatten(2).permute(2, 0, 1), sd['feat_emb.weight'], sd['feat_emb.bias'])
    for layer in range(O.n_layers_of(sd)):
        q = O.transformer_layer(sd, f'ft_layers.{layer}', q, pos, n_head)
    E = q.shape[-1]
    logits = F.linear(F.layer_norm(q, (E,), sd['idx_pred_layer.0.weight'], sd['idx_pred_layer.0.bias']),
                      sd['idx_pred_layer.1.weight']).permute(1, 0, 2)
    _, top_idx = torch.topk(F.softmax(logits, dim=2), 1, dim=2)
    quant = O.get_codebook_feat(sd, top_idx, [B, 16, 16, 256])
    if adain_on:
        quant = O.adain(quant, lq_feat)
    fuse = {O.FUSE_GENERATOR_BLOCK[s]: (f'fuse_convs_dict.{s}', enc_feats[s]) for s in connect_list}
    out = generator_forward(decoder_sd(sd), quant, fuse=fuse, w=w)
    return out, logits, lq_feat, top_idx


def vqae_forward(sd, x, beta=0.25):
    """VQAutoEncoder.forward (vqgan_arch.py:385-389) in fp16 mode -> (out float64, min_encoding_indices); the quantizer is
    the fp32 oracle's."""
    z, _ = O.encoder_forward(sd, x)
    quant, _, stats = O.vq_forward(sd, z, beta)
    return generator_forward(decoder_sd(sd), quant), stats['min_encoding_indices']
