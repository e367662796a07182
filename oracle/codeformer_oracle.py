"""CPU oracle for the CodeFormer hot path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this file.  The product (``codeformer_b200``)
never does; it fails loudly when its CUDA library is missing.

What this is
------------
A functional (state-dict in, tensors out) restatement, in fp32 on the CPU, of the
algorithm the reference implements in

    /root/reference/basicsr/archs/vqgan_arch.py      (VQGAN encoder / generator / quantizer)
    /root/reference/basicsr/archs/codeformer_arch.py (Transformer, AdaIN, SFT fusion, forward)

The reference itself contains no arithmetic: every op is a call into a third-party
dependency that is not under /root/reference -- **PyTorch** (``requirements.txt:12``
asks for ``torch>=1.7.1``, unpinned; this image has torch 2.11.0+cu128, CPU backend
oneDNN/MKL).  The restatement therefore calls the same published torch operators
(``conv2d``, ``group_norm``, ``softmax``, ``layer_norm``, ``gelu``, ``bmm`` ...) at the
reference's own call sites, each cited below, and spells out explicitly the pieces the
reference gets through ``nn.MultiheadAttention`` (slow path of
``torch.nn.functional.multi_head_attention_forward``).

Parity pinning
--------------
The reference ships no tests, golden vectors or fixtures for this path (SURVEY.md §4,
§8c) => **"parity unpinned" by the reference**.  We pin it ourselves:
``oracle/gen_golden.py`` imports the *unmodified* reference modules in the build
container (``oracle/ref_shim.py``), runs them on seeded weights and committed input
faces and stores their outputs under ``tests/golden/``; ``tests/test_oracle.py`` checks
this restatement against those vectors (and, when /root/reference is present, directly
against the live reference modules).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor
SD = Dict[str, Tensor]

# -----------------------------------------------------------------------------
# architecture constants (codeformer_arch.py:166, :194-206)
# -----------------------------------------------------------------------------
NF = 64
CH_MULT = (1, 2, 2, 4, 4, 8)
RES_BLOCKS = 2
ATTN_RES = (16,)
IMG_SIZE = 512
EMB_DIM = 256
FUSE_ENCODER_BLOCK = {'512': 2, '256': 5, '128': 8, '64': 11, '32': 14, '16': 18}   # codeformer_arch.py:204
FUSE_GENERATOR_BLOCK = {'16': 6, '32': 9, '64': 12, '128': 15, '256': 18, '512': 21}  # codeformer_arch.py:206


def encoder_plan(nf=NF, ch_mult=CH_MULT, res_blocks=RES_BLOCKS, resolution=IMG_SIZE,
                 attn_resolutions=ATTN_RES, in_channels=3, emb_dim=EMB_DIM) -> List[tuple]:
    """Block list of ``Encoder.__init__`` (vqgan_arch.py:229-267) as (kind, cin, cout)."""
    plan = [('conv', in_channels, nf)]
    curr = resolution
    in_ch_mult = (1,) + tuple(ch_mult)
    cin = nf
    for i in range(len(ch_mult)):
        cin = nf * in_ch_mult[i]
        cout = nf * ch_mult[i]
        for _ in range(res_blocks):
            plan.append(('res', cin, cout))
            cin = cout
            if curr in attn_resolutions:
                plan.append(('attn', cin, cin))
        if i != len(ch_mult) - 1:
            plan.append(('down', cin, cin))
            curr //= 2
    plan += [('res', cin, cin), ('attn', cin, cin), ('res', cin, cin), ('norm', cin, cin), ('conv', cin, emb_dim)]
    return plan


def generator_plan(nf=NF, ch_mult=CH_MULT, res_blocks=RES_BLOCKS, resolution=IMG_SIZE,
                   attn_resolutions=ATTN_RES, emb_dim=EMB_DIM) -> List[tuple]:
    """Block list of ``Generator.__init__`` (vqgan_arch.py:276-316)."""
    cin = nf * ch_mult[-1]
    curr = resolution // 2 ** (len(ch_mult) - 1)
    plan = [('conv', emb_dim, cin), ('res', cin, cin), ('attn', cin, cin), ('res', cin, cin)]
    for i in reversed(range(len(ch_mult))):
        cout = nf * ch_mult[i]
        for _ in range(res_blocks):
            plan.append(('res', cin, cout))
            cin = cout
            if curr in attn_resolutions:
                plan.append(('attn', cin, cin))
        if i != 0:
            plan.append(('up', cin, cin))
            curr *= 2
    plan += [('norm', cin, cin), ('conv', cin, 3)]
    return plan


# -----------------------------------------------------------------------------
# vqgan_arch.py leaf ops
# -----------------------------------------------------------------------------
def group_norm(sd: SD, p: str, x: Tensor) -> Tensor:
    """``normalize`` = GroupNorm(32, C, eps=1e-6, affine) -- vqgan_arch.py:14-15."""
    return F.group_norm(x, 32, sd[p + '.weight'], sd[p + '.bias'], eps=1e-6)


def swish(x: Tensor) -> Tensor:
    """vqgan_arch.py:18-20."""
    return x * torch.sigmoid(x)


def conv(sd: SD, p: str, x: Tensor, stride: int = 1, padding: int = 1) -> Tensor:
    return F.conv2d(x, sd[p + '.weight'], sd[p + '.bias'], stride=stride, padding=padding)


def resblock(sd: SD, p: str, x_in: Tensor) -> Tensor:
    """``ResBlock.forward`` -- vqgan_arch.py:153-164."""
    x = group_norm(sd, p + '.norm1', x_in)
    x = swish(x)
    x = conv(sd, p + '.conv1', x)
    x = group_norm(sd, p + '.norm2', x)
    x = swish(x)
    x = conv(sd, p + '.conv2', x)
    if (p + '.conv_out.weight') in sd:                      # in_channels != out_channels
        x_in = conv(sd, p + '.conv_out', x_in, padding=0)
    return x + x_in


def attnblock(sd: SD, p: str, x: Tensor) -> Tensor:
    """``AttnBlock.forward`` -- vqgan_arch.py:202-226 (single head, scale C^-1/2, softmax over keys)."""
    h_ = group_norm(sd, p + '.norm', x)
    q = conv(sd, p + '.q', h_, padding=0)
    k = conv(sd, p + '.k', h_, padding=0)
    v = conv(sd, p + '.v', h_, padding=0)
    b, c, h, w = q.shape
    q = q.reshape(b, c, h * w).permute(0, 2, 1)
    k = k.reshape(b, c, h * w)
    w_ = torch.bmm(q, k) * (int(c) ** (-0.5))
    w_ = F.softmax(w_, dim=2)
    v = v.reshape(b, c, h * w)
    w_ = w_.permute(0, 2, 1)
    h_ = torch.bmm(v, w_).reshape(b, c, h, w)
    h_ = conv(sd, p + '.proj_out', h_, padding=0)
    return x + h_


def downsample(sd: SD, p: str, x: Tensor) -> Tensor:
    """``Downsample.forward`` -- vqgan_arch.py:122-126 (zero pad right/bottom, 3x3 stride 2)."""
    x = F.pad(x, (0, 1, 0, 1), mode='constant', value=0)
    return conv(sd, p + '.conv', x, stride=2, padding=0)


def upsample(sd: SD, p: str, x: Tensor) -> Tensor:
    """``Upsample.forward`` -- vqgan_arch.py:134-138 (nearest x2, then 3x3)."""
    x = F.interpolate(x, scale_factor=2.0, mode='nearest')
    return conv(sd, p + '.conv', x)


def run_block(sd: SD, p: str, kind: str, x: Tensor) -> Tensor:
    if kind == 'conv':
        return conv(sd, p, x)
    if kind == 'res':
        return resblock(sd, p, x)
    if kind == 'attn':
        return attnblock(sd, p, x)
    if kind == 'down':
        return downsample(sd, p, x)
    if kind == 'up':
        return upsample(sd, p, x)
    if kind == 'norm':
        return group_norm(sd, p, x)
    raise ValueError(kind)


def encoder_forward(sd: SD, x: Tensor, taps: Sequence[int] = (), collect: Optional[dict] = None
                    ) -> Tuple[Tensor, Dict[str, Tensor]]:
    """``Encoder.forward`` (vqgan_arch.py:269-273) + the taps of codeformer_arch.py:226-230.
    ``collect`` (tests): every block output is stored under 'enc.<i>'."""
    feats: Dict[str, Tensor] = {}
    for i, (kind, _, _) in enumerate(encoder_plan()):
        x = run_block(sd, f'encoder.blocks.{i}', kind, x)
        if collect is not None:
            collect[f'enc.{i}'] = x
        if i in taps:
            feats[str(x.shape[-1])] = x.clone()
    return x, feats


def vq_forward(sd: SD, z: Tensor, beta: float = 0.25):
    """``VectorQuantizer.forward`` -- vqgan_arch.py:33-70."""
    E = sd['quantize.embedding.weight']
    K, D = E.shape
    z = z.permute(0, 2, 3, 1).contiguous()
    zf = z.view(-1, D)
    d = (zf ** 2).sum(dim=1, keepdim=True) + (E ** 2).sum(1) - 2 * torch.matmul(zf, E.t())
    mean_distance = torch.mean(d)
    idx = torch.argmin(d, dim=1).unsqueeze(1)
    onehot = torch.zeros(idx.shape[0], K).to(z)
    onehot.scatter_(1, idx, 1)
    z_q = torch.matmul(onehot, E).view(z.shape)
    loss = torch.mean((z_q - z) ** 2) + beta * torch.mean((z_q - z) ** 2)
    z_q = z + (z_q - z)
    e_mean = torch.mean(onehot, dim=0)
    perplexity = torch.exp(-torch.sum(e_mean * torch.log(e_mean + 1e-10)))
    z_q = z_q.permute(0, 3, 1, 2).contiguous()
    return z_q, loss, {'perplexity': perplexity, 'min_encodings': onehot,
                       'min_encoding_indices': idx, 'mean_distance': mean_distance}


def get_codebook_feat(sd: SD, indices: Tensor, shape) -> Tensor:
    """``VectorQuantizer.get_codebook_feat`` -- vqgan_arch.py:72-84 (one-hot @ E == gather)."""
    E = sd['quantize.embedding.weight']
    indices = indices.view(-1, 1)
    onehot = torch.zeros(indices.shape[0], E.shape[0]).to(indices)
    onehot.scatter_(1, indices, 1)
    z_q = torch.matmul(onehot.to(E.dtype), E)
    if shape is not None:
        z_q = z_q.view(shape).permute(0, 3, 1, 2).contiguous()
    return z_q


# -----------------------------------------------------------------------------
# codeformer_arch.py
# -----------------------------------------------------------------------------
def calc_mean_std(feat: Tensor, eps: float = 1e-5):
    """codeformer_arch.py:12-26 (UNBIASED variance + eps)."""
    b, c = feat.shape[:2]
    var = feat.view(b, c, -1).var(dim=2) + eps
    std = var.sqrt().view(b, c, 1, 1)
    mean = feat.view(b, c, -1).mean(dim=2).view(b, c, 1, 1)
    return mean, std


def adain(content: Tensor, style: Tensor) -> Tensor:
    """``adaptive_instance_normalization`` -- codeformer_arch.py:29-43."""
    size = content.size()
    s_mean, s_std = calc_mean_std(style)
    c_mean, c_std = calc_mean_std(content)
    normalized = (content - c_mean.expand(size)) / c_std.expand(size)
    return normalized * s_std.expand(size) + s_mean.expand(size)


def mha(sd: SD, p: str, q_in: Tensor, k_in: Tensor, v_in: Tensor, n_head: int) -> Tensor:
    """``nn.MultiheadAttention`` as reached from codeformer_arch.py:126: query is key but
    not value => three separate projections with the rows [Wq;Wk;Wv] of in_proj_weight,
    ``need_weights=True`` => explicit q*sqrt(1/d) -> bmm -> softmax -> bmm -> out_proj
    (torch.nn.functional.multi_head_attention_forward, slow path).  Tokens are seq-first
    [L, B, E]."""
    L, B, E = q_in.shape
    hd = E // n_head
    W = sd[p + '.in_proj_weight']
    bias = sd[p + '.in_proj_bias']
    q = F.linear(q_in, W[:E], bias[:E])
    k = F.linear(k_in, W[E:2 * E], bias[E:2 * E])
    v = F.linear(v_in, W[2 * E:], bias[2 * E:])
    q = q.view(L, B * n_head, hd).transpose(0, 1)
    k = k.view(L, B * n_head, hd).transpose(0, 1)
    v = v.view(L, B * n_head, hd).transpose(0, 1)
    q = q * math.sqrt(1.0 / float(hd))
    a = torch.bmm(q, k.transpose(-2, -1))
    a = F.softmax(a, dim=-1)
    o = torch.bmm(a, v)
    o = o.transpose(0, 1).contiguous().view(L * B, E)
    o = F.linear(o, sd[p + '.out_proj.weight'], sd[p + '.out_proj.bias'])
    return o.view(L, B, E)


def transformer_layer(sd: SD, p: str, tgt: Tensor, pos: Tensor, n_head: int) -> Tensor:
    """``TransformerSALayer.forward`` -- codeformer_arch.py:118-134 (pre-LN, dropout 0, erf GELU)."""
    E = tgt.shape[-1]
    t2 = F.layer_norm(tgt, (E,), sd[p + '.norm1.weight'], sd[p + '.norm1.bias'])
    qk = t2 + pos
    t2 = mha(sd, p + '.self_attn', qk, qk, t2, n_head)
    tgt = tgt + t2
    t2 = F.layer_norm(tgt, (E,), sd[p + '.norm2.weight'], sd[p + '.norm2.bias'])
    t2 = F.linear(F.gelu(F.linear(t2, sd[p + '.linear1.weight'], sd[p + '.linear1.bias'])),
                  sd[p + '.linear2.weight'], sd[p + '.linear2.bias'])
    return tgt + t2


def fuse_sft(sd: SD, p: str, enc_feat: Tensor, dec_feat: Tensor, w: float) -> Tensor:
    """``Fuse_sft_block.forward`` -- codeformer_arch.py:151-157."""
    enc = resblock(sd, p + '.encode_enc', torch.cat([enc_feat, dec_feat], dim=1))
    scale = conv(sd, p + '.scale.2', F.leaky_relu(conv(sd, p + '.scale.0', enc), 0.2))
    shift = conv(sd, p + '.shift.2', F.leaky_relu(conv(sd, p + '.shift.0', enc), 0.2))
    residual = w * (dec_feat * scale + shift)
    return dec_feat + residual


def n_layers_of(sd: SD) -> int:
    n = 0
    while f'ft_layers.{n}.norm1.weight' in sd:
        n += 1
    return n


def codeformer_forward(sd: SD, x: Tensor, w: float = 0, code_only: bool = False, adain_on: bool = False,
                       connect_list: Sequence[str] = ('32', '64', '128', '256'), n_head: int = 8,
                       return_intermediates: bool = False, collect: Optional[dict] = None):
    """``CodeFormer.forward`` -- codeformer_arch.py:223-280."""
    taps = [FUSE_ENCODER_BLOCK[s] for s in connect_list]
    lq_feat, enc_feats = encoder_forward(sd, x, taps, collect)
    B = x.shape[0]
    pos = sd['position_emb'].unsqueeze(1).repeat(1, B, 1)                                  # :235
    q = F.linear(lq_feat.flatten(2).permute(2, 0, 1), sd['feat_emb.weight'], sd['feat_emb.bias'])  # :237
    for l in range(n_layers_of(sd)):                                                        # :240-241
        q = transformer_layer(sd, f'ft_layers.{l}', q, pos, n_head)
        if collect is not None:
            collect[f'ft.{l}'] = q
    E = q.shape[-1]
    logits = F.linear(F.layer_norm(q, (E,), sd['idx_pred_layer.0.weight'], sd['idx_pred_layer.0.bias']),
                      sd['idx_pred_layer.1.weight'])                                        # :244
    logits = logits.permute(1, 0, 2)                                                        # :245
    if code_only:
        return logits, lq_feat
    soft = F.softmax(logits, dim=2)                                                         # :257
    _, top_idx = torch.topk(soft, 1, dim=2)                                                 # :258
    quant = get_codebook_feat(sd, top_idx, [B, 16, 16, 256])                                # :259
    if adain_on:
        quant = adain(quant, lq_feat)                                                       # :266
    x = quant
    if collect is not None:
        collect['quant'] = quant
    fuse = [FUSE_GENERATOR_BLOCK[s] for s in connect_list]
    inter = {}
    for i, (kind, _, _) in enumerate(generator_plan()):                                     # :272-277
        x = run_block(sd, f'generator.blocks.{i}', kind, x)
        if collect is not None:
            collect[f'gen.{i}'] = x
        if i in fuse:
            size = str(x.shape[-1])
            if w > 0:
                x = fuse_sft(sd, f'fuse_convs_dict.{size}', enc_feats[size], x, w)
                if collect is not None:
                    collect[f'fuse.{size}'] = x
    if return_intermediates:
        inter.update(top_idx=top_idx, quant=quant, enc_feats=enc_feats)
        return x, logits, lq_feat, inter
    return x, logits, lq_feat


def vqae_forward(sd: SD, x: Tensor, beta: float = 0.25):
    """``VQAutoEncoder.forward`` -- vqgan_arch.py:385-389."""
    z, _ = encoder_forward(sd, x)
    quant, loss, stats = vq_forward(sd, z, beta)
    x = quant
    for i, (kind, _, _) in enumerate(generator_plan()):
        x = run_block(sd, f'generator.blocks.{i}', kind, x)
    return x, loss, stats
