"""Drop-in ``nn.Module`` mirrors of the reference networks, executing on libcfb200 (sm_90a).

Same constructor signatures, ``state_dict`` keys/shapes and ``forward`` return tuples as

    CodeFormer      /root/reference/basicsr/archs/codeformer_arch.py:160-280
    VQAutoEncoder   /root/reference/basicsr/archs/vqgan_arch.py:326-389
    VectorQuantizer /root/reference/basicsr/archs/vqgan_arch.py:24-84

so ``net = ARCH_REGISTRY.get('CodeFormer')(...).to(device); net.load_state_dict(ckpt['params_ema']);
net.eval(); net(x, w=w, adain=True)[0]`` (inference_codeformer.py:135-143, 204-206) works unchanged.

PyTorch is plumbing here: the modules only *hold* parameters (so ``.to()``, ``load_state_dict`` and
``named_parameters`` behave like the reference) and allocate output / workspace tensors.  All
arithmetic is in the CUDA library behind the C ABI of ``include/cfb200.h``; there is no eager-PyTorch
or CPU fallback -- a missing library, a CPU tensor or a failing kernel raises ``RuntimeError``.
Inference only (the reference's callers run under ``torch.no_grad()``); autograd is not provided.
"""
from __future__ import annotations

import ctypes
import math
import os
import threading
from typing import Dict, Optional

import numpy as np
import torch
from torch import nn

from . import _lib
from . import spec as S
from .native import NativeHandle, Precision
from .registry import ARCH_REGISTRY


# ------------------------------------------------------------------------------------------------
# parameter holders: same attribute names and default initialisation as the torch layers the
# reference instantiates, but no forward -- they are containers, the math is in libcfb200.
# ------------------------------------------------------------------------------------------------
class _ParamsOnly(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError(f'{type(self).__name__} is a parameter holder of codeformer_b200; the arithmetic runs '
                           'inside libcfb200 through the owning network\'s forward')


class _Conv(_ParamsOnly):
    """Parameters of nn.Conv2d(cin, cout, k) (weight OIHW + bias), default init of torch."""

    def __init__(self, cin, cout, k):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin, k, k))
        self.bias = nn.Parameter(torch.empty(cout))
        bound = 1.0 / math.sqrt(cin * k * k)
        nn.init.uniform_(self.weight, -bound, bound)
        nn.init.uniform_(self.bias, -bound, bound)


class _Linear(_ParamsOnly):
    def __init__(self, cin, cout, bias=True):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin))
        bound = 1.0 / math.sqrt(cin)
        nn.init.uniform_(self.weight, -bound, bound)
        if bias:
            self.bias = nn.Parameter(torch.empty(cout))
            nn.init.uniform_(self.bias, -bound, bound)
        else:
            self.register_parameter('bias', None)


class _Norm(_ParamsOnly):
    """Parameters of GroupNorm(32, C, eps=1e-6) (vqgan_arch.py:14-15) or LayerNorm(C)."""

    def __init__(self, c):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(c))
        self.bias = nn.Parameter(torch.zeros(c))


class _ResBlock(_ParamsOnly):
    """vqgan_arch.py:141-151"""

    def __init__(self, cin, cout):
        super().__init__()
        self.in_channels, self.out_channels = cin, cout
        self.norm1 = _Norm(cin)
        self.conv1 = _Conv(cin, cout, 3)
        self.norm2 = _Norm(cout)
        self.conv2 = _Conv(cout, cout, 3)
        if cin != cout:
            self.conv_out = _Conv(cin, cout, 1)


class _AttnBlock(_ParamsOnly):
    """vqgan_arch.py:167-200"""

    def __init__(self, c):
        super().__init__()
        self.in_channels = c
        self.norm = _Norm(c)
        self.q = _Conv(c, c, 1)
        self.k = _Conv(c, c, 1)
        self.v = _Conv(c, c, 1)
        self.proj_out = _Conv(c, c, 1)


class _Resample(_ParamsOnly):
    """Downsample / Upsample (vqgan_arch.py:117-138): one 3x3 conv named ``conv``."""

    def __init__(self, c):
        super().__init__()
        self.conv = _Conv(c, c, 3)


class _BlockStack(_ParamsOnly):
    """Encoder / Generator (vqgan_arch.py:229-323): ``blocks`` ModuleList with the reference's order."""

    def __init__(self, plan):
        super().__init__()
        blocks = []
        for kind, cin, cout, _ in plan:
            if kind == 'conv':
                blocks.append(_Conv(cin, cout, 3))
            elif kind == 'res':
                blocks.append(_ResBlock(cin, cout))
            elif kind == 'attn':
                blocks.append(_AttnBlock(cin))
            elif kind in ('down', 'up'):
                blocks.append(_Resample(cin))
            elif kind == 'norm':
                blocks.append(_Norm(cin))
        self.blocks = nn.ModuleList(blocks)


class _Embedding(_ParamsOnly):
    def __init__(self, k, d):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(k, d))
        nn.init.uniform_(self.weight, -1.0 / k, 1.0 / k)          # vqgan_arch.py:31


def _require_cuda(x, what):
    if not (torch.is_tensor(x) and x.is_cuda):
        raise RuntimeError(f'{what}: codeformer_b200 runs on a CUDA device only (got {getattr(x, "device", type(x))}); '
                           'there is no CPU fallback')
    if x.dtype != torch.float32:
        raise RuntimeError(f'{what}: expected float32, got {x.dtype}')


class VectorQuantizer(nn.Module):
    """``VectorQuantizer`` of vqgan_arch.py:24-84 on libcfb200 (``cfb_vq_nearest`` / ``cfb_codebook_lookup``)."""

    def __init__(self, codebook_size, emb_dim, beta):
        super().__init__()
        self.codebook_size = codebook_size
        self.emb_dim = emb_dim
        self.beta = beta
        self.embedding = _Embedding(codebook_size, emb_dim)

    def forward(self, z, return_min_encodings=True):
        _require_cuda(z, 'VectorQuantizer.forward')
        lib = _lib.load()
        z = z.contiguous()
        B, D, H, W = z.shape
        if D != self.emb_dim:
            raise RuntimeError(f'VectorQuantizer: expected {self.emb_dim} channels, got {D}')
        E = self.embedding.weight.detach().contiguous()
        with torch.cuda.device(z.device):
            if lib.cfb_vq_fast_supported(B, H, W, D, self.codebook_size) and E.dtype == torch.float32:
                return self._forward_fused(lib, z, E, return_min_encodings)
            zq = torch.empty_like(z)
            idx = torch.empty((B * H * W, 1), dtype=torch.int64, device=z.device)
            stats = torch.empty(4, dtype=torch.float32, device=z.device)
            onehot = torch.empty((B * H * W, self.codebook_size), dtype=torch.float32, device=z.device) \
                if return_min_encodings else None
            wsb = lib.cfb_vq_workspace_bytes(B, H * W, D, self.codebook_size)
            ws = torch.empty(int(wsb), dtype=torch.uint8, device=z.device)
            _lib.check(lib.cfb_vq_nearest(_lib.ptr(z), _lib.ptr(E), B, H, W, D, self.codebook_size, float(self.beta),
                                          _lib.ptr(zq), _lib.ptr(idx), _lib.ptr(stats), _lib.ptr(onehot),
                                          _lib.ptr(ws), wsb, _lib.stream(z.device)), 'cfb_vq_nearest')
        return zq, stats[0], {'perplexity': stats[1], 'min_encodings': onehot,
                              'min_encoding_indices': idx, 'mean_distance': stats[2]}

    # Fused path (include/cfb200.h: cfb_vq_nearest_fast): the split codebook + |e|^2 are prepared once per embedding version and
    # the workspace is kept per shape.  The library runs the whole forward as ONE kernel (conv_tc.cu: vq_fused_kernel), so a call
    # is one launch on the caller's tensors.
    def _forward_fused(self, lib, z, E, return_min_encodings):
        dev = z.device
        B, D, H, W = z.shape
        K = self.codebook_size
        cache = self.__dict__.setdefault('_cfb_vq', {})
        w = self.embedding.weight
        sig = (w.data_ptr(), w._version, str(dev))
        if cache.get('sig') != sig:
            prep = torch.empty(int(lib.cfb_vq_prepared_bytes(K, D)), dtype=torch.uint8, device=dev)
            _lib.check(lib.cfb_vq_prepare(_lib.ptr(E), K, D, _lib.ptr(prep), prep.numel(), _lib.stream(dev)), 'cfb_vq_prepare')
            cache.clear()
            cache.update(sig=sig, prep=prep, E=E)
        prep, E = cache['prep'], cache['E']
        T = B * H * W
        # the kept workspace is only scratch of one launch; calls of one module are ordered by the caller's stream
        keep_ws = not torch.cuda.is_current_stream_capturing()
        ws = cache.setdefault('ws', {}).get((B, H, W)) if keep_ws else None
        if ws is None:
            ws = torch.empty(int(lib.cfb_vq_fast_workspace_bytes(B, H * W, D, K)), dtype=torch.uint8, device=dev)
            if keep_ws:
                if len(cache['ws']) >= 4:
                    cache['ws'].pop(next(iter(cache['ws'])))
                cache['ws'][(B, H, W)] = ws
        zq = torch.empty_like(z)
        idx = torch.empty((T, 1), dtype=torch.int64, device=dev)
        stats = torch.empty(4, dtype=torch.float32, device=dev)
        onehot = torch.empty((T, K), dtype=torch.float32, device=dev) if return_min_encodings else None
        _lib.check(lib.cfb_vq_nearest_fast(_lib.ptr(z), _lib.ptr(E), _lib.ptr(prep), B, H, W, D, K, float(self.beta),
                                           _lib.ptr(zq), _lib.ptr(idx), _lib.ptr(stats), _lib.ptr(onehot), _lib.ptr(ws),
                                           ws.numel(), _lib.stream(dev)), 'cfb_vq_nearest_fast')
        return zq, stats[0], {'perplexity': stats[1], 'min_encodings': onehot, 'min_encoding_indices': idx, 'mean_distance': stats[2]}

    def get_codebook_feat(self, indices, shape):
        """vqgan_arch.py:72-84: indices -> codebook rows; ``shape`` = [B,H,W,C] gives an NCHW result."""
        if not indices.is_cuda:
            raise RuntimeError('get_codebook_feat: CUDA tensors only')
        lib = _lib.load()
        idx = indices.reshape(-1).to(torch.int64).contiguous()
        E = self.embedding.weight.detach().contiguous()
        if shape is None:
            B, H, W = idx.numel(), 1, 1
        else:
            B, H, W, C = shape
            if C != self.emb_dim or B * H * W != idx.numel():
                raise RuntimeError('get_codebook_feat: shape does not match the indices')
        with torch.cuda.device(idx.device):
            out = torch.empty((B, self.emb_dim, H, W), dtype=torch.float32, device=idx.device)
            _lib.check(lib.cfb_codebook_lookup(_lib.ptr(idx), _lib.ptr(E), B, H, W, self.emb_dim, self.codebook_size,
                                               _lib.ptr(out), _lib.stream(idx.device)), 'cfb_codebook_lookup')
        return out.view(B, self.emb_dim) if shape is None else out


@ARCH_REGISTRY.register()
class VQAutoEncoder(Precision, NativeHandle):
    """Mirror of ``VQAutoEncoder`` (vqgan_arch.py:326-389), quantizer='nearest'.

    ``set_precision`` selects the precision of the decoder convs -- the generator's and the Fuse_sft_blocks' (not the
    AttnBlocks', not the last conv).  The encoder, the Transformer and the quantizer are the same in both precisions, so
    ``logits``, ``lq_feat`` and the code indices are bit-identical; only the decoded image changes.  'fp16' needs the
    tensor-core engine ('auto' or 'tc'): with ``set_engine('f32')`` the forward raises."""

    _KIND = 0
    stream_lanes = 1                  # >1: sub-batches run on separate CUDA streams; the persistent conv CTAs already own every
                                      # SM, so off by default
    stream_lanes_min_faces = 4        # only split when every lane gets at least this many faces

    def __init__(self, img_size, nf, ch_mult, quantizer='nearest', res_blocks=2, attn_resolutions=[16],
                 codebook_size=1024, emb_dim=256, beta=0.25, gumbel_straight_through=False, gumbel_kl_weight=1e-8,
                 model_path=None):
        super().__init__('net')
        object.__setattr__(self, '_cfb_ws', {})
        object.__setattr__(self, '_cfb_graphs', {})
        if quantizer != 'nearest':
            raise NotImplementedError("codeformer_b200 builds the 'nearest' quantizer only (the Gumbel quantizer is "
                                      'training-only in the reference, SURVEY.md §2.1)')
        self.in_channels = 3
        self.nf = nf
        self.n_blocks = res_blocks
        self.codebook_size = codebook_size
        self.embed_dim = emb_dim
        self.ch_mult = list(ch_mult)
        self.resolution = img_size
        self.attn_resolutions = list(attn_resolutions)
        self.quantizer_type = quantizer
        self.encoder = _BlockStack(S.encoder_plan(nf, ch_mult, res_blocks, img_size, attn_resolutions, 3, emb_dim))
        self.beta = beta
        self.quantize = VectorQuantizer(codebook_size, emb_dim, beta)
        self.generator = _BlockStack(S.generator_plan(nf, ch_mult, res_blocks, img_size, attn_resolutions, emb_dim))
        if model_path is not None:                                   # vqgan_arch.py:373-382
            chkpt = torch.load(model_path, map_location='cpu')
            if 'params_ema' in chkpt:
                self.load_state_dict(chkpt['params_ema'])
            elif 'params' in chkpt:
                self.load_state_dict(chkpt['params'])
            else:
                raise ValueError('Wrong params!')

    # ---- native handle: what differs from NativeHandle ----------------------------------------------
    def _cfb_config(self) -> '_lib.CfbConfig':
        c = _lib.CfbConfig()
        c.kind = self._KIND
        c.img_size, c.nf, c.n_ch_mult = self.resolution, self.nf, len(self.ch_mult)
        for i, m in enumerate(self.ch_mult):
            c.ch_mult[i] = m
        c.res_blocks = self.n_blocks
        c.n_attn_res = len(self.attn_resolutions)
        for i, r in enumerate(self.attn_resolutions):
            c.attn_res[i] = r
        c.codebook_size, c.emb_dim, c.beta = self.codebook_size, self.embed_dim, float(self.beta)
        return c

    def _create_args(self):
        return (ctypes.byref(self._cfb_config()),)

    def _handle(self):
        if self._net is None:
            super()._handle()
            _lib.check(_lib.load().cfb_net_set_engine(self._net, getattr(self, '_cfb_engine', 0)), 'cfb_net_set_engine')
        return self._net

    def _prepare(self, device):
        prepared = super()._prepare(device)
        if prepared:
            self._cfb_graphs.clear()                   # captured launch sequences bake in the old weight copies
        return prepared

    def _cfb_side_streams(self, device, count):
        pool = self._cfb_ws.setdefault(('streams', device.index), [])
        while len(pool) < count:
            pool.append(torch.cuda.Stream(device=device))
        return pool

    def _cfb_workspace(self, device, batch, lane=0, sweep_k=0):
        lib = _lib.load()
        key = (device.index, torch.cuda.current_stream(device).cuda_stream, lane)
        need = lib.cfb_sweep_workspace_bytes(self._net, batch, sweep_k) if sweep_k else lib.cfb_workspace_bytes(self._net, batch)
        if need < 0:
            _lib.check(1, 'cfb_sweep_workspace_bytes' if sweep_k else 'cfb_workspace_bytes')
        ws = self._cfb_ws.get(key)
        if ws is None or ws.numel() < need:
            self._cfb_ws.pop(key, None)
            ws = None                                  # the old buffer is free before the larger one is allocated
            ws = torch.empty(int(need), dtype=torch.uint8, device=device)   # owned by the module (the caller may
            self._cfb_ws[key] = ws                                          # empty_cache() after every face)
        return ws

    def _check_input(self, x):
        _require_cuda(x, type(self).__name__ + '.forward')
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[2] != self.resolution or x.shape[3] != self.resolution:
            raise RuntimeError(f'expected input [B,3,{self.resolution},{self.resolution}], got {tuple(x.shape)}')
        return x.contiguous()

    def set_engine(self, engine: str = 'auto'):
        """Engine of the dense convs/linears: 'auto' (wgmma tensor cores wherever the shape allows), 'f32'
        (fp32 CUDA-core implicit GEMM) or 'tc' (wgmma only).  Both are CUDA kernels of libcfb200."""
        code = {'auto': 0, 'f32': 1, 'tc': 2}[engine]
        object.__setattr__(self, '_cfb_engine', code)
        self._cfb_graphs.clear()
        if self._net is not None:
            _lib.check(_lib.load().cfb_net_set_engine(self._net, code), 'cfb_net_set_engine')

    def capture(self, stage: str, dst: Optional[torch.Tensor]):
        """Parity hook (cfb_net_capture): copy the NHWC activation after ``stage`` into ``dst`` on the next forwards."""
        if self._net is None:
            raise RuntimeError('capture: run one forward (or load weights on the device) first')
        hooks = getattr(self, '_cfb_hooks', set())
        (hooks.add if dst is not None else hooks.discard)(stage)
        object.__setattr__(self, '_cfb_hooks', hooks)
        self._cfb_graphs.clear()                       # hooks add copies to the launch sequence
        _lib.check(_lib.load().cfb_net_capture(self._net, stage.encode(), _lib.ptr(dst),
                                               0 if dst is None else dst.numel()), 'cfb_net_capture')

    @property
    def last_launch_count(self) -> int:
        return 0 if self._net is None else int(_lib.load().cfb_last_launch_count(self._net))

    # ---- VQAutoEncoder.forward  vqgan_arch.py:385-389 -------------------------------------------
    def forward(self, x, return_min_encodings=True):
        """-> (x_hat [B,3,H,W], codebook_loss, {perplexity, min_encodings, min_encoding_indices, mean_distance}), exactly
        the reference's tuple (vqgan_arch.py:65-70,385-389).  ``min_encodings`` is the [B*256, K] one-hot (1 MB per face);
        callers that only index ``[0]`` (scripts/inference_vqgan.py:46) may pass ``return_min_encodings=False`` to skip it."""
        x = self._check_input(x)
        lib = _lib.load()
        B = x.shape[0]
        dev = x.device
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            ws = self._cfb_workspace(dev, B)
            out = torch.empty_like(x)
            n_tok = B * (self.resolution >> (len(self.ch_mult) - 1)) ** 2
            idx = torch.empty((n_tok, 1), dtype=torch.int64, device=dev)
            stats = torch.empty(4, dtype=torch.float32, device=dev)
            onehot = torch.empty((n_tok, self.codebook_size), dtype=torch.float32, device=dev) \
                if return_min_encodings else None
            _lib.check(lib.cfb_vqae_forward(self._net, _lib.ptr(x), _lib.ptr(out), _lib.ptr(idx), _lib.ptr(stats),
                                            _lib.ptr(onehot), B, _lib.ptr(ws), ws.numel(), _lib.stream(dev)),
                       'cfb_vqae_forward')
        return out, stats[0], {'perplexity': stats[1], 'min_encodings': onehot,
                               'min_encoding_indices': idx, 'mean_distance': stats[2]}


class _MHA(_ParamsOnly):
    """Parameters of nn.MultiheadAttention(E, heads) (codeformer_arch.py:102)."""

    def __init__(self, e):
        super().__init__()
        self.in_proj_weight = nn.Parameter(torch.empty(3 * e, e))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * e))
        self.out_proj = _Linear(e, e)
        nn.init.xavier_uniform_(self.in_proj_weight)
        nn.init.zeros_(self.out_proj.bias)


class _TransformerSALayer(_ParamsOnly):
    """codeformer_arch.py:99-113"""

    def __init__(self, e, dim_mlp):
        super().__init__()
        self.self_attn = _MHA(e)
        self.linear1 = _Linear(e, dim_mlp)
        self.linear2 = _Linear(dim_mlp, e)
        self.norm1 = _Norm(e)
        self.norm2 = _Norm(e)


class _FuseSft(_ParamsOnly):
    """codeformer_arch.py:136-149"""

    def __init__(self, c):
        super().__init__()
        self.encode_enc = _ResBlock(2 * c, c)
        self.scale = nn.ModuleDict({'0': _Conv(c, c, 3), '2': _Conv(c, c, 3)})
        self.shift = nn.ModuleDict({'0': _Conv(c, c, 3), '2': _Conv(c, c, 3)})


def fidelity_weights(w, n, device=None):
    """The fidelity weight ``w`` of the CodeFormer forwards for ``n`` faces.  A number (anything ``float()`` takes, a 0-d array
    or tensor included) is one weight for every face and comes back as a float: the scalar path.  One weight per face -- a
    sequence of n numbers, a floating numpy array or a floating tensor of shape [n], on the host or on the CUDA ``device`` --
    comes back as a contiguous float32 tensor [n] where it was given.  A wrong length or shape, or a CUDA tensor on another
    device than ``device``, raises RuntimeError; a non-floating array or tensor (or a sequence of non-numbers) ValueError."""
    if torch.is_tensor(w):
        if w.dim() == 0:
            return float(w)
        if not w.dtype.is_floating_point:
            raise ValueError(f'w: per-face fidelity weights must be floating point, got a {w.dtype} tensor')
        if w.is_cuda and device is not None and w.device != torch.device(device):
            raise RuntimeError(f'w: per-face fidelity weights are on {w.device}, the faces on {torch.device(device)}')
        t = w.detach()
    elif isinstance(w, (np.ndarray, list, tuple)):
        a = np.asarray(w)
        if a.ndim == 0:
            return float(a)
        ok = 'f' if isinstance(w, np.ndarray) else 'fiub'          # a sequence may hold Python ints
        if a.dtype.kind not in ok:
            raise ValueError(f'w: per-face fidelity weights must be floating point, got {a.dtype}')
        t = torch.from_numpy(a.astype(np.float32))
    else:
        return float(w)
    if t.dim() != 1 or t.shape[0] != n:
        raise RuntimeError(f'w: expected one fidelity weight per face, shape [{n}], got {tuple(t.shape)}')
    return t.to(torch.float32).contiguous()


def sweep_weights(ws, device=None):
    """The K fidelity weights of a sweep (``CodeFormer.forward_u8_sweep``, ``restore_images_sweep``): a 1-D sequence of
    numbers, a floating numpy array or a floating tensor of K >= 1 values, on the host or on the CUDA ``device`` -> a contiguous
    float32 tensor [K] where it was given.  An empty, 0-d or multi-dimensional ``ws``, a non-floating array or tensor or a
    sequence of non-numbers raises ValueError; a CUDA tensor on another device than ``device`` RuntimeError."""
    if torch.is_tensor(ws):
        if not ws.dtype.is_floating_point:
            raise ValueError(f'ws: fidelity weights must be floating point, got a {ws.dtype} tensor')
        if ws.is_cuda and device is not None and ws.device != torch.device(device):
            raise RuntimeError(f'ws: fidelity weights are on {ws.device}, the faces on {torch.device(device)}')
        t = ws.detach()
    elif isinstance(ws, (np.ndarray, list, tuple)):
        try:
            a = np.asarray(ws)
        except ValueError as err:
            raise ValueError(f'ws: expected a 1-D sequence of fidelity weights ({err})') from None
        if a.dtype.kind not in ('f' if isinstance(ws, np.ndarray) else 'fiub'):
            raise ValueError(f'ws: fidelity weights must be floating point, got {a.dtype}')
        t = torch.from_numpy(a.astype(np.float32))
    else:
        raise ValueError(f'ws: expected a 1-D sequence, array or tensor of fidelity weights, got {type(ws).__name__}')
    if t.dim() != 1 or t.shape[0] == 0:
        raise ValueError(f'ws: expected K >= 1 fidelity weights in one dimension, got shape {tuple(t.shape)}')
    return t.to(torch.float32).contiguous()


def sweep_chunks(n_faces, k, max_batch):
    """Chunk plan of a fidelity sweep over ``n_faces`` faces at ``k`` weights: consecutive [lo, hi) ranges of
    ``max(1, max_batch // k)`` faces, so that the decoder batch (faces x k) stays within ``max_batch`` when k <= max_batch."""
    step = max(1, int(max_batch) // max(1, int(k)))
    return [(lo, min(n_faces, lo + step)) for lo in range(0, n_faces, step)]


def _weights_on(w, dev):
    """A per-face weight tensor of fidelity_weights on CUDA device ``dev`` (host values go through pinned memory: no sync)."""
    return w if w.is_cuda else w.pin_memory().to(dev, non_blocking=True)


def restore_chunks(n_faces, max_batch):
    """Chunk plan of ``CodeFormer.restore_faces``: consecutive [lo, hi) ranges of <= max_batch faces; a chunk of >= 16 faces
    is split in two so the host-side staging of one half overlaps the GPU work of the other."""
    bounds = []
    max_batch = max(1, int(max_batch))
    for lo in range(0, n_faces, max_batch):
        hi = min(n_faces, lo + max_batch)
        if hi - lo >= 16:
            mid = lo + (hi - lo + 1) // 2
            bounds += [(lo, mid), (mid, hi)]
        else:
            bounds.append((lo, hi))
    return bounds


@ARCH_REGISTRY.register()
class CodeFormer(VQAutoEncoder):
    """Mirror of ``CodeFormer`` (codeformer_arch.py:160-280)."""

    _KIND = 1

    def __init__(self, dim_embd=512, n_head=8, n_layers=9, codebook_size=1024, latent_size=256,
                 connect_list=['32', '64', '128', '256'], fix_modules=['quantize', 'generator'], vqgan_path=None):
        super().__init__(512, 64, [1, 2, 2, 4, 4, 8], 'nearest', 2, [16], codebook_size)
        if vqgan_path is not None:                                  # codeformer_arch.py:168-170
            self.load_state_dict(torch.load(vqgan_path, map_location='cpu')['params_ema'])
        if fix_modules is not None:                                 # :172-175
            for module in fix_modules:
                for param in getattr(self, module).parameters():
                    param.requires_grad = False
        self.connect_list = list(connect_list)
        self.n_layers = n_layers
        self.n_head = n_head
        self.dim_embd = dim_embd
        self.dim_mlp = dim_embd * 2
        self.latent_size = latent_size
        self.position_emb = nn.Parameter(torch.zeros(latent_size, dim_embd))
        self.feat_emb = _Linear(256, dim_embd)
        self.ft_layers = nn.Sequential(*[_TransformerSALayer(dim_embd, self.dim_mlp) for _ in range(n_layers)])
        self.idx_pred_layer = nn.Sequential(_Norm(dim_embd), _Linear(dim_embd, codebook_size, bias=False))
        self.channels = dict(S.FUSE_CHANNELS)
        self.fuse_encoder_block = dict(S.FUSE_ENCODER_BLOCK)
        self.fuse_generator_block = dict(S.FUSE_GENERATOR_BLOCK)
        self.fuse_convs_dict = nn.ModuleDict()
        for f_size in self.connect_list:
            self.fuse_convs_dict[f_size] = _FuseSft(self.channels[f_size])

    def _cfb_config(self):
        c = super()._cfb_config()
        c.dim_embd, c.n_head, c.n_layers, c.latent_size = self.dim_embd, self.n_head, self.n_layers, self.latent_size
        c.n_connect = len(self.connect_list)
        for i, s in enumerate(self.connect_list):
            c.connect[i] = int(s)
        return c

    def forward(self, x, w=0, detach_16=True, code_only=False, adain=False):
        """-> (out [B,3,512,512], logits [B,256,K], lq_feat [B,256,16,16]); ``code_only`` -> (logits, lq_feat).
        ``detach_16`` only affects autograd in the reference (:263-264) and is accepted for signature parity.
        ``w`` is one fidelity weight, or one per face (``fidelity_weights``): face i then equals the call on that face alone
        with ``w[i]``, bit for bit (``cfb_codeformer_forward_wv``)."""
        x = self._check_input(x)
        lib = _lib.load()
        B = x.shape[0]
        dev = x.device
        w, adain, code_only = fidelity_weights(w, B, dev), bool(adain), bool(code_only)
        per_face = torch.is_tensor(w)

        def launch(src, wv, logits, lq_feat, out, ws):
            if wv is None:
                _lib.check(lib.cfb_codeformer_forward(self._net, _lib.ptr(src), _lib.ptr(out), _lib.ptr(logits), _lib.ptr(lq_feat),
                                                      None, src.shape[0], w, int(adain), int(code_only), _lib.ptr(ws), ws.numel(),
                                                      _lib.stream(dev)), 'cfb_codeformer_forward')
            else:
                _lib.check(lib.cfb_codeformer_forward_wv(self._net, _lib.ptr(src), _lib.ptr(out), _lib.ptr(logits),
                                                         _lib.ptr(lq_feat), None, src.shape[0], _lib.ptr(wv), int(adain),
                                                         int(code_only), _lib.ptr(ws), ws.numel(), _lib.stream(dev)),
                           'cfb_codeformer_forward_wv')
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            # per-face weights are data: one graph per batch size serves every w vector (copied in before each replay)
            if per_face:
                w = _weights_on(w, dev)
                key, inputs = ('wv', dev.index, B, adain, code_only, self._precision), (x, w)
            else:
                key, inputs = (dev.index, B, w, adain, code_only, self._precision), (x,)
            bufs = self._graphed(key, inputs, lambda: (
                torch.empty_like(x), torch.empty_like(w) if per_face else None,
                torch.empty((B, self.latent_size, self.codebook_size), dtype=torch.float32, device=dev),
                torch.empty((B, 256, 16, 16), dtype=torch.float32, device=dev), None if code_only else torch.empty_like(x),
                torch.empty(int(lib.cfb_workspace_bytes(self._net, B)), dtype=torch.uint8, device=dev)), launch)
            if bufs is not None:
                _, _, logits, lq, out, _ = bufs
                return (logits.clone(), lq.clone()) if code_only else (out.clone(), logits.clone(), lq.clone())
            logits = torch.empty((B, self.latent_size, self.codebook_size), dtype=torch.float32, device=dev)
            lq_feat = torch.empty((B, 256, 16, 16), dtype=torch.float32, device=dev)
            out = None if code_only else torch.empty_like(x)
            # Faces are independent, so a batch is run as `lanes` contiguous sub-batches on separate CUDA streams:
            # the tensor-bound conv kernels of one lane overlap the HBM-bound operand-prep / GroupNorm / attention
            # kernels of the other (results are bit-identical to the single-stream run: no cross-face op exists).
            want = int(os.environ.get('CFB_STREAM_LANES', self.stream_lanes))
            lanes = want if B >= want * self.stream_lanes_min_faces else 1
            lanes = max(1, min(lanes, B))
            cur = torch.cuda.current_stream(dev)
            bounds = [(i * B) // lanes for i in range(lanes + 1)]
            side = self._cfb_side_streams(dev, lanes - 1)
            for li in range(lanes):
                lo, hi = bounds[li], bounds[li + 1]
                st = cur if li == 0 else side[li - 1]
                if li > 0:
                    st.wait_stream(cur)                       # inputs / weights produced on the caller's stream
                with torch.cuda.stream(st):
                    launch(x[lo:hi], w[lo:hi] if per_face else None, logits[lo:hi], lq_feat[lo:hi],
                           None if out is None else out[lo:hi], self._cfb_workspace(dev, hi - lo, lane=li))
            for li in range(1, lanes):
                cur.wait_stream(side[li - 1])                 # results are ordered on the caller's stream again
        if code_only:
            return logits, lq_feat
        return out, logits, lq_feat

    # The reference's callers feed ONE face per call (inference_codeformer.py:197-206); at that size the forward is ~440
    # small launches and launch latency dominates.  Small batches are therefore replayed from a CUDA graph captured once
    # per (batch, w, adain, code_only, precision): static input/output buffers, same kernels, same results.  Per-face weights
    # are an input buffer like the faces, so their key holds no w and one graph serves every w vector.
    cuda_graph_max_batch = 4
    cuda_graph_cache_size = 6

    def _graphed(self, key, inputs, buffers, launch):
        """``launch(*bufs)`` replayed from the CUDA graph cached under ``key`` (the key holds the precision: the launch
        sequence depends on it).  On a miss ``buffers()`` makes the static buffers, the first ``len(inputs)`` of which are the
        inputs, and the graph is captured.  ``inputs`` (the faces first) are copied into them before every run.  Returns the
        buffers after the replay (the caller clones what it returns), or None where the plain launch path runs instead."""
        x = inputs[0]
        if not 0 < x.shape[0] <= self.cuda_graph_max_batch or os.environ.get('CFB_CUDA_GRAPH', '1') == '0' \
                or getattr(self, '_cfb_hooks', None) or torch.cuda.is_current_stream_capturing():
            return None
        ent = self._cfb_graphs.pop(key, None)              # re-inserted below: dict order = least recently used first
        if ent is None:
            while len(self._cfb_graphs) >= self.cuda_graph_cache_size:      # callers sweep w (Gradio slider): evict the LRU
                self._cfb_graphs.pop(next(iter(self._cfb_graphs)))          # entry only; each pins one workspace
            bufs = buffers()
            for b, t in zip(bufs, inputs):
                b.copy_(t)
            launch(*bufs)                                    # eager warm-up: one-time function attributes, lazy module load
            torch.cuda.current_stream(x.device).synchronize()
            g = torch.cuda.CUDAGraph()
            try:
                with torch.cuda.graph(g):
                    launch(*bufs)
                ent = (g, bufs)
            except Exception:                                # capture not possible here: keep the plain launch path
                ent = False
        self._cfb_graphs[key] = ent
        if ent is False:
            return None
        g, bufs = ent
        for b, t in zip(bufs, inputs):
            b.copy_(t)
        g.replay()
        return bufs

    # ---- SURVEY.md section 8 rows f1 / f2: the caller's plumbing and per-face loop ----------------------------------
    def forward_u8(self, faces_bgr, w=0.5, adain=True, inpaint=False):
        """``cfb_codeformer_forward_u8``: DEVICE uint8 [B,512,512,3] HWC BGR faces (``face_helper.cropped_faces`` as they
        are) -> restored faces, same layout and dtype.  Bit-for-bit the reference chain img2tensor(face/255.) ->
        normalize(.5,.5) -> net(x, w, adain)[0] -> tensor2img(rgb2bgr, min_max=(-1,1)).astype(uint8)
        (inference_codeformer.py:199-213) with the conversions fused into the first and last conv.

        ``inpaint=True`` (``cfb_codeformer_inpaint_u8``) is inference_inpainting.py:64-75 (there ``w=1, adain=False`` on the
        codebook-512, 3-connect net): the output keeps the input face except where the face is white (255, 255, 255), the mask
        the script builds, i.e. ``(1-mask)*input + mask*output`` before ``tensor2img``, fused into the last conv.

        ``w`` is one fidelity weight, or one per face (``fidelity_weights``; ``cfb_codeformer_forward_u8_wv`` /
        ``cfb_codeformer_inpaint_u8_wv``): face i equals the call on that face alone with ``w[i]``, byte for byte.  With per-face
        weights the Fuse_sft_blocks run for every face (a face with w <= 0 blends with 0), so in fp16 precision their operand
        range guard can fail a batch whose scalar calls would have skipped them."""
        if not torch.is_tensor(faces_bgr) or not faces_bgr.is_cuda or faces_bgr.dtype != torch.uint8:
            raise RuntimeError('forward_u8 expects a CUDA uint8 tensor')
        if faces_bgr.dim() != 4 or tuple(faces_bgr.shape[1:]) != (512, 512, 3):
            raise RuntimeError(f'forward_u8 expects [B,512,512,3] HWC BGR faces, got {tuple(faces_bgr.shape)}')
        lib = _lib.load()
        faces_bgr = faces_bgr.contiguous()
        B, dev = faces_bgr.shape[0], faces_bgr.device
        w, adain, inpaint = fidelity_weights(w, B, dev), bool(adain), bool(inpaint)
        per_face = torch.is_tensor(w)
        name = ('cfb_codeformer_inpaint_u8' if inpaint else 'cfb_codeformer_forward_u8') + ('_wv' if per_face else '')
        fn = getattr(lib, name)
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            if B == 0:
                return torch.empty_like(faces_bgr)

            def launch(src, wv, dst, ws):
                _lib.check(fn(self._net, _lib.ptr(src), _lib.ptr(dst), None, None, None, B, w if wv is None else _lib.ptr(wv),
                              int(adain), _lib.ptr(ws), ws.numel(), _lib.stream(dev)), name)
            if per_face:
                w = _weights_on(w, dev)
                key, inputs = ('u8wv', dev.index, B, adain, inpaint, self._precision), (faces_bgr, w)
            else:
                key, inputs = ('u8', dev.index, B, w, adain, inpaint, self._precision), (faces_bgr,)
            bufs = self._graphed(key, inputs, lambda: (
                torch.empty_like(faces_bgr), torch.empty_like(w) if per_face else None, torch.empty_like(faces_bgr),
                torch.empty(int(lib.cfb_workspace_bytes(self._net, B)), dtype=torch.uint8, device=dev)), launch)
            if bufs is not None:
                return bufs[2].clone()
            out = torch.empty_like(faces_bgr)
            launch(faces_bgr, w if per_face else None, out, self._cfb_workspace(dev, B))
        return out

    def forward_u8_sweep(self, faces_bgr, ws, adain=True):
        """A fidelity sweep (``cfb_codeformer_sweep_u8``): DEVICE uint8 [B,512,512,3] HWC BGR faces, each restored at every
        weight of ``ws`` (``sweep_weights``: K >= 1 values, shared by all faces) -> CUDA uint8 [B,K,512,512,3].  The encoder,
        the Transformer, the code lookup and AdaIN run once per face; only the generator and the Fuse_sft_blocks run B*K
        times.  ``[b, k]`` equals ``forward_u8(faces_bgr[b:b+1], w=ws[k], adain=adain)``, byte for byte; as with per-face
        weights, the Fuse_sft_blocks run for every weight (w <= 0 or NaN blends with 0), so in fp16 precision their operand
        range guard can fail a sweep whose scalar calls would have skipped them."""
        if not torch.is_tensor(faces_bgr) or not faces_bgr.is_cuda or faces_bgr.dtype != torch.uint8:
            raise RuntimeError('forward_u8_sweep expects a CUDA uint8 tensor')
        if faces_bgr.dim() != 4 or tuple(faces_bgr.shape[1:]) != (512, 512, 3):
            raise RuntimeError(f'forward_u8_sweep expects [B,512,512,3] HWC BGR faces, got {tuple(faces_bgr.shape)}')
        lib = _lib.load()
        faces_bgr = faces_bgr.contiguous()
        B, dev = faces_bgr.shape[0], faces_bgr.device
        ws, adain = sweep_weights(ws, dev), bool(adain)
        K = ws.shape[0]
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            if B == 0:
                return torch.empty((0, K, 512, 512, 3), dtype=torch.uint8, device=dev)
            wv = _weights_on(ws, dev).repeat(B)           # [B*K], face-major: decoder face b*K + k takes ws[k]

            def launch(src, wv, dst, ws_buf):
                _lib.check(lib.cfb_codeformer_sweep_u8(self._net, _lib.ptr(src), _lib.ptr(dst), None, None, None, B, K,
                                                       _lib.ptr(wv), int(adain), _lib.ptr(ws_buf), ws_buf.numel(),
                                                       _lib.stream(dev)), 'cfb_codeformer_sweep_u8')
            # the weights are a static input: one graph per (B, K) serves every ws
            bufs = self._graphed(('u8sweep', dev.index, B, K, adain, self._precision), (faces_bgr, wv), lambda: (
                torch.empty_like(faces_bgr), torch.empty_like(wv),
                torch.empty((B, K, 512, 512, 3), dtype=torch.uint8, device=dev),
                torch.empty(int(lib.cfb_sweep_workspace_bytes(self._net, B, K)), dtype=torch.uint8, device=dev)), launch)
            if bufs is not None:
                return bufs[2].clone()
            out = torch.empty((B, K, 512, 512, 3), dtype=torch.uint8, device=dev)
            launch(faces_bgr, wv, out, self._cfb_workspace(dev, B, sweep_k=K))
        return out

    def restore_faces(self, faces, w=0.5, adain=True, max_batch=32, device=None, on_error='input', inpaint=False):
        """Batched front-end for the caller loop ``for cropped_face in face_helper.cropped_faces`` of
        inference_codeformer.py:197-214 (one face per call there).  ``faces``: a list of uint8 [512,512,3] BGR arrays (or one
        [B,512,512,3] array / CPU uint8 tensor).  Returns the list of restored uint8 BGR faces in order -- what the loop
        passes to ``face_helper.add_restored_face``.  Faces go through pinned uint8 staging (0.79 MB per face each way)
        in chunks of ``max_batch``.  ``on_error='input'`` mirrors the reference's fallback (:209-211: on any failure the
        restored face is the input face); ``'raise'`` re-raises.  ``inpaint=True`` is the loop of inference_inpainting.py
        (``forward_u8(inpaint=True)``; its fallback, :78-80, is the input face as well).  ``w``: one fidelity weight or one per
        face (``fidelity_weights``), each chunk taking its faces' weights; a chunk that fails (in fp16 precision the
        Fuse_sft_blocks of per-face weights run even for faces with w <= 0) falls back on its own."""
        if torch.is_tensor(faces):
            arr = faces.detach().cpu().numpy()
        elif isinstance(faces, np.ndarray):
            arr = faces
        else:
            faces = list(faces)
            arr = np.stack(faces) if faces else np.zeros((0, 512, 512, 3), np.uint8)
        if arr.ndim == 3:
            arr = arr[None]
        if arr.dtype != np.uint8 or arr.ndim != 4 or tuple(arr.shape[1:]) != (512, 512, 3):
            raise RuntimeError(f'restore_faces expects uint8 [512,512,3] BGR faces, got {arr.dtype} {tuple(arr.shape)}')
        if on_error not in ('input', 'raise'):
            raise RuntimeError("on_error must be 'input' or 'raise'")
        dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        w = fidelity_weights(w, arr.shape[0], dev)
        if torch.is_tensor(w):
            w = _weights_on(w, dev)                    # once: the chunks take device slices (no host sync per chunk)
        max_batch = max(1, int(max_batch))
        self.last_restore_errors = []
        # chunks of <= max_batch faces; a chunk of >= 16 is split in two so that the host-side staging copies of one half
        # overlap the GPU work of the other (per-face GPU time is flat above 16 faces)
        bounds = restore_chunks(arr.shape[0], max_batch)
        results = [None] * len(bounds)
        pending = []                                   # (chunk index, pinned output, event) in flight on the stream

        def drain(upto):
            while len(pending) > upto:
                k, pout, ev = pending.pop(0)
                lo, hi = bounds[k]
                try:
                    ev.synchronize()
                    # kernels report a pipeline time-out / fp16 operand overflow through a status word instead of
                    # trapping: turn it into the exception the reference's per-face fallback expects
                    _lib.check(_lib.load().cfb_check_async_status(), 'restore_faces')
                    results[k] = pout.numpy().copy()
                except RuntimeError as err:
                    if on_error == 'raise':
                        raise
                    self.last_restore_errors.append((lo, str(err)))
                    results[k] = arr[lo:hi].copy()

        with torch.cuda.device(dev):
            for k, (lo, hi) in enumerate(bounds):
                B = hi - lo
                try:
                    key = ('pin', dev.index, B, k & 1, threading.get_ident())      # staging is per caller thread (app.py:282)
                    pin = self._cfb_ws.get(key)
                    if pin is None:
                        pin = (torch.empty((B, 512, 512, 3), dtype=torch.uint8, pin_memory=True),
                               torch.empty((B, 512, 512, 3), dtype=torch.uint8, pin_memory=True))
                        self._cfb_ws[key] = pin
                    drain(1)                           # the buffers of chunk k-2 (same parity) are free again
                    pin[0].copy_(torch.from_numpy(np.ascontiguousarray(arr[lo:hi])))
                    out = self.forward_u8(pin[0].to(dev, non_blocking=True), w=w[lo:hi] if torch.is_tensor(w) else w,
                                          adain=adain, inpaint=inpaint)
                    pin[1].copy_(out, non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record(torch.cuda.current_stream(dev))
                    pending.append((k, pin[1], ev))
                except RuntimeError as err:
                    if on_error == 'raise':
                        raise
                    self.last_restore_errors.append((lo, str(err)))
                    results[k] = arr[lo:hi].copy()
            drain(0)
        restored = []
        for res in results:
            restored.extend(res[i] for i in range(res.shape[0]))
        return restored

    def forward_host(self, x_host, w=0, adain=False, device=None):
        """End-to-end call with HOST tensors (``cfb_codeformer_forward_host``): pinned x -> H2D -> forward ->
        D2H of out/logits/lq_feat -> one stream sync.  Returns pinned host tensors."""
        lib = _lib.load()
        if x_host.is_cuda or x_host.dtype != torch.float32:
            raise RuntimeError('forward_host expects a float32 CPU tensor')
        dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        x_host = x_host.contiguous()
        B = x_host.shape[0]
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            ws = self._cfb_workspace(dev, B)
            iob = lib.cfb_host_io_bytes(self._net, B)
            key = ('io', dev.index)
            io = self._cfb_ws.get(key)
            if io is None or io.numel() < iob:
                io = torch.empty(int(iob), dtype=torch.uint8, device=dev)
                self._cfb_ws[key] = io
            out = torch.empty(x_host.shape, dtype=torch.float32, pin_memory=True)
            logits = torch.empty((B, self.latent_size, self.codebook_size), dtype=torch.float32, pin_memory=True)
            lq = torch.empty((B, 256, 16, 16), dtype=torch.float32, pin_memory=True)
            _lib.check(lib.cfb_codeformer_forward_host(self._net, _lib.ptr(x_host), _lib.ptr(out), _lib.ptr(logits),
                                                       _lib.ptr(lq), B, float(w), int(bool(adain)), _lib.ptr(io),
                                                       io.numel(), _lib.ptr(ws), ws.numel(), _lib.stream(dev)),
                       'cfb_codeformer_forward_host')
        return out, logits, lq
