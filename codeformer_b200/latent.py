"""Latent codes on the device: the third field of ``FFHQBlindDataset`` and scores of CodeFormer's code prediction.

    generate_latent_gt   scripts/generate_latent_gt.py: the VQGAN codes of every ground-truth face and of its mirror image,
                         as the dict ``FFHQBlindDataset(latent_gt_path=...)`` loads (ffhq_blind_dataset.py:49-53, 192-196)
    code_scores          the two stage-2 terms of codeformer_idx_model.py:100-115 per face: the cross-entropy of the
                         ``code_only`` logits against ground-truth codes, and the distance of ``lq_feat`` to their codebook rows

Both run on libcfb200 (``cfb_latent_codes_u8``, ``cfb_codeformer_code_only_u8`` / ``cfb_codeformer_forward``,
``cfb_code_scores``); there is no CPU fallback.  Inference only.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib


def _faces_u8(images):
    """uint8 [N,S,S,3] BGR faces: a CUDA tensor as it is, or host images (a list of arrays, one array, a CPU tensor) -> numpy."""
    if torch.is_tensor(images):
        if images.is_cuda:
            return images
        images = images.numpy()
    if isinstance(images, np.ndarray):
        return images
    images = list(images)
    if not images:
        raise ValueError('generate_latent_gt: no images')
    return np.stack([np.asarray(im) for im in images])


def generate_latent_gt(images, names, vqgan, max_batch=32):
    """scripts/generate_latent_gt.py on the device.  ``images``: uint8 [512,512,3] BGR faces (``cv2.imread`` as it is) -- a
    list of arrays, one [N,512,512,3] array, or a CPU or CUDA uint8 tensor; ``names``: one key per image (the script uses the
    file name without its extension).  ``vqgan``: a ``VQAutoEncoder`` (or ``CodeFormer``) on a CUDA device with its weights.

    Returns the script's dict ``{'orig': {name: np.int64 [16,16]}, 'hflip': {name: ...}}``, ``orig`` first and names in the
    caller's order; ``torch.save`` of it is the file ``FFHQBlindDataset(latent_gt_path=...)`` loads.  The values equal the
    script's loop body -- ``vqgan.quantize(vqgan.encoder(img))[2]['min_encoding_indices'].view(16, 16)`` on
    ``img2tensor(img / 255., bgr2rgb=True, float32=True)`` + ``normalize(0.5, 0.5)``, and on ``cv2.flip(img, 1)`` of it for
    ``hflip`` -- bit for bit.  The faces go to the device in chunks of ``max_batch``; each chunk is one encoder pass over its
    faces and their mirror images (``VQAutoEncoder.latent_codes_u8(hflip=True)``).  (The script calls ``encoder(img, True)``,
    which raises ``TypeError`` in the reference; the encoder takes one argument.)"""
    faces = _faces_u8(images)
    names = list(names)
    R = vqgan.resolution
    if faces.dtype not in (np.uint8, torch.uint8) or faces.ndim != 4 or tuple(faces.shape[1:]) != (R, R, 3):
        raise RuntimeError(f'generate_latent_gt expects uint8 [N,{R},{R},3] BGR faces, got {faces.dtype} {tuple(faces.shape)}')
    if len(names) != faces.shape[0]:
        raise ValueError(f'generate_latent_gt: {faces.shape[0]} images but {len(names)} names')
    if len(set(names)) != len(names):
        raise ValueError('generate_latent_gt: names must be unique (they are the keys of the dict)')
    dev = faces.device if torch.is_tensor(faces) else next(vqgan.parameters()).device
    if dev.type != 'cuda':
        raise RuntimeError('generate_latent_gt: the VQAutoEncoder must be on a CUDA device; there is no CPU fallback')
    step = max(1, int(max_batch))
    orig, flip = [], []
    for lo in range(0, faces.shape[0], step):
        chunk = faces[lo:lo + step]
        if not torch.is_tensor(chunk):
            chunk = torch.from_numpy(np.ascontiguousarray(chunk)).pin_memory().to(dev, non_blocking=True)
        o, f = vqgan.latent_codes_u8(chunk, hflip=True)
        orig.append(o.cpu())
        flip.append(f.cpu())
    orig = torch.cat(orig).numpy() if orig else np.zeros((0, 16, 16), np.int64)
    flip = torch.cat(flip).numpy() if flip else np.zeros((0, 16, 16), np.int64)
    return {'orig': {n: orig[i].copy() for i, n in enumerate(names)},
            'hflip': {n: flip[i].copy() for i, n in enumerate(names)}}


def code_scores(net, lq, gt_codes, max_batch=32):
    """How well CodeFormer's Transformer predicts ground-truth latent codes, per face (``cfb_code_scores``, float64).

    ``net``: a ``CodeFormer`` on a CUDA device.  ``lq``: the degraded faces, CUDA uint8 [B,512,512,3] BGR (``degrade_faces``
    output, read as ``forward_u8`` reads faces) or CUDA fp32 [B,3,512,512] in [-1,1] as the training tensors are.
    ``gt_codes``: CUDA int64 [B,16,16] or [B,256], e.g. ``generate_latent_gt`` / ``latent_codes_u8`` of the ground truth.

    The net runs ``code_only`` (no decoder) in chunks of ``max_batch`` faces.  Returns a dict of CUDA tensors:
      ``cross_entropy`` float64 [B]: mean over tokens of logsumexp(logits_t) - logits_t[gt_t];
      ``accuracy``      float64 [B]: share of tokens whose predicted code (the argmax of the logits) is the ground truth;
      ``feat_mse``      float64 [B]: mean over tokens x channels of (E[gt_t] - lq_feat_t)^2;
      ``top_idx``       int64 [B,256]: the predicted codes.
    Every face's values depend on that face alone (not on B or ``max_batch``).  The stage-2 losses of
    codeformer_idx_model.py:100-115 on a batch are ``0.5 * cross_entropy.mean()`` (the cross-entropy term with
    ``entropy_loss_weight`` 0.5) and ``feat_mse.mean()`` (``l_feat_encoder`` before its ``feat_loss_weight``), computed here in
    float64.  A NaN logit gives that face a NaN cross-entropy; a ground-truth index outside [0, codebook_size) raises
    ``RuntimeError`` (the call synchronises the stream to find out)."""
    if not hasattr(net, 'latent_size') or not hasattr(net, 'idx_pred_layer'):
        raise RuntimeError('code_scores: net must be a CodeFormer (it scores the code_only logits)')
    if not torch.is_tensor(lq) or not lq.is_cuda:
        raise RuntimeError('code_scores: lq must be a CUDA tensor; there is no CPU fallback')
    if not torch.is_tensor(gt_codes) or not gt_codes.is_cuda:
        raise RuntimeError('code_scores: gt_codes must be a CUDA tensor; there is no CPU fallback')
    if lq.dtype == torch.uint8:
        if lq.dim() != 4 or tuple(lq.shape[1:]) != (512, 512, 3):
            raise RuntimeError(f'code_scores: uint8 faces must be [B,512,512,3] HWC BGR, got {tuple(lq.shape)}')
    elif lq.dtype == torch.float32:
        if lq.dim() != 4 or tuple(lq.shape[1:]) != (3, 512, 512):
            raise RuntimeError(f'code_scores: fp32 faces must be [B,3,512,512], got {tuple(lq.shape)}')
    else:
        raise RuntimeError(f'code_scores: lq must be uint8 or float32, got {lq.dtype}')
    B, dev = lq.shape[0], lq.device
    S, K, D = net.latent_size, net.codebook_size, net.embed_dim
    if gt_codes.dtype != torch.int64:
        raise RuntimeError(f'code_scores: gt_codes must be int64, got {gt_codes.dtype}')
    if gt_codes.device != dev:
        raise RuntimeError(f'code_scores: gt_codes are on {gt_codes.device}, the faces on {dev}')
    if tuple(gt_codes.shape) not in ((B, 16, 16), (B, S)) or 16 * 16 != S:
        raise RuntimeError(f'code_scores: gt_codes must be [{B},16,16] or [{B},{S}], got {tuple(gt_codes.shape)}')
    gt = gt_codes.reshape(B, S).contiguous()
    lq = lq.contiguous()
    lib = _lib.load()
    scores = torch.empty((B, 3), dtype=torch.float64, device=dev)
    top_idx = torch.empty((B, S), dtype=torch.int64, device=dev)
    step = max(1, int(max_batch))
    with net._lock, torch.cuda.device(dev):
        net._prepare(dev)
        st = _lib.stream(dev)
        E = net.quantize.embedding.weight.detach()
        if E.device != dev or E.dtype != torch.float32:
            raise RuntimeError('code_scores: the net must be on the faces\' device in float32')
        E = E.contiguous()
        for lo in range(0, B, step):
            hi = min(B, lo + step)
            n = hi - lo
            ws = net._cfb_workspace(dev, n)
            logits = torch.empty((n, S, K), dtype=torch.float32, device=dev)
            lq_feat = torch.empty((n, D, 16, 16), dtype=torch.float32, device=dev)
            if lq.dtype == torch.uint8:
                _lib.check(lib.cfb_codeformer_code_only_u8(net._net, _lib.ptr(lq[lo:hi]), _lib.ptr(logits), _lib.ptr(lq_feat),
                                                           _lib.ptr(top_idx[lo:hi]), n, _lib.ptr(ws), ws.numel(), st),
                           'cfb_codeformer_code_only_u8')
            else:
                _lib.check(lib.cfb_codeformer_forward(net._net, _lib.ptr(lq[lo:hi]), None, _lib.ptr(logits), _lib.ptr(lq_feat),
                                                      _lib.ptr(top_idx[lo:hi]), n, 0.0, 0, 1, _lib.ptr(ws), ws.numel(), st),
                           'cfb_codeformer_forward')
            feat = torch.empty((n, S, D), dtype=torch.float32, device=dev)
            _lib.check(lib.cfb_nchw_to_nhwc(_lib.ptr(lq_feat), _lib.ptr(feat), n, D, S, st), 'cfb_nchw_to_nhwc')
            _lib.check(lib.cfb_code_scores(_lib.ptr(logits), _lib.ptr(top_idx[lo:hi]), _lib.ptr(gt[lo:hi]), _lib.ptr(feat),
                                           _lib.ptr(E), n, S, K, D, _lib.ptr(scores[lo:hi]), st), 'cfb_code_scores')
        torch.cuda.current_stream(dev).synchronize()
        _lib.check(lib.cfb_check_async_status(), 'code_scores')
    return {'cross_entropy': scores[:, 0], 'accuracy': scores[:, 1] / S, 'feat_mse': scores[:, 2], 'top_idx': top_idx}
