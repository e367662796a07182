"""Restatements for the latent-code tests: the loop body of scripts/generate_latent_gt.py and the stage-2 terms of
codeformer_idx_model.py:100-115 in float64.  Test infrastructure; the product never imports it."""
import cv2
import numpy as np
import torch

from oracle.plumbing_oracle import face_to_input


def script_latent_gt(images, names, vqgan, device):
    """scripts/generate_latent_gt.py:42-66 with the one-argument encoder call: for 'orig' then 'hflip', every image
    (uint8 [H,W,3] BGR) -> cv2.flip(img, 1) for hflip -> img2tensor(img / 255., bgr2rgb=True, float32=True) +
    normalize(0.5, 0.5) -> vqgan.encoder -> vqgan.quantize -> min_encoding_indices.view(16, 16) as numpy."""
    latent = {'orig': {}, 'hflip': {}}
    for kind in ['orig', 'hflip']:
        for img, name in zip(images, names):
            img = np.array(img)
            if kind == 'hflip':
                cv2.flip(img, 1, img)
            x = torch.from_numpy(face_to_input(img[None])).to(device)
            with torch.no_grad():
                z = vqgan.encoder(x)
                _, _, log = vqgan.quantize(z)
            latent[kind][name] = log['min_encoding_indices'].view(16, 16).cpu().numpy()
    return latent


def cross_entropy_f64(logits, gt):
    """Per face: mean over tokens of logsumexp(logits_t) - logits_t[gt_t], in float64.  logits [B,T,K], gt [B,T]."""
    lg = logits.double()
    m = lg.max(dim=2, keepdim=True).values
    lse = m.squeeze(2) + torch.log(torch.exp(lg - m).sum(dim=2))
    return (lse - lg.gather(2, gt.unsqueeze(2)).squeeze(2)).mean(dim=1)


def feat_mse_f64(codebook, gt, lq_feat):
    """Per face: mean over tokens x channels of (E[gt_t] - lq_feat_t)^2 in float64.  lq_feat NCHW [B,D,16,16]."""
    B, D = lq_feat.shape[:2]
    q = lq_feat.double().permute(0, 2, 3, 1).reshape(B, -1, D)
    e = codebook.double()[gt]
    return ((e - q) ** 2).mean(dim=(1, 2))
