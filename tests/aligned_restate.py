"""Restatements of the face-only scripts' caller loops, shared by the GPU tests of the aligned-face path
(tests/test_gpu_aligned.py) and pinned on the reference's own functions by tests/test_aligned_restate_cpu.py.

inpaint_blend     inference_inpainting.py:68-74: mask where the normalised input sums to 3 over its channels, then
                  (1-mask)*input + mask*output in float32 (torch, on whatever device the tensors live)
aligned_crop      inference_codeformer.py:182-184: cv2.resize(img, (512, 512), INTER_LINEAR), then is_gray(img, threshold=10)
"""
import numpy as np
import torch

from codeformer_b200.wholeimage import is_gray


def inpaint_mask(x):
    """float32 [B,3,H,W] normalised RGB input -> float32 [B,1,H,W]: 1 where the channel sum equals 3 (:68-71)."""
    m = torch.zeros((x.shape[0], 1) + tuple(x.shape[2:]), dtype=torch.float32, device=x.device)
    m[torch.sum(x, dim=1, keepdim=True) == 3] = 1.0
    return m


def inpaint_blend(x, out):
    """(1-mask)*input + mask*output (:74) for a batch."""
    mask = inpaint_mask(x)
    return (1 - mask) * x + mask * out


def aligned_crop(img):
    """-> (the 512x512 crop, its gray flag), as the --has_aligned branch makes them from one image."""
    import cv2
    crop = cv2.resize(np.asarray(img), (512, 512), interpolation=cv2.INTER_LINEAR)
    return crop, is_gray(crop, threshold=10)
