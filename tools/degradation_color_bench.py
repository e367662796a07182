"""Timing of the colorization and inpainting inputs (codeformer_b200.degradation with COLORIZATION_OPTIONS /
INPAINTING_OPTIONS) on one GPU against the same stages on the host (cv2 and torchvision, as FFHQBlindDataset runs them).
Device events around warmed-up calls (medians of --iters), host wall clocks; the card, its power limit and clocks, and the
host's CPU and thread counts printed first, in the same run.

  colorization  ms per 512 x 512 face of degrade_faces at B = 32, with the preset's probabilities and with every colour
                stage drawn (probabilities 1), against the host chain: cv2 blur / resize / JPEG / resize, the numpy shift,
                cv2 gray and torchvision's color_jitter_pt ops on the CPU
  inpainting    ms per face of degrade_faces at B = 32 (the masks are drawn on the host with PIL, timed apart), against the
                host's where(mask, 255, gt) in float as the dataset computes it

    python tools/degradation_color_bench.py [--iters 10]
"""
import argparse
import os
import random
import sys
import time

import cv2
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import codeformer_b200 as cb                                   # noqa: E402
from codeformer_b200 import degradation as DG                  # noqa: E402
from tools.arcface_bench import event_ms, faces                # noqa: E402
from tools.detection_bench import card                         # noqa: E402


def host_color(gt_u8, p, in_size=512):
    """The dataset's float path on the host: chain, shift, gray, torchvision ops, round."""
    import torchvision.transforms.functional as TF
    if p['kernel'] is not None:
        img = cv2.filter2D(gt_u8.astype(np.float32) / 255., -1, p['kernel'])
        img = cv2.resize(img, (p['size'], p['size']), interpolation=cv2.INTER_LINEAR)
        img = np.clip(img + p['noise'], 0, 1)
        _, enc = cv2.imencode('.jpg', img * 255., [int(cv2.IMWRITE_JPEG_QUALITY), p['quality']])
        img = np.float32(cv2.imdecode(enc, 1)) / 255.
        img = cv2.resize(img, (in_size, in_size), interpolation=cv2.INTER_LINEAR)
    else:
        img = gt_u8.astype(np.float32) / 255.
    if p['mask'] is not None:
        img = np.where(p['mask'][..., None] != 0, 1., img)
    if p['jitter'] is not None:
        img = np.clip(img + p['jitter'], 0, 1)
    if p['gray']:
        img = np.tile(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)[:, :, None], [1, 1, 3])
    t = torch.from_numpy(np.ascontiguousarray(img[..., ::-1].transpose(2, 0, 1))).float()
    for op, f in p['jitter_pt'] or []:
        t = getattr(TF, f'adjust_{op}')(t, f)
    return np.clip((t * 255.).round(), 0, 255).to(torch.uint8).numpy()


def sample(n, seed, opts, **over):
    return DG.sample_degradations(n, py_rng=random.Random(seed), np_rng=np.random.RandomState(seed),
                                  torch_rng=torch.Generator().manual_seed(seed), **dict(opts, **over))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--host-faces', type=int, default=8)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    print(card(), f'| host: {os.cpu_count()} CPUs, cv2 threads {cv2.getNumThreads()}, torch threads '
          f'{torch.get_num_threads()}', flush=True)
    gt = faces(32)
    gt_np = gt.cpu().numpy()
    n = args.host_faces
    runs = (('colorization (preset)', DG.COLORIZATION_OPTIONS, {}),
            ('colorization (every stage)', DG.COLORIZATION_OPTIONS,
             dict(color_jitter_prob=1.0, color_jitter_pt_prob=1.0, gray_prob=0.0)),
            ('inpainting', DG.INPAINTING_OPTIONS, {}))
    for name, opts, over in runs:
        t0 = time.perf_counter()
        params = sample(32, 0, opts, **over)
        t_sample = (time.perf_counter() - t0) * 1e3 / 32
        ms = event_ms(lambda: cb.degrade_faces(gt, params), args.iters)
        host_color(gt_np[0], params[0])               # imports and first-call set-up stay out of the host time
        t0 = time.perf_counter()
        for i in range(n):
            host_color(gt_np[i], params[i])
        t_host = (time.perf_counter() - t0) * 1e3 / n
        print(f'{name}: degrade_faces B=32 {ms / 32:.3f} ms per face; host {t_host:.1f} ms per face (mean of {n}), '
              f'{t_host / (ms / 32):.0f}x; host sampler {t_sample:.2f} ms per face', flush=True)
    # the colour stages' own share: the chain without them, same parameters
    params = sample(32, 0, DG.COLORIZATION_OPTIONS, color_jitter_prob=1.0, color_jitter_pt_prob=1.0)
    plain = [dict(p, jitter=None, gray=False, jitter_pt=None) for p in params]
    a = event_ms(lambda: cb.degrade_faces(gt, plain), args.iters)
    b = event_ms(lambda: cb.degrade_faces(gt, params), args.iters)
    print(f'stage-2 chain B=32: {a / 32:.3f} ms per face without colour stages, {b / 32:.3f} with every one', flush=True)


if __name__ == '__main__':
    main()
