"""Timing of the synthetic degradation chain (codeformer_b200.degradation) on one GPU against the same chain on the host with
cv2, and of one degrade -> restore -> score loop.  Device events around warmed-up calls (medians of --iters), host wall
clocks; the card, its power limit and clocks, and the host's cv2 thread count printed first.

  (a) ms per 512 x 512 face of degrade_faces at B = 1 and B = 32, stage-2 and stage-3 ranges, against the host chain
      (cv2.filter2D, resize, noise, imencode / imdecode, resize), and the share of the host sampler (kernel + noise draw)
  (b) 32 faces: degrade_faces -> forward_u8_sweep (4 weights) -> psnr_ssim + lpips_distance + identity_similarity on
      seeded random weights, with the share of each stage

    python tools/degradation_bench.py [--iters 10]
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
from codeformer_b200 import spec as S                          # noqa: E402
from codeformer_b200.arcface import random_arcface_state_dict  # noqa: E402
from oracle import lpips_oracle as LO                          # noqa: E402
from tools.arcface_bench import event_ms, faces                # noqa: E402
from tools.detection_bench import card                         # noqa: E402


def host_chain(gt_u8, p, in_size=512):
    img = cv2.filter2D(gt_u8.astype(np.float32) / 255., -1, p['kernel'])
    img = cv2.resize(img, (p['size'], p['size']), interpolation=cv2.INTER_LINEAR)
    img = np.clip(img + p['noise'], 0, 1)
    _, enc = cv2.imencode('.jpg', img * 255., [int(cv2.IMWRITE_JPEG_QUALITY), p['quality']])
    img = np.float32(cv2.imdecode(enc, 1)) / 255.
    img = cv2.resize(img, (in_size, in_size), interpolation=cv2.INTER_LINEAR)
    return np.clip((img * 255.).round(), 0, 255).astype(np.uint8)


def sample(n, seed, ranges):
    return DG.sample_degradations(n, py_rng=random.Random(seed), np_rng=np.random.RandomState(seed), **ranges)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--host-faces', type=int, default=8)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    print(card(), f'| host: {os.cpu_count()} CPUs, cv2 threads {cv2.getNumThreads()}', flush=True)
    gt = faces(32)
    gt_np = gt.cpu().numpy()
    for name, r in (('stage2', DG.STAGE2_RANGES), ('stage3', DG.STAGE3_RANGES)):
        t0 = time.perf_counter()
        params = sample(32, 0, r)
        t_sample = (time.perf_counter() - t0) * 1e3 / 32
        full = sum(2 * p['size'] >= 512 for p in params)      # faces whose blur covers every source pixel
        for B in (1, 32):
            ms = event_ms(lambda: cb.degrade_faces(gt[:B], params[:B]), args.iters)
            print(f'{name} B={B}: degrade_faces {ms / B:.3f} ms per face', flush=True)
        n = args.host_faces
        t0 = time.perf_counter()
        for i in range(n):
            host_chain(gt_np[i], params[i])
        t_host = (time.perf_counter() - t0) * 1e3 / n
        print(f'{name}: host chain {t_host:.1f} ms per face (mean of {n}); host sampler {t_sample:.2f} ms per face '
              f'({full} of 32 faces blurred in full, 2 * size >= 512); '
              f'device B=32 is {t_host / (ms / 32):.0f}x faster than the host chain; '
              f'the sampler is {100 * t_sample / (t_sample + ms / 32):.0f} % of sampler + device time', flush=True)
    # (b) one evaluation loop on seeded weights
    cf = cb.CodeFormer().to('cuda').eval()
    cf.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    lp = cb.LPIPS().to('cuda')
    lp.load_state_dict(LO.random_lpips_state_dict(1), strict=True)
    arc = cb.ResNetArcFace('IRBlock', [2, 2, 2, 2], use_se=False)
    arc.load_state_dict(random_arcface_state_dict(seed=1), strict=True)
    arc = arc.to('cuda')
    ws = [0.25, 0.5, 0.75, 1.0]
    params = sample(32, 1, DG.STAGE2_RANGES)
    lq, _ = cb.degrade_faces(gt, params)
    sweep = cf.forward_u8_sweep(lq, ws)
    t = {'degrade': event_ms(lambda: cb.degrade_faces(gt, params), args.iters),
         'forward_u8_sweep': event_ms(lambda: cf.forward_u8_sweep(lq, ws), max(3, args.iters // 2)),
         'psnr_ssim': event_ms(lambda: cb.psnr_ssim(sweep, gt), args.iters),
         'lpips_distance': event_ms(lambda: cb.lpips_distance(sweep, gt, lp), args.iters),
         'identity_similarity': event_ms(lambda: cb.identity_similarity(arc, gt, sweep), args.iters)}
    tot = sum(t.values())
    print(f'loop, 32 faces x {len(ws)} weights: {tot:.1f} ms: ' +
          ', '.join(f'{k} {v:.2f} ms ({100 * v / tot:.1f} %)' for k, v in t.items()), flush=True)


if __name__ == '__main__':
    main()
