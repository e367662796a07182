"""Timing of ResNetArcFace([2,2,2,2]) identity embeddings on one GPU; seeded random weights, the committed faces plus seeded
noise faces.  Device events around warmed-up calls, medians of --iters, the card, its power limit and clocks printed first.

  (a) embeddings/s of forward_u8 at B = 32 and B = 256
  (b) scoring a 32-face x 4-weight sweep: identity_similarity(net, faces, sweep) next to forward_u8_sweep(faces, ws) itself

    python tools/arcface_bench.py [--iters 10]
"""
import argparse
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import codeformer_b200 as cb                                   # noqa: E402
from codeformer_b200 import arcface as A, spec as S            # noqa: E402
from tools.detection_bench import card                         # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'


def event_ms(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def faces(n):
    f = np.load(os.path.join(ROOT, 'tests', 'golden', 'faces.npz'))['faces']
    extra = np.random.default_rng(0).integers(0, 256, size=(max(0, n - len(f)), 512, 512, 3), dtype=np.uint8)
    return torch.from_numpy(np.concatenate([f, extra])[:n]).to(DEV)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    print(card(), flush=True)
    net = cb.ResNetArcFace('IRBlock', [2, 2, 2, 2], use_se=False)
    net.load_state_dict(A.random_arcface_state_dict(seed=1), strict=True)
    net = net.to(DEV).eval()
    f256 = faces(256)
    for B in (32, 256):
        ms = event_ms(lambda: net.forward_u8(f256[:B]), args.iters)
        print(f'forward_u8 B={B}: {ms:.3f} ms per call, {B / ms * 1e3:.0f} embeddings/s', flush=True)
    cf = cb.CodeFormer().to(DEV).eval()
    cf.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    f32, ws = f256[:32], [0.25, 0.5, 0.75, 1.0]
    sweep = cf.forward_u8_sweep(f32, ws)
    t_sweep = event_ms(lambda: cf.forward_u8_sweep(f32, ws), max(3, args.iters // 2))
    t_score = event_ms(lambda: cb.identity_similarity(net, f32, sweep), args.iters)
    print(f'32 faces x 4 weights: forward_u8_sweep {t_sweep:.1f} ms, identity_similarity over the 32 + 128 faces '
          f'{t_score:.2f} ms ({100 * t_score / t_sweep:.2f} % of the sweep)', flush=True)


if __name__ == '__main__':
    main()
