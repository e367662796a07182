"""Timing of the FID Inception-v3 and the FID statistics on one GPU; seeded random weights (oracle/fid_oracle.py), the
committed faces plus seeded noise faces.  Device events around warmed-up calls, medians of --iters, the card, its power limit
and clocks printed first.

  (a) features/s of InceptionV3.forward_u8 on 512 x 512 uint8 faces at B = 32 and 256, against the oracle's torch module on
      cuDNN (the same input stage in torch) with TF32 and with fp32
  (b) fid_statistics + frechet_distance on the device against np.cov + scipy's sqrtm (calculate_fid) on the host, N = 3000
  (c) a 32-face x 4-weight sweep scored with fid_scores next to forward_u8_sweep itself

    python tools/fid_bench.py [--iters 10]
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import codeformer_b200 as cb                                   # noqa: E402
from codeformer_b200 import spec as S                          # noqa: E402
from oracle import fid_oracle as fo                            # noqa: E402
from tools.arcface_bench import event_ms, faces                # noqa: E402
from tools.detection_bench import card                         # noqa: E402

DEV = 'cuda:0'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    print(card(), flush=True)
    sd = fo.random_fid_state_dict(1)
    net = cb.InceptionV3().to(DEV)
    net.load_state_dict(sd, strict=True)
    f = faces(256)
    mod = fo.reference_model({k: v for k, v in sd.items()}).to(DEV)
    for B in (32, 256):
        ms = event_ms(lambda: net.forward_u8(f[:B], max_batch=B), args.iters)
        line = f'forward_u8 512x512 B={B}: {ms:.2f} ms, {B / ms * 1e3:.0f} features/s'
        x = f[:B].flip(-1).permute(0, 3, 1, 2).float().div(255).contiguous()
        for tf32 in (True, False):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            mt = event_ms(lambda: mod(x), args.iters)
            line += f'; torch cuDNN {"TF32" if tf32 else "fp32"} {mt:.2f} ms ({B / mt * 1e3:.0f}/s)'
        print(line, flush=True)
        del x
    del mod
    torch.cuda.empty_cache()
    rng = np.random.default_rng(0)
    xa = (rng.normal(size=(3000, 2048)) @ (rng.normal(size=(2048, 2048)) / 45)).astype(np.float32)
    xb = (1.1 * rng.normal(size=(3000, 2048)) @ (rng.normal(size=(2048, 2048)) / 45)).astype(np.float32)
    ta, tb = torch.from_numpy(xa).to(DEV), torch.from_numpy(xb).to(DEV)
    ms_stats = event_ms(lambda: cb.fid_statistics(ta), args.iters)
    sa, sb = cb.fid_statistics(ta), cb.fid_statistics(tb)
    ms_dist = event_ms(lambda: cb.frechet_distance(sa, sb), max(3, args.iters // 2))
    t0 = time.perf_counter()
    ma, ca = np.mean(xa, axis=0), np.cov(xa, rowvar=False)
    t1 = time.perf_counter()
    mb_, cb_ = np.mean(xb, axis=0), np.cov(xb, rowvar=False)
    t2 = time.perf_counter()
    host = cb.calculate_fid(ma, ca, mb_, cb_)
    t3 = time.perf_counter()
    dev = cb.frechet_distance(sa, sb)
    print(f'N=3000 x 2048: fid_statistics {ms_stats:.2f} ms, frechet_distance {ms_dist:.1f} ms on the device; host np.cov '
          f'{(t1 - t0) * 1e3:.0f} ms, calculate_fid (scipy sqrtm) {(t3 - t2) * 1e3:.0f} ms; FID device {dev:.6f} host {host:.6f}',
          flush=True)
    cf = cb.CodeFormer().to(DEV).eval()
    cf.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    ws = [0.25, 0.5, 0.75, 1.0]
    ref = f[:32]
    sweep = cf.forward_u8_sweep(ref, ws)
    stats = cb.fid_statistics(cb.inception_features(f[32:96], net))
    t_sweep = event_ms(lambda: cf.forward_u8_sweep(ref, ws), max(3, args.iters // 2))
    t_score = event_ms(lambda: cb.fid_scores(sweep, stats, net), max(3, args.iters // 2))
    print(f'32 faces x 4 weights: forward_u8_sweep {t_sweep:.1f} ms, fid_scores over the 128 images {t_score:.1f} ms '
          f'({100 * t_score / t_sweep:.1f} % of the sweep)', flush=True)


if __name__ == '__main__':
    main()
