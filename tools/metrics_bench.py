"""Timing of the restoration metrics (codeformer_b200.psnr_ssim) on one GPU, against the host restatement of basicsr's
calculate_psnr / calculate_ssim (oracle/metrics_oracle.py, numpy + cv2) on the same data.  Device events around warmed-up
calls, medians of --iters; the card, its power limit and clocks printed first.

  (a) 32 pairs of 512^2 uint8 faces, RGB and Y
  (b) a 32-face x 4-weight sweep [32,4,512,512,3] scored against its [32,512,512,3] ground truth, next to the
      forward_u8_sweep that produced it (seeded CodeFormer weights)
  (c) one 2160 x 3840 uint8 pair
  (d) the SSIM kernel alone (the raw C ABI call with want_psnr = 0) on (a): its float64 FMA / multiply rate from the
      instruction count of the algorithm, against the fp64 and HBM bounds of an H100 SXM's data sheet

The host times are per pair, measured on --host-pairs pairs (the host takes about half a second per 512^2 face).

    python tools/metrics_bench.py [--iters 20] [--host-pairs 2]
"""
import argparse
import ctypes
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import codeformer_b200 as cb                                   # noqa: E402
from codeformer_b200 import _lib, spec as S                    # noqa: E402
from oracle import metrics_oracle as MO                        # noqa: E402
from tools.detection_bench import card                         # noqa: E402

DEV = 'cuda:0'
FP64_FMA_PER_S = 34e12 / 2        # H100 SXM data sheet: 34 TFLOP/s fp64 without tensor cores, at up to 700 W
HBM_BYTES_PER_S = 3.35e12
TILE, HALO = 32, 42               # ssim_tile_kernel's output tile and halo (metrics.cu)


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


def host_ms(a, b, y, pairs):
    """Host restatement: PSNR + SSIM per pair, in ms (median over `pairs` pairs)."""
    ts = []
    for i in range(pairs):
        t = time.perf_counter()
        MO.psnr(a[i], b[i], 0, 'HWC', y)
        MO.ssim(a[i], b[i], 0, 'HWC', y)
        ts.append((time.perf_counter() - t) * 1e3)
    return statistics.median(ts)


def ssim_work(pairs, h, w, ce):
    """fp64 FMA + multiply instructions and the unique input bytes (uint8) of ssim_tile_kernel over `pairs` pairs."""
    tiles = -(-(h - 10) // TILE) * -(-(w - 10) // TILE)
    per_tile = HALO * TILE * 11 * (5 + 3) + TILE * TILE * 11 * 5     # horizontal: 5 FMA + 3 products per tap; vertical: 5 FMA
    return pairs * ce * tiles * per_tile, pairs * 2 * h * w * 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--host-pairs', type=int, default=2)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    print(card(), flush=True)
    rng = np.random.default_rng(0)
    gt = rng.integers(0, 256, (32, 512, 512, 3), dtype=np.uint8)
    rs = np.clip(gt.astype(np.int16) + rng.integers(-20, 21, gt.shape, dtype=np.int16), 0, 255).astype(np.uint8)
    gt_d, rs_d = torch.from_numpy(gt).to(DEV), torch.from_numpy(rs).to(DEV)

    for y in (False, True):                                                    # (a)
        ms = event_ms(lambda: cb.psnr_ssim(rs_d, gt_d, 0, y), args.iters)
        h = host_ms(rs, gt, y, args.host_pairs)
        print(f'(a) 32 x 512^2 uint8 {"Y" if y else "RGB"}: device {ms:.3f} ms ({ms / 32 * 1e3:.1f} us per pair); host '
              f'{h:.1f} ms per pair -> {32 * h / ms:.0f}x', flush=True)

    cf = cb.CodeFormer().to(DEV).eval()                                        # (b)
    cf.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    ws = [0.25, 0.5, 0.75, 1.0]
    sweep = cf.forward_u8_sweep(gt_d, ws)
    t_sweep = event_ms(lambda: cf.forward_u8_sweep(gt_d, ws), max(3, args.iters // 4))
    t_score = event_ms(lambda: cb.psnr_ssim(sweep, gt_d), args.iters)
    sw = sweep.cpu().numpy()
    h = host_ms(sw[:, 0], gt, False, args.host_pairs)
    print(f'(b) 32 faces x 4 weights: forward_u8_sweep {t_sweep:.1f} ms, psnr_ssim over the 128 pairs {t_score:.3f} ms '
          f'({100 * t_score / t_sweep:.2f} % of the sweep); host {128 * h / 1e3:.1f} s for the 128 pairs', flush=True)

    big_gt = rng.integers(0, 256, (1, 2160, 3840, 3), dtype=np.uint8)            # (c)
    big = np.clip(big_gt.astype(np.int16) + rng.integers(-20, 21, big_gt.shape, dtype=np.int16), 0, 255).astype(np.uint8)
    bg_d, bb_d = torch.from_numpy(big_gt).to(DEV), torch.from_numpy(big).to(DEV)
    ms = event_ms(lambda: cb.psnr_ssim(bb_d, bg_d), args.iters)
    h = host_ms(big, big_gt, False, 1)
    print(f'(c) one 2160x3840 uint8 pair: device {ms:.3f} ms; host {h:.0f} ms -> {h / ms:.0f}x', flush=True)

    lib = _lib.load()                                                          # (d)
    out = torch.empty(32, dtype=torch.float64, device=DEV)
    need = lib.cfb_psnr_ssim_workspace_bytes(32, 512, 512, 3, 0, 0)
    wsb = torch.empty(int(need), dtype=torch.uint8, device=DEV)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def ssim_only():
        _lib.check(lib.cfb_psnr_ssim(_lib.ptr(rs_d), _lib.ptr(gt_d), 0, 32, 1, 512, 512, 3, 0, 0, 0, 1, None, _lib.ptr(out),
                                     _lib.ptr(wsb), need, st), 'cfb_psnr_ssim')
    ms = event_ms(ssim_only, args.iters)
    ops, nbytes = ssim_work(32, 512, 512, 3)
    t_fp64, t_hbm = ops / FP64_FMA_PER_S * 1e3, nbytes / HBM_BYTES_PER_S * 1e3
    print(f'(d) SSIM kernel, 32 x 512^2 RGB: {ms:.3f} ms, {ops / 1e9:.2f} G fp64 FMA + multiply instructions -> '
          f'{ops / ms / 1e9:.2f} T/s = {100 * ops / ms / 1e9 / (FP64_FMA_PER_S / 1e12):.0f} % of the fp64 data-sheet rate; '
          f'bounds: fp64 {t_fp64:.3f} ms, HBM {t_hbm:.4f} ms ({"fp64" if t_fp64 > t_hbm else "HBM"}-bound)', flush=True)


if __name__ == '__main__':
    main()
