"""RRDBNet precision modes on one GPU: fp32 (split fp16 x3, the default) against fp16 (single pass), alternated in one process
over --rounds rounds, medians of each.  Reports
  * one 480x480 tile of RRDBNet(3, 3, scale=2, 23 blocks) (RealESRGANer tile 400 + 2 x 40 pad), CUDA events;
  * RealESRGANer.enhance of a synthetic 1920x1080 uint8 image with tile=400, tile_pad=40 (host clock around a synchronised call);
  * for context, oracle/rrdbnet_oracle.py on cuDNN on the same tile: fp32 (allow_tf32=False), TF32, and fp16 (state dict and
    input .half() on CUDA, the reference's half=True);
  * --profile: the summed time of each CUDA kernel of one tile forward per mode (torch.profiler), e.g. the GEN conv kernels.

    python tools/rrdb_precision_bench.py [--rounds 3] [--iters 10] [--profile]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import codeformer_b200 as cb                                   # noqa: E402
from codeformer_b200 import spec as S                           # noqa: E402
from oracle import rrdbnet_oracle as RO                         # noqa: E402

MODES = ('fp32', 'fp16')


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                        # noqa: BLE001
        pl = f'unknown ({e})'
    return f'{name}, power limit / max SM clock: {pl}'


def timed(fn, iters, warmup=2):
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
    return float(np.median(ts))


def wall(fn, iters, warmup=1):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--profile', action='store_true')
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    dev = 'cuda:0'
    print(card())
    sd = S.random_state_dict(S.rrdbnet_spec(3, 3, 2, 64, 23, 32), 21)
    net = cb.RRDBNet(3, 3, scale=2, num_feat=64, num_block=23, num_grow_ch=32)
    net.load_state_dict(sd, strict=True)
    net = net.to(dev).eval()
    x = torch.rand(1, 3, 480, 480, generator=torch.Generator().manual_seed(4)).to(dev)
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for mode in MODES:
            net.set_precision(mode)
            net(x)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                net(x)
                torch.cuda.synchronize()
            print(f'--- {mode}: kernels of one 480x480 tile forward')
            print(prof.key_averages().table(sort_by='cuda_time_total', row_limit=8, max_name_column_width=110))
        return
    img = np.random.default_rng(0).integers(0, 256, (1080, 1920, 3), dtype=np.uint8)
    up = cb.RealESRGANer(scale=2, model=net, tile=400, tile_pad=40, pre_pad=0, device=dev)
    res = {m: {'tile': [], 'enhance': []} for m in MODES}
    outs = {}
    for _ in range(args.rounds):
        for mode in MODES:
            net.set_precision(mode)
            res[mode]['tile'].append(timed(lambda: net(x), args.iters))
            res[mode]['enhance'].append(wall(lambda: up.enhance(img, outscale=2), max(1, args.iters // 5)))
            outs[mode] = net(x)
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    sd_half = {k: v.half() for k, v in sd_dev.items()}
    torch.backends.cudnn.allow_tf32 = False
    ref = {'cudnn fp32': timed(lambda: RO.rrdbnet_forward(sd_dev, x, scale=2, num_block=23), args.iters)}
    ref_out = RO.rrdbnet_forward(sd_dev, x, scale=2, num_block=23)
    torch.backends.cudnn.allow_tf32 = True
    ref['cudnn tf32'] = timed(lambda: RO.rrdbnet_forward(sd_dev, x, scale=2, num_block=23), args.iters)
    xh = x.half()
    ref['cudnn fp16'] = timed(lambda: RO.rrdbnet_forward(sd_half, xh, scale=2, num_block=23), args.iters)
    half_out = RO.rrdbnet_forward(sd_half, xh, scale=2, num_block=23).float()
    for mode in MODES:
        t, e = np.median(res[mode]['tile']), np.median(res[mode]['enhance'])
        print(f'{mode}: 480x480 x2 tile {t:.2f} ms (rounds {", ".join(f"{v:.2f}" for v in res[mode]["tile"])}); '
              f'enhance 1920x1080 tile 400 pad 40: {e:.1f} ms (rounds {", ".join(f"{v:.1f}" for v in res[mode]["enhance"])}); '
              f'max-abs vs cuDNN fp32 {float((outs[mode] - ref_out).abs().max()):.2e}')
    for k, v in ref.items():
        print(f'oracle on {k}: 480x480 x2 tile {v:.2f} ms')
    print(f'oracle cuDNN fp16 (.half()) max-abs vs cuDNN fp32 {float((half_out - ref_out).abs().max()):.2e}')


if __name__ == '__main__':
    main()
