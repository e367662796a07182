"""Timing of LPIPS-VGG on one GPU; seeded random weights (the oracle's He-scaled layout), the committed faces plus seeded
noise faces.  Device events around warmed-up calls, medians of --iters, the card, its power limit and clocks printed first.

  (a) pairs/s of forward_u8 on 512 x 512 faces at B = 1 and B = 32
  (b) scoring a 32-face x 4-weight sweep: lpips_distance(sweep, faces, net) next to forward_u8_sweep(faces, ws) itself
  (c) one 2160 x 3840 pair
  (d) the same network as a torch module (oracle/lpips_oracle.py) on cuDNN, B = 32, TF32 off and torch's default

    python tools/lpips_bench.py [--iters 10]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import codeformer_b200 as cb                                   # noqa: E402
from codeformer_b200 import spec as S                          # noqa: E402
from oracle import lpips_oracle as LO                          # noqa: E402
from tools.arcface_bench import event_ms, faces                # noqa: E402
from tools.detection_bench import card                         # noqa: E402

DEV = 'cuda:0'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    print(card(), flush=True)
    sd = LO.random_lpips_state_dict(1)
    net = cb.LPIPS().to(DEV)
    net.load_state_dict(sd, strict=True)
    f = faces(64)
    ref, cand = f[:32], f[32:]
    for B in (1, 32):
        ms = event_ms(lambda: net.forward_u8(ref[:B], cand[:B]), args.iters)
        print(f'forward_u8 512x512 B={B}: {ms:.3f} ms per call, {B / ms * 1e3:.1f} pairs/s', flush=True)
    cf = cb.CodeFormer().to(DEV).eval()
    cf.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    ws = [0.25, 0.5, 0.75, 1.0]
    sweep = cf.forward_u8_sweep(ref, ws)
    t_sweep = event_ms(lambda: cf.forward_u8_sweep(ref, ws), max(3, args.iters // 2))
    t_score = event_ms(lambda: cb.lpips_distance(sweep, ref, net), args.iters)
    print(f'32 faces x 4 weights: forward_u8_sweep {t_sweep:.1f} ms, lpips_distance over the 32 + 128 images '
          f'{t_score:.1f} ms ({100 * t_score / t_sweep:.1f} % of the sweep)', flush=True)
    del cf, sweep
    g = torch.Generator(device=DEV).manual_seed(0)
    big = torch.randint(0, 256, (2, 2160, 3840, 3), dtype=torch.uint8, device=DEV, generator=g)
    ms = event_ms(lambda: net.forward_u8(big[:1], big[1:]), max(3, args.iters // 2), warmup=1)
    print(f'one 2160x3840 pair: {ms:.1f} ms (workspace {net._ws.numel() / 2**30:.2f} GiB)', flush=True)
    del big
    net._ws = None
    torch.cuda.empty_cache()
    mod = LO.LPIPS().to(DEV)
    mod.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    x0 = (ref.flip(-1).permute(0, 3, 1, 2).float() / 127.5 - 1).contiguous()
    x1 = (cand.flip(-1).permute(0, 3, 1, 2).float() / 127.5 - 1).contiguous()
    for tf32 in (False, True):
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        ms = event_ms(lambda: mod(x0, x1), args.iters)
        print(f'torch module on cuDNN (TF32 {"on" if tf32 else "off"}) B=32: {ms:.3f} ms per call, {32 / ms * 1e3:.1f} pairs/s',
              flush=True)


if __name__ == '__main__':
    main()
