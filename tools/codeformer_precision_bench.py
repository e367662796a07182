"""CodeFormer precision modes on one GPU: fp32 (split fp16 x3 everywhere, the default) against fp16 (single-pass generator and
Fuse_sft_block convs), alternated in one process over --rounds rounds, medians of each.  Reports
  * one batch-32 CodeFormer.forward(w=0.5, adain=True) step, CUDA events (the model and inputs of bench.py);
  * CodeFormer.restore_faces of 32 uint8 faces (host clock around the synchronised call, staging included);
  * single-face latency, forward of one face (the CUDA-graph path), CUDA events;
  * output deltas of the fp16 mode on the committed fixture faces (w=0.5, adain): max-abs of `out` against the fp32 mode,
    and the histogram of the uint8 level differences of the restored faces;
  * --profile (a separate run): the summed time of each CUDA kernel of one batch-32 step per mode (torch.profiler).
The card name, power limit and maximum SM clock are read in the same run.

    python tools/codeformer_precision_bench.py [--rounds 3] [--iters 10] [--profile] [--batch 32]
"""
import argparse
import collections
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import codeformer_b200 as cb                                   # noqa: E402
from codeformer_b200 import spec as S                           # noqa: E402
from tests.util import faces_input, golden                      # noqa: E402

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


def profile_step(net, x):
    from torch.profiler import ProfilerActivity, profile
    for mode in MODES:
        net.set_precision(mode)
        for _ in range(2):
            net(x, w=0.5, adain=True)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            net(x, w=0.5, adain=True)
            torch.cuda.synchronize()
        per = collections.defaultdict(lambda: [0, 0.0])
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                per[ev.name][0] += 1
                per[ev.name][1] += ev.time_range.elapsed_us() / 1e3
        total = sum(v[1] for v in per.values())
        conv = sum(v[1] for k, v in per.items() if 'conv_tc_kernel' in k)
        print(f'--- {mode}: kernel time of one batch-{x.shape[0]} step {total:.2f} ms, conv_tc_kernel {conv:.2f} ms')
        print(f'{"ms":>9} {"share":>7} {"calls":>6}  kernel')
        for name, (calls, ms) in sorted(per.items(), key=lambda kv: -kv[1][1])[:24]:
            print(f'{ms:9.3f} {100 * ms / total:6.2f}% {calls:6d}  {name[:150]}')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--profile', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('codeformer_precision_bench: no CUDA device')
    torch.set_grad_enabled(False)
    print(card())
    net = cb.CodeFormer(dim_embd=512, codebook_size=1024, n_head=8, n_layers=9,
                        connect_list=['32', '64', '128', '256']).cuda().eval()
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    g = torch.Generator().manual_seed(100)
    x = torch.randn(args.batch, 3, 512, 512, generator=g).clamp_(-1, 1).cuda()
    if args.profile:
        profile_step(net, x)
        return
    faces_rgb = golden('faces.npz')['faces']
    faces_bgr = np.ascontiguousarray(faces_rgb[..., ::-1])
    many = [faces_bgr[i % len(faces_bgr)] for i in range(args.batch)]
    x1 = faces_input(slice(0, 1)).cuda()
    res = {m: collections.defaultdict(list) for m in MODES}
    for _ in range(args.rounds):
        for mode in MODES:
            net.set_precision(mode)
            res[mode]['step'].append(timed(lambda: net(x, w=0.5, adain=True), args.iters))
            res[mode]['restore'].append(wall(lambda: net.restore_faces(many, w=0.5, adain=True, on_error='raise'),
                                             max(1, args.iters // 2)))
            res[mode]['single'].append(timed(lambda: net(x1, w=0.5, adain=True), 3 * args.iters))
    for mode in MODES:
        r = res[mode]
        step = np.median(r['step'])
        print(f'{mode}: B={args.batch} step {step:.2f} ms = {1e3 * args.batch / step:.1f} faces/s '
              f'(rounds {", ".join(f"{v:.2f}" for v in r["step"])}); restore_faces {args.batch} u8 faces '
              f'{np.median(r["restore"]):.1f} ms (rounds {", ".join(f"{v:.1f}" for v in r["restore"])}); single face '
              f'{np.median(r["single"]):.2f} ms (rounds {", ".join(f"{v:.2f}" for v in r["single"])})')
    # output deltas on the committed faces
    xf = faces_input().cuda()
    outs, u8 = {}, {}
    for mode in MODES:
        net.set_precision(mode)
        outs[mode] = [net(xf[i:i + 1], w=0.5, adain=True) for i in range(xf.shape[0])]
        u8[mode] = np.stack(net.restore_faces(list(faces_bgr), w=0.5, adain=True, on_error='raise'))
    d_out = max(float((a[0] - b[0]).abs().max()) for a, b in zip(outs['fp32'], outs['fp16']))
    same_codes = all(torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]) for a, b in zip(outs['fp32'], outs['fp16']))
    d = np.abs(u8['fp32'].astype(np.int32) - u8['fp16'].astype(np.int32)).ravel()
    hist = np.bincount(d)
    print(f'{len(faces_bgr)} fixture faces, fp16 vs fp32 mode: out max-abs {d_out:.3e}; logits and lq_feat bit-identical: '
          f'{same_codes}')
    print('uint8 level differences of the restored faces: ' +
          ', '.join(f'{k}: {int(v)} ({100 * v / d.size:.3f} %)' for k, v in enumerate(hist) if v))


if __name__ == '__main__':
    main()
