"""Per-shape time of the halo conv kernels of CodeFormer.forward on their default tiles vs 128 x 64 pixel-major tiles (CFB_TC_BN=64).

Every distinct 3x3 stride-1 / Upsample conv shape of the forward with Cout % 128 == 0 (128 x 128 tiles by default) and the
Cout = 64 shapes at 512^2 (channel-major 128 x 64 tiles by default; the raw-plane row times the kernel without the fused
transform) is timed alone with CUDA events by cfb_debug_time_conv at batch 32.  CFB_TC_BN is read once per process, so the two settings run
in separate processes, alternating A/B/A/B (--rounds), and the median per setting is reported.  Nominal FLOPs are the conv's
2*M*N*K (Upsample: of the 3x3 conv at the output resolution, as the forward's FLOP count has them); the fraction is of the
H100 SXM data-sheet dense bf16/fp16 rate.  The card name and power limit are read in the same run.

    python tools/conv_tile_sweep.py [--rounds 2] [--batch 32] [--reps 10]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK_TFLOPS = 989.0

# (H of the conv's input, Cin, Cout, mode, GroupNorm+SiLU fused transform); mode 0 = 3x3 'same', 2 = Upsample (nearest x2 + 3x3)
SHAPES = [
    (256, 64, 128, 0, True), (256, 128, 128, 0, True), (128, 128, 128, 0, True), (64, 128, 256, 0, True),
    (64, 256, 256, 0, True), (32, 256, 256, 0, True), (16, 256, 512, 0, True), (16, 512, 512, 0, True),
    (32, 512, 256, 0, True), (128, 256, 128, 0, True), (256, 256, 128, 0, True),
    (16, 512, 512, 2, False), (32, 256, 256, 2, False), (64, 256, 256, 2, False), (128, 128, 128, 2, False),
    (256, 128, 128, 2, False),
    (512, 64, 64, 0, True), (512, 128, 64, 0, True), (512, 64, 64, 0, False),
]

CHILD = r'''
import ctypes, json, sys
import torch
sys.path.insert(0, %r)
from codeformer_b200 import _lib
lib = _lib.load()
N, reps = int(sys.argv[1]), int(sys.argv[2])
res = []
for H, Cin, Cout, mode, xf in json.loads(sys.argv[3]):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(N, H, H, Cin, generator=g).cuda()
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (9 * Cin) ** 0.5).cuda()
    Ho = 2 * H if mode == 2 else H
    out = torch.empty(N, Ho, Ho, Cout, device='cuda')
    sc = (1 + 0.1 * torch.randn(N, Cin, generator=g)).cuda() if xf else None
    sh = (0.1 * torch.randn(N, Cin, generator=g)).cuda() if xf else None
    wsb = lib.cfb_conv2d_workspace_bytes(N, H, H, Cin, Cout, 3, mode)
    ws = torch.empty(int(wsb), dtype=torch.uint8, device='cuda')
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ms = ctypes.c_float(0)
    for _ in range(2):                        # the first call warms the module and the weight split
        _lib.check(lib.cfb_debug_time_conv(_lib.ptr(x), _lib.ptr(w), _lib.ptr(out), N, H, H, Cin, Cout, 3, mode, reps,
                                           _lib.ptr(ws), wsb, st, _lib.ptr(sc), _lib.ptr(sh), 1 if xf else 0,
                                           ctypes.byref(ms)), 'cfb_debug_time_conv')
    res.append(float(ms.value))
    del x, w, out, ws
    torch.cuda.empty_cache()
print('RESULT ' + json.dumps(res))
''' % ROOT


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def run_side(bn, batch, reps):
    env = dict(os.environ)
    env.pop('CFB_TC_BN', None)
    if bn == 64:
        env['CFB_TC_BN'] = '64'
    p = subprocess.run([sys.executable, '-c', CHILD, str(batch), str(reps), json.dumps(SHAPES)], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=1800)
    if p.returncode != 0:
        raise RuntimeError(p.stdout[-2000:] + p.stderr[-2000:])
    line = [ln for ln in p.stdout.splitlines() if ln.startswith('RESULT ')][-1]
    return json.loads(line[len('RESULT '):])


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--rounds', type=int, default=2, help='A/B pairs (each side runs in its own process)')
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--reps', type=int, default=10, help='launches per CUDA-event timing')
    args = ap.parse_args()
    card = gpu_info()
    times = {64: [], None: []}           # 64: CFB_TC_BN=64; None: default tiles
    for _ in range(args.rounds):
        for bn in (64, None):
            times[bn].append(run_side(bn, args.batch, args.reps))
    print(json.dumps({'gpu': card, 'batch': args.batch, 'rounds': args.rounds}))
    for i, (H, Cin, Cout, mode, xf) in enumerate(SHAPES):
        Ho = 2 * H if mode == 2 else H
        flops = 2.0 * args.batch * Ho * Ho * Cout * Cin * 9
        row = {'shape': f'{"up" if mode == 2 else "conv"} {Cin}->{Cout} @{Ho}^2{" gn+silu" if xf else " raw"}',
               'gflop': round(flops / 1e9, 1)}
        for bn, key in ((64, 'bn64'), (None, 'default')):
            ms = [t[i] for t in times[bn]]
            med = statistics.median(ms)
            tf = flops / (med * 1e-3) / 1e12
            row[key] = {'ms': round(med, 4), 'ms_min': round(min(ms), 4), 'ms_max': round(max(ms), 4),
                        'tflops': round(tf, 1), 'frac': round(tf / PEAK_TFLOPS, 4)}
        row['speedup'] = round(row['bn64']['ms'] / row['default']['ms'], 3)
        print(json.dumps(row))


if __name__ == '__main__':
    main()
