"""GPU time per kernel of one warm batch-32 CodeFormer.forward(w=0.5, adain=True), from torch.profiler (CUDA activities).

The model and inputs are those of bench.py (random-init weights of seed 1, a synthetic clamped-normal batch).  Three untraced
forwards warm every shape first; the traced forward runs alone and is synchronised before the profiler stops.  Kernels are
grouped by their full name, template arguments included, so the tile kinds of conv_tc_kernel<BN, CPG, HALO, XF, GEN, K1, CM>
appear as separate rows.  The card name and power limit are read in the same run.

    python tools/step_kernel_shares.py [--batch 32] [--top 30]
"""
import argparse
import collections
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--top', type=int, default=30, help='rows printed (the total covers every kernel)')
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import codeformer_b200 as cb
    from codeformer_b200 import spec as S
    if not torch.cuda.is_available():
        raise SystemExit('step_kernel_shares: no CUDA device')
    torch.set_grad_enabled(False)
    net = cb.CodeFormer(dim_embd=512, codebook_size=1024, n_head=8, n_layers=9,
                        connect_list=['32', '64', '128', '256']).cuda().eval()
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    g = torch.Generator().manual_seed(100)
    x = torch.randn(args.batch, 3, 512, 512, generator=g).clamp_(-1, 1).cuda()
    for _ in range(3):
        net(x, w=0.5, adain=True)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        net(x, w=0.5, adain=True)
        torch.cuda.synchronize()
    per = collections.defaultdict(lambda: [0, 0.0])
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            per[ev.name][0] += 1
            per[ev.name][1] += ev.time_range.elapsed_us() / 1e3       # us -> ms
    total = sum(v[1] for v in per.values())
    print(f'gpu: {gpu_info()}  batch {args.batch}  kernel time {total:.2f} ms ({len(per)} kernel names)')
    print(f'{"ms":>9} {"share":>7} {"calls":>6}  kernel')
    for name, (calls, ms) in sorted(per.items(), key=lambda kv: -kv[1][1])[:args.top]:
        print(f'{ms:9.3f} {100 * ms / total:6.2f}% {calls:6d}  {name[:160]}')


if __name__ == '__main__':
    main()
