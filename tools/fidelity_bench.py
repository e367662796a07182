"""Timing of per-face fidelity weights on one GPU (seeded weights, the committed faces; device results of forward_u8):
  (1) a slider sweep: 20 distinct w at B=1, one forward_u8 call each, scalar w against a per-face vector of one value.  Wall
      time per call including the eager warm-up and the CUDA-graph capture a new w costs the scalar path (the per-face path
      captures once), median of --rounds sweeps on a fresh module each;
  (2) B=32 faces with 4 distinct w: one per-face call against 4 scalar calls, one per group of 8 faces (what a service has to
      do without per-face weights).  Device events, the two alternated, median of --iters;
  (3) B=32 with one w: the per-face call (uniform vector) against the scalar call, to show what the per-image lookup in the
      SFT epilogue costs.  Device events, alternated, median of --iters.

    python tools/fidelity_bench.py [--iters 10] [--rounds 3]
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
from tools.detection_bench import card                         # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'


def fresh_net():
    net = cb.CodeFormer().to(DEV).eval()
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1))
    return net


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    f = np.load(os.path.join(ROOT, 'tests', 'golden', 'faces.npz'))['faces'][..., ::-1]
    faces = torch.from_numpy(np.ascontiguousarray(np.stack([f[i % len(f)] for i in range(32)]))).to(DEV)
    print(card(), flush=True)
    sweep = [round(0.05 * (i + 1), 2) for i in range(20)]

    # (1) slider sweep at B=1
    res = {'scalar': [], 'per_face': []}
    for _ in range(args.rounds):
        for kind in ('scalar', 'per_face'):
            net = fresh_net()
            net.forward_u8(faces[:1], w=0.5)                 # module load, weight upload: not part of the sweep
            torch.cuda.synchronize()
            t = time.perf_counter()
            for w in sweep:
                net.forward_u8(faces[:1], w=w if kind == 'scalar' else [w])
            torch.cuda.synchronize()
            res[kind].append((time.perf_counter() - t) * 1e3 / len(sweep))
            del net
    for kind, v in res.items():
        print(f'(1) slider sweep, 20 w at B=1, {kind:8s}: {np.median(v):8.2f} ms per call (rounds: '
              + ', '.join(f'{x:.2f}' for x in v) + ')', flush=True)

    net = fresh_net()
    # (2) 4 distinct w at B=32
    groups = [0.2, 0.4, 0.6, 0.8]
    wv = torch.tensor([groups[i % 4] for i in range(32)], device=DEV)
    idx = [torch.arange(g, 32, 4, device=DEV) for g in range(4)]
    sub = [faces[i].contiguous() for i in idx]
    one = lambda: net.forward_u8(faces, w=wv)                              # noqa: E731
    grouped = lambda: [net.forward_u8(s, w=w) for s, w in zip(sub, groups)]   # noqa: E731
    out = one()
    for k, (i, w) in enumerate(zip(idx, groups)):
        assert torch.equal(out[i], net.forward_u8(sub[k], w=w)), 'per-face result differs from the grouped scalar call'
    t = {'one per-face call': [], '4 grouped scalar calls': []}
    for _ in range(2):
        one(), grouped()
    for _ in range(args.iters):
        t['one per-face call'].append(event_ms(one))
        t['4 grouped scalar calls'].append(event_ms(grouped))
    for k, v in t.items():
        print(f'(2) B=32, 4 distinct w, {k:24s}: {np.median(v):8.2f} ms  ({32e3 / np.median(v):6.1f} faces/s)', flush=True)

    # (3) uniform w at B=32: per-face vector vs scalar
    wu = torch.full((32,), 0.5, device=DEV)
    assert torch.equal(net.forward_u8(faces, w=wu), net.forward_u8(faces, w=0.5))
    t = {'scalar w': [], 'per-face w': []}
    for _ in range(2):
        net.forward_u8(faces, w=0.5), net.forward_u8(faces, w=wu)
    for _ in range(args.iters):
        t['scalar w'].append(event_ms(lambda: net.forward_u8(faces, w=0.5)))
        t['per-face w'].append(event_ms(lambda: net.forward_u8(faces, w=wu)))
    for k, v in t.items():
        print(f'(3) B=32, one w, {k:10s}: {np.median(v):8.2f} ms  ({32e3 / np.median(v):6.1f} faces/s)', flush=True)


if __name__ == '__main__':
    main()
