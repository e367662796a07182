"""Timing of fidelity sweeps (one face at several w) on one GPU; seeded random weights, the committed faces and synthetic
frames, every output checked for byte equality in the same run.

Faces, in fp32 and fp16 precision (device events, warm-ups of every timed call, the three variants alternated, medians):
  (a) 1 face x K = 5 (the slider case), (b) 32 faces x K = 4:
      sweep      forward_u8_sweep(faces, ws)
      K calls    K forward_u8(faces, w=ws[k])
      per-face   one forward_u8 of the B*K repeated faces with per-face w

Whole images: 8 frames of 1080x1920 with 1 and 3 faces each (RetinaFace-ResNet50 runs in full; its candidates are fixed
faces, tools/wholeimage_bench.py), K = 4, ParseNet masks, with and without a device RealESRGANer background (RRDBNet x2, 23
blocks, tile 400): restore_images_sweep against K restore_images calls.  Host clock around synchronised calls, alternated
rounds, medians.

    python tools/fidelity_sweep_bench.py [--iters 5] [--rounds 2] [--skip-faces] [--skip-images]
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


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def wall_ms(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def faces_case(net, faces, ws, iters, label):
    B, K = faces.shape[0], len(ws)
    rep = faces.repeat_interleave(K, 0)
    wv = torch.tensor(ws * B, dtype=torch.float32, device=DEV)
    calls = {'sweep': lambda: net.forward_u8_sweep(faces, ws),
             'K calls': lambda: [net.forward_u8(faces, w=w) for w in ws],
             'per-face': lambda: net.forward_u8(rep, w=wv)}
    got = calls['sweep']()
    singles = calls['K calls']()
    pf = calls['per-face']().view(B, K, 512, 512, 3)
    same = torch.equal(got, pf) and all(torch.equal(got[:, k], singles[k]) for k in range(K))
    for fn in calls.values():                                  # warm-ups (graph captures included)
        fn()
    t = {k: [] for k in calls}
    for _ in range(iters):
        for k, fn in calls.items():
            t[k].append(event_ms(fn))
    base = np.median(t['K calls'])
    for k, v in t.items():
        m = np.median(v)
        print(f'{label} {k:9s}: {m:9.2f} ms  {B * K * 1e3 / m:7.1f} restored faces/s  x{base / m:5.2f} vs K calls', flush=True)
    print(f'{label} outputs byte-equal (sweep vs K calls vs per-face call): {same}', flush=True)
    return same


def images_case(net, det, parser, frames, ws, bg, rounds, label):
    calls = {'sweep': lambda: cb.restore_images_sweep(frames, net, det, ws, parser=parser, bg_upsampler=bg, max_batch=32),
             'K calls': lambda: [cb.restore_images(frames, net, det, parser=parser, w=w, bg_upsampler=bg, max_batch=32)
                                 for w in ws]}
    got, ref = calls['sweep'](), calls['K calls']()
    same = all(np.array_equal(a, b) for k in range(len(ws)) for a, b in zip(got[k], ref[k]))
    t = {k: [] for k in calls}
    for _ in range(rounds):
        for k, fn in calls.items():
            t[k].append(wall_ms(fn))
    base = np.median(t['K calls'])
    for k, v in t.items():
        m = np.median(v)
        print(f'{label} {k:8s}: {m:9.1f} ms  {m / len(frames):7.1f} ms per frame (all K)  x{base / m:5.2f} vs K calls  '
              f'(rounds: ' + ', '.join(f'{x:.0f}' for x in v) + ')', flush=True)
    print(f'{label} outputs byte-equal: {same}', flush=True)
    return same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--skip-faces', action='store_true')
    ap.add_argument('--skip-images', action='store_true')
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    print(card(), flush=True)
    rng = np.random.default_rng(7)
    f = np.load(os.path.join(ROOT, 'tests', 'golden', 'faces.npz'))['faces'][..., ::-1]
    faces = torch.from_numpy(np.ascontiguousarray(np.stack([f[i % len(f)] for i in range(32)]))).to(DEV)
    net = cb.CodeFormer().to(DEV).eval()
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1))
    ok = True
    for precision in () if args.skip_faces else ('fp32', 'fp16'):
        net.set_precision(precision)
        ws5 = [float(x) for x in np.round(rng.uniform(0.1, 1.0, 5), 3)]
        ws4 = [float(x) for x in np.round(rng.uniform(0.1, 1.0, 4), 3)]
        ok &= faces_case(net, faces[:1], ws5, args.iters * 4, f'[{precision}] (a) 1 face  x K=5')
        ok &= faces_case(net, faces, ws4, args.iters, f'[{precision}] (b) 32 faces x K=4')
    net.set_precision('fp32')
    net._cfb_ws.clear()                 # the B*K = 128 workspace of (b): room for the background upsampler
    net._cfb_graphs.clear()
    torch.cuda.empty_cache()
    if not args.skip_images:
        from tools.wholeimage_bench import nets
        from oracle.pasteback_oracle import synthetic_background
        frames = [synthetic_background(1080, 1920, s) for s in range(8)]
        rrdb = cb.RRDBNet(3, 3, scale=2, num_block=23)
        rrdb.load_state_dict(S.random_state_dict(S.rrdbnet_spec(3, 3, 2, 64, 23, 32), 11))
        bg = cb.RealESRGANer(scale=2, model=rrdb, tile=400, tile_pad=40, pre_pad=0, device=DEV)
        ws = [0.3, 0.5, 0.7, 1.0]
        for k in (1, 3):
            _, det, parser = nets(k)
            for up, name in ((None, 'no bg'), (bg, 'device bg')):
                ok &= images_case(net, det, parser, frames, ws, up, args.rounds,
                                  f'[fp32] 8 frames 1080x1920, {k} face(s), K=4, {name:9s}')
    print('all outputs byte-equal:', bool(ok), flush=True)
    if not ok:
        sys.exit(1)


if __name__ == '__main__':
    main()
