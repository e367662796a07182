"""Per-image time of whole-image paste-back on the GPU (codeformer_b200.pasteback.paste_faces, use_parse, upscale 2).

A synthetic 1080x1440 BGR image with 3 and with 8 faces (seeded similarity transforms, ~300 px faces), restored faces
[N,512,512,3] already on the device.  Median per-image milliseconds from CUDA events after warm-up, split into
ParseNet (resize + img2tensor + the network + argmax) and the paste kernels (masks, blurs, composites, one read-back).
``--cpu`` also times the numpy oracle (oracle/pasteback_oracle.py) on the same inputs, for the ratio.  Prints the card
and its power limit beside the numbers.

    python tools/pasteback_bench.py [--iters 20] [--cpu] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def similarity(scale, deg, cx, cy):
    a = np.deg2rad(deg)
    c, s = np.cos(a) * scale, np.sin(a) * scale
    return np.array([[c, -s, cx - (c * 256 - s * 256)], [s, c, cy - (s * 256 + c * 256)]])


def inputs(n, seed=0, h=1080, w=1440, upscale=2):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    faces = rng.integers(0, 256, (n, 512, 512, 3), dtype=np.uint8)
    inv = []
    for i in range(n):
        T = similarity(rng.uniform(0.5, 0.65), rng.uniform(-20, 20), 200 + (i % 4) * 340, 250 + (i // 4) * 520)
        inv.append(T * upscale)      # get_inverse_affine: the inverse of the crop affine (image -> face), times upscale
    return img, faces, inv


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except Exception:        # noqa: BLE001
        return torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--cpu', action='store_true')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('pasteback_bench needs a CUDA device')
    from codeformer_b200 import init_parsing_model
    from codeformer_b200 import pasteback as PB
    from codeformer_b200.parsing import parsenet_spec, random_parsenet_state_dict
    net = init_parsing_model(device='cpu')
    net.load_state_dict(random_parsenet_state_dict(parsenet_spec(512, 512, 32, 64, 19, 10, (32, 256)), 41), strict=False)
    net = net.cuda()
    res = {'card': card(), 'image': '1080x1440', 'upscale': 2, 'use_parse': True}
    for n in (3, 8):
        img, faces, inv = inputs(n)
        d_img, d_faces = torch.from_numpy(img).cuda(), torch.from_numpy(faces).cuda()
        adj = PB.adjust_inverse_affines([m.copy() for m in inv], 2, False)
        t_parse, t_paste, t_all = [], [], []
        for it in range(args.warmup + args.iters):
            e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            e[0].record()
            masks = PB.parse_masks(d_faces, net)
            e[1].record()
            PB._paste(d_img, d_faces, adj, 2, 512, masks, None)
            e[2].record()
            torch.cuda.synchronize()
            if it >= args.warmup:
                t_parse.append(e[0].elapsed_time(e[1]))
                t_paste.append(e[1].elapsed_time(e[2]))
                t_all.append(e[0].elapsed_time(e[2]))
        r = {'gpu_ms': float(np.median(t_all)), 'parsenet_ms': float(np.median(t_parse)), 'paste_ms': float(np.median(t_paste))}
        if args.cpu:
            from oracle import pasteback_oracle as O
            m = PB.parse_masks(d_faces, net).cpu().numpy()
            t0 = time.perf_counter()
            O.paste_faces(img, list(faces), [x.copy() for x in inv], 2, m)
            r['host_oracle_ms'] = (time.perf_counter() - t0) * 1e3
        res[f'faces_{n}'] = r
        print(n, 'faces', json.dumps(r), flush=True)
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
