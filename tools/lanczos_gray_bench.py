"""Times of the device INTER_LANCZOS4 resize, the gray colour transfer and restore_images on gray frames.

  * ``resize_lanczos4`` of 2160x3840 frames (the x2plus output of a 1080p frame) to x0.5, x1.5 and x2, batch 1 and 8, against
    ``cv2.resize(..., INTER_LANCZOS4)`` on the host (cv2's own thread count), with the bytes the kernel reads and writes over
    its time;
  * ``gray_adain_faces`` for 32 faces of 512x512;
  * ``restore_images(only_center_face=True)`` on 8 gray 1080p frames, one face per frame (seeded RetinaFace / CodeFormer /
    ParseNet weights on synthetic frames: without ``only_center_face`` those weights report about 200 boxes per frame),
    without an upsampler and with ``upscale=4`` through a seeded x2 RRDBNet (23 blocks, 400-pixel tiles).

Median milliseconds from CUDA events after warm-up (a host clock around a synchronise for restore_images, which reads its
result back).  Prints the card, its power limit and maximum SM clock beside the numbers.  Reads nothing outside the repository.

    python tools/lanczos_gray_bench.py [--iters 20] [--parts resize,adain,restore] [--out results.json]
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


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except Exception:        # noqa: BLE001
        return torch.cuda.get_device_name()


def event_ms(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def wall_ms(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--parts', default='resize,adain,restore')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('lanczos_gray_bench needs a CUDA device')
    import cv2
    import codeformer_b200 as cb
    from codeformer_b200 import spec as S
    res = {'card (name, power limit, max SM clock)': card(), 'cv2_threads': cv2.getNumThreads()}
    parts = args.parts.split(',')
    rng = np.random.default_rng(0)
    h, w = 2160, 3840
    if 'resize' in parts:
        frames = rng.integers(0, 256, (8, h, w, 3), dtype=np.uint8)
        d_frames = torch.from_numpy(frames).cuda()
    for name, f in (('x0.5', 0.5), ('x1.5', 1.5), ('x2', 2.0)) if 'resize' in parts else ():
        size = (int(w * f), int(h * f))
        t0 = time.perf_counter()
        for _ in range(3):
            ref = cv2.resize(frames[0], size, interpolation=cv2.INTER_LANCZOS4)
        host = (time.perf_counter() - t0) / 3 * 1e3
        assert np.array_equal(cb.resize_lanczos4(d_frames[0], size).cpu().numpy(), ref), 'resize_lanczos4 differs from cv2'
        r = {'host_cv2_ms_per_frame': host}
        for n in (1, 8):
            ms = event_ms(lambda: cb.resize_lanczos4(d_frames[:n], size), args.warmup, args.iters)
            moved = n * 3 * (h * w + size[0] * size[1])
            r[f'batch_{n}'] = {'gpu_ms': ms, 'ms_per_frame': ms / n, 'GB_per_s_read_plus_written': moved / ms / 1e6}
        res[f'resize_lanczos4_2160x3840_{name}'] = r
        print(name, json.dumps(r), flush=True)
    if 'adain' in parts:
        faces = torch.from_numpy(rng.integers(0, 256, (2, 32, 512, 512, 3), dtype=np.uint8)).cuda()
        res['gray_adain_faces_32x512x512'] = {'gpu_ms': event_ms(lambda: cb.gray_adain_faces(faces[0], faces[1]), args.warmup, args.iters)}
        print('gray_adain_faces', json.dumps(res['gray_adain_faces_32x512x512']), flush=True)
    if 'restore' in parts:
        from codeformer_b200.detection import random_retinaface_state_dict
        from codeformer_b200.parsing import parsenet_spec, random_parsenet_state_dict
        from oracle import pasteback_oracle as O
        net = cb.ARCH_REGISTRY.get('CodeFormer')(dim_embd=512, codebook_size=1024, n_head=8, n_layers=9,
                                                 connect_list=['32', '64', '128', '256']).cuda()
        net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
        det = cb.RetinaFace().cuda()
        det.load_state_dict(random_retinaface_state_dict(1, class_gain=8.0, class_bias=2.0), strict=True)
        parser = cb.init_parsing_model(device='cpu')
        parser.load_state_dict(random_parsenet_state_dict(parsenet_spec(512, 512, 32, 64, 19, 10, (32, 256)), 41), strict=False)
        net, det, parser = net.eval(), det.eval(), parser.cuda().eval()
        rrdb = cb.RRDBNet(3, 3, scale=2, num_block=23)
        rrdb.load_state_dict(S.random_state_dict(S.rrdbnet_spec(3, 3, 2, 64, 23, 32), 11))
        up = cb.RealESRGANer(scale=2, model=rrdb, tile=400, tile_pad=40, pre_pad=0, device='cuda')
        gray = [cv2.cvtColor(cv2.cvtColor(O.synthetic_background(1080, 1920, s), cv2.COLOR_BGR2GRAY), cv2.COLOR_GRAY2BGR)
                for s in range(8)]
        print('restore_images: networks ready', flush=True)
        t0 = time.perf_counter()
        _, crops, _ = cb.restore_images(gray, net, det, parser=parser, only_center_face=True, return_faces=True)
        r = {'faces': int(sum(c.shape[0] for c in crops))}
        print('restore_images: first call', json.dumps(r), f'{time.perf_counter() - t0:.1f} s', flush=True)
        it = max(2, args.iters // 5)
        r['upscale_2_no_upsampler_ms'] = wall_ms(lambda: cb.restore_images(gray, net, det, parser=parser, only_center_face=True), 0, it)
        print('restore_images', json.dumps(r), flush=True)
        r['upscale_4_x2_upsampler_ms'] = wall_ms(lambda: cb.restore_images(gray, net, det, parser=parser, only_center_face=True, upscale=4, bg_upsampler=up), 1, it)
        res['restore_images_8_gray_1080p'] = r
        print('restore_images', json.dumps(r), flush=True)
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
