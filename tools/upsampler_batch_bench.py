"""RealESRGANer timing on one GPU, per image: the host ``enhance`` chain (float32 conversion and colour swap on the host, the
tile loop at batch 1, fp32 download, uint8 conversion in numpy) against ``enhance_batch`` (uint8 tiles of all images
through batched RRDBNet forwards on the device).  RealESRGAN x2 (RRDBNet 23 blocks, seeded weights) with tile=400,
tile_pad=40, pre_pad=0, in fp32 and fp16; frames of 640x853 and 1080x1920 at batch 1 and 8, restored faces of 512x512 at
batch 1, 3 and 24.  The host chain takes host images and returns host images; enhance_batch takes and returns CUDA tensors,
as restore_images uses it.  Wall clock (ending in a device synchronise) for both, device events for enhance_batch.

    python tools/upsampler_batch_bench.py [--iters 3] [--cases frame640:1,frame640:8,frame1080:1,frame1080:8,face:1,face:3,face:24]
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import codeformer_b200 as cb                                   # noqa: E402
from codeformer_b200 import spec as S                           # noqa: E402
from tools.detection_bench import card                          # noqa: E402

SIZES = {'frame640': (640, 853), 'frame1080': (1080, 1920), 'face': (512, 512)}


def host_enhance(er, img):
    """``enhance`` of a uint8 BGR image through the generic chain (the parent's only path)."""
    import cv2
    x = cv2.cvtColor(img.astype(np.float32) / 255, cv2.COLOR_BGR2RGB)
    return (er._run(x) * 255.0).round().astype(np.uint8)


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


def events(fn, iters):
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=3)
    ap.add_argument('--cases', default='frame640:1,frame640:8,frame1080:1,frame1080:8,face:1,face:3,face:24')
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    dev = 'cuda:0'
    print(card(), '| RealESRGAN x2 (RRDBNet 23 blocks), tile=400 tile_pad=40 pre_pad=0')
    net = cb.RRDBNet(3, 3, scale=2, num_block=23)
    net.load_state_dict(S.random_state_dict(S.rrdbnet_spec(3, 3, 2, 64, 23, 32), 1))
    net = net.to(dev).eval()
    er = cb.RealESRGANer(scale=2, model=net, tile=400, tile_pad=40, pre_pad=0, device=dev)
    for precision in ('fp32', 'fp16'):
        net.set_precision(precision)
        for case in args.cases.split(','):
            kind, b = case.split(':')
            b = int(b)
            h, w = SIZES[kind]
            imgs = np.random.default_rng(b).integers(0, 256, (b, h, w, 3), dtype=np.uint8)
            x = torch.from_numpy(imgs).to(dev)
            out = er.enhance_batch(x)
            assert np.array_equal(out[0].cpu().numpy(), host_enhance(er, imgs[0])), 'enhance_batch differs from enhance'
            groups = er.tile_groups(b, h, w, tile_bytes=lambda n, th, tw: cb._lib.load().cfb_rrdb_workspace_bytes(
                net._handle(), n, th, tw))
            host_ms = wall(lambda: [host_enhance(er, im) for im in imgs], args.iters)
            batch_ms = wall(lambda: er.enhance_batch(x), args.iters)
            batch_ev = events(lambda: er.enhance_batch(x), args.iters)
            print(f'{precision} {kind} {h}x{w} batch {b}: host enhance {host_ms / b:.1f} ms/image, enhance_batch '
                  f'{batch_ms / b:.1f} ms/image wall, {batch_ev / b:.1f} ms/image device events '
                  f'({len(groups)} forwards for {sum(len(r) for _, _, r in groups)} tiles); {host_ms / batch_ms:.2f}x',
                  flush=True)


if __name__ == '__main__':
    main()
