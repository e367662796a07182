"""Face detector timing on one GPU: detect_faces per image (host uint8 in, numpy out), the forward alone (CUDA events),
and the oracle's torch module (cuDNN) on the same card as a comparison point.  --model picks RetinaFace-ResNet50 or
YOLOv5l-face (whose forward runs on the letterboxed canvas, 672x864 for a 640x853 image).  --profile prints the kernel
shares of one forward under torch.profiler instead (run it separately: tracing slows the host).

    python tools/detection_bench.py [--model retinaface_resnet50|yolov5l] [--sizes 640x853,1080x1440] [--iters 20] [--profile]
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import codeformer_b200 as cb                                   # noqa: E402
from codeformer_b200 import detection as D                      # noqa: E402
from codeformer_b200 import yolov5face as Y                     # noqa: E402
from oracle import retinaface_oracle as RO                      # noqa: E402
from oracle import yolov5face_oracle as YO                      # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                        # noqa: BLE001
        pl = f'unknown ({e})'
    return f'{name}, power limit / max SM clock: {pl}'


def timed(fn, iters, warmup=3):
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='640x853,1080x1440')
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--profile', action='store_true')
    ap.add_argument('--model', default='retinaface_resnet50', choices=['retinaface_resnet50', 'yolov5l'])
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    dev = 'cuda:0'
    print(card(), '|', args.model)
    if args.model == 'yolov5l':
        sd = Y.random_yolov5l_state_dict(1)
        net = cb.YOLOv5lFace().to(dev)
        det = cb.YoloDetector('yolov5l.yaml', device=dev)
        det.detector = net
        oracle_forward = YO.forward
    else:
        sd = D.random_retinaface_state_dict(1)
        net = det = cb.RetinaFace().to(dev)
        oracle_forward = RO.forward
    net.load_state_dict(sd, strict=True)
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    for s in args.sizes.split(','):
        h, w = (int(v) for v in s.split('x'))
        img = np.random.default_rng(0).integers(0, 256, (h, w, 3), dtype=np.uint8)
        x = (YO.preprocess([img]) if args.model == 'yolov5l' else RO.input_from_u8(img)).to(dev)
        if args.profile:
            net(x)
            torch.cuda.synchronize()
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                net(x)
                torch.cuda.synchronize()
            print(f'--- {h}x{w} (input {x.shape[2]}x{x.shape[3]}): kernel shares of one forward')
            print(prof.key_averages().table(sort_by='cuda_time_total', row_limit=15))
            continue
        faces = det.detect_faces(img)
        det_ms = timed(lambda: det.detect_faces(img), args.iters)
        fwd_ms = timed(lambda: net(x), args.iters)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        ref_fp32 = timed(lambda: oracle_forward(sd_dev, x), args.iters)
        torch.backends.cudnn.allow_tf32 = True
        ref_tf32 = timed(lambda: oracle_forward(sd_dev, x), args.iters)
        print(f'{h}x{w} (network input {x.shape[2]}x{x.shape[3]}): detect_faces {det_ms:.2f} ms/image (host uint8 in, numpy out), forward {fwd_ms:.2f} ms; '
              f'oracle torch module on cuDNN: {ref_fp32:.2f} ms (allow_tf32=False), {ref_tf32:.2f} ms (default, TF32 convs); '
              f'{0 if faces is None else len(faces)} faces of the random weights')


if __name__ == '__main__':
    main()
