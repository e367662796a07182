"""RealESRGANer timing for 16-bit and float images on one GPU: ``enhance_batch`` (the float32 conversion and the per-image
max_range fused into RRDBNet's first and last convs, tiles of many images through one forward, integer results written on
the device) against ``_enhance_host`` (conversion on the host, the tile loop at batch 1, fp32 download, rounding in numpy).
RealESRGAN x2 (RRDBNet 23 blocks, seeded weights) with tile=400, tile_pad=40, pre_pad=0, fp32:

  * frame16: 1080x1920 uint16 frames (values over the full 16-bit range), batch 1 and 8;
  * face64: 32 float64 faces of 512x512 (gray faces as ``add_restored_face`` leaves them, below 256), ``enhance_batch`` in
    batches of 1 and 8 against ``_enhance_host`` on each face;
  * restore: ``restore_images(only_center_face=True)`` on 8 dark gray 1080p frames with the x2 face upsampler, the parent's
    route (``enhance`` on the host per gray face, here ``_enhance_host`` behind an object that is not a RealESRGANer) against
    the chunk's gray faces in one ``enhance_batch``.  Seeded RetinaFace / CodeFormer / ParseNet weights on synthetic frames.

Host times are wall clock; device times are CUDA events around calls that take and return CUDA tensors, both medians.  Every
case first checks the bytes against ``_enhance_host``.  Prints the card, its power limit and maximum SM clock beside the numbers.

    python tools/upsampler_wide_bench.py [--iters 3] [--parts frame16,face64,restore] [--out results.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.lanczos_gray_bench import card, event_ms, wall_ms          # noqa: E402


class HostUpsampler:
    """The parent's route for gray faces: ``enhance`` on the host, one face per call."""

    def __init__(self, er):
        self.er = er

    def enhance(self, img, outscale=None):
        return self.er._enhance_host(img, outscale)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--parts', default='frame16,face64,restore')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('upsampler_wide_bench needs a CUDA device')
    import cv2
    import codeformer_b200 as cb
    from codeformer_b200 import spec as S
    torch.set_grad_enabled(False)
    dev = 'cuda'
    parts = args.parts.split(',')
    res = {'card (name, power limit, max SM clock)': card(), 'model': 'RealESRGAN x2 (RRDBNet 23 blocks), tile=400 tile_pad=40 pre_pad=0, fp32'}
    print(json.dumps(res), flush=True)
    rrdb = cb.RRDBNet(3, 3, scale=2, num_block=23)
    rrdb.load_state_dict(S.random_state_dict(S.rrdbnet_spec(3, 3, 2, 64, 23, 32), 11))
    er = cb.RealESRGANer(scale=2, model=rrdb, tile=400, tile_pad=40, pre_pad=0, device=dev)
    rng = np.random.default_rng(0)

    def compare(name, imgs, batches):
        d = torch.from_numpy(imgs).to(dev)
        for i in (0, len(imgs) - 1):
            ref = er._enhance_host(imgs[i])[0]
            got = er.enhance_batch(d[i:i + 1])[0].cpu().numpy()
            assert got.dtype == ref.dtype and np.array_equal(got, ref), f'{name}: enhance_batch differs from _enhance_host'
        n = len(imgs)
        r = {'dtype': str(imgs.dtype), 'images': n,
             'host_ms_per_image': wall_ms(lambda: [er._enhance_host(im) for im in imgs], args.warmup, args.iters) / n}
        for b in batches:
            def run():
                for lo in range(0, n, b):
                    er.enhance_batch(d[lo:lo + b])
            ms = event_ms(run, args.warmup, args.iters)
            r[f'batch_{b}_device_ms_per_image'] = ms / n
            r[f'batch_{b}_speedup'] = r['host_ms_per_image'] / (ms / n)
        res[name] = r
        print(name, json.dumps(r), flush=True)

    if 'frame16' in parts:
        frames = rng.integers(0, 65536, (8, 1080, 1920, 3)).astype(np.uint16)
        compare('frame16_1080x1920', frames[:1], [1])
        compare('frame16_1080x1920_x8', frames, [8])
    if 'face64' in parts:
        faces = np.clip(rng.normal(120.0, 40.0, (32, 512, 512, 3)), -5.0, 250.0)          # float64, below 256
        compare('face64_512x512_x32', faces, [1, 8])
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
        gray = [(cv2.cvtColor(cv2.cvtColor(O.synthetic_background(1080, 1920, s), cv2.COLOR_BGR2GRAY), cv2.COLOR_GRAY2BGR)
                 * 0.5).astype(np.uint8) for s in range(8)]
        host = HostUpsampler(er)

        def run(up):
            return cb.restore_images(gray, net, det, parser=parser, only_center_face=True, face_upsampler=up, return_faces=True)
        before, crops, _ = run(host)
        after = run(er)[0]
        assert all(np.array_equal(a, b) for a, b in zip(before, after)), 'restore_images: device faces differ from host faces'
        r = {'frames': len(gray), 'faces': int(sum(c.shape[0] for c in crops)),
             'before_host_enhance_per_face_ms': wall_ms(lambda: run(host), 0, args.iters),
             'after_enhance_batch_ms': wall_ms(lambda: run(er), 0, args.iters)}
        r['speedup'] = r['before_host_enhance_per_face_ms'] / r['after_enhance_batch_ms']
        res['restore_images_8_dark_gray_1080p_face_upsampler_x2'] = r
        print('restore', json.dumps(r), flush=True)
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
