"""Timing of the face-only device paths on one GPU (seeded weights, committed faces and whole images):
  (1) CodeFormer.forward_u8 with the inpainting blend fused into the last conv against the plain forward_u8, B=32, on the
      inpainting configuration (codebook 512, connections 32/64/128, w=1, adain=False).  Device events, the two alternated,
      median of --iters calls each;
  (2) restore_aligned on 64 crops of 256x256 (half of them gray) against the per-crop loop of inference_codeformer.py
      --has_aligned with this package's drop-ins (host cv2.resize and is_gray, restore_faces of one face, add_restored_face).
      Wall time to the last result on the host, median of --rounds; results must be equal;
  (3) the gray test of 8 frames of 1080x1920: one cfb_is_gray_u8 launch and one read-back against the torch reductions it
      replaced (six reductions and six host synchronisations per frame).  Wall time, median of --iters.

    python tools/aligned_bench.py [--iters 10] [--rounds 3]
"""
import argparse
import os
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import codeformer_b200 as cb                                   # noqa: E402
from codeformer_b200 import spec as S                          # noqa: E402
from codeformer_b200.wholeimage import _device_is_gray, is_gray   # noqa: E402
from tools.detection_bench import card                         # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
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
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def torch_is_gray(img, threshold=10):
    """The per-image torch reductions restore_images used before cfb_is_gray_u8 (same decision)."""
    x = img.to(torch.int64)
    n = x.shape[0] * x.shape[1]
    total = 0.0
    for a, b in ((0, 1), (1, 2), (2, 0)):
        d = x[:, :, a] - x[:, :, b]
        s, s2 = int(d.sum()), int((d * d).sum())
        total += (n * s2 - s * s) / (n * n)
    return bool(total / 3.0 <= threshold)


def net_of(seed, **kw):
    net = cb.CodeFormer(**{k: (list(v) if k == 'connect_list' else v) for k, v in kw.items()}).to(DEV).eval()
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(**kw), seed))
    return net


def bench_inpaint(iters):
    net = net_of(4, codebook_size=512, connect_list=('32', '64', '128'))
    base = np.load(os.path.join(GOLDEN, 'faces.npz'))['faces'][..., ::-1]
    faces = np.stack([np.roll(base[i % 4], 37 * (i // 4), axis=1) for i in range(32)])
    faces[:, 150:260, 120:400] = 255                     # the white holes the inpainting model fills
    d = torch.from_numpy(np.ascontiguousarray(faces)).to(DEV)
    plain = lambda: net.forward_u8(d, w=1, adain=False)              # noqa: E731
    inp = lambda: net.forward_u8(d, w=1, adain=False, inpaint=True)  # noqa: E731
    for _ in range(3):
        plain(), inp()
    tp, ti = [], []
    for _ in range(iters):
        tp.append(event_ms(plain))
        ti.append(event_ms(inp))
    torch.cuda.synchronize()
    cb.check_async_status()
    sp, si = f'{min(tp):.2f}-{max(tp):.2f}', f'{min(ti):.2f}-{max(ti):.2f}'
    tp, ti = float(np.median(tp)), float(np.median(ti))
    print(f'(1) B=32 inpainting config: forward_u8 {tp:.2f} ms = {32e3 / tp:.1f} faces/s (range {sp} ms) | '
          f'forward_u8(inpaint=True) {ti:.2f} ms = {32e3 / ti:.1f} faces/s (range {si} ms) | ratio {ti / tp:.4f}', flush=True)


def aligned_crops(n):
    import cv2
    imgs = [cv2.imread(os.path.join(GOLDEN, 'whole_imgs', f'{k}.jpg'), cv2.IMREAD_COLOR) for k in ('00', '01', '03', '04', '05')]
    out = []
    for i in range(n):
        img = np.roll(imgs[i % len(imgs)], 13 * i, axis=1)
        crop = cv2.resize(img, (256, 256), interpolation=cv2.INTER_AREA)
        if i % 2:
            crop = cv2.cvtColor(cv2.cvtColor(crop, cv2.COLOR_BGR2GRAY), cv2.COLOR_GRAY2BGR)
        out.append(np.ascontiguousarray(crop))
    return out


def per_face_loop(crops, net):
    import cv2
    res = []
    for img in crops:
        img = cv2.resize(img, (512, 512), interpolation=cv2.INTER_LINEAR)
        helper = SimpleNamespace(is_gray=is_gray(img, threshold=10), restored_faces=[])
        restored = net.restore_faces([img], w=0.5, adain=True)[0]
        cb.add_restored_face(helper, restored, img)
        res.append(helper.restored_faces[0])
    return res


def bench_aligned(rounds):
    net = net_of(1)
    crops = aligned_crops(64)
    per_face_loop(crops[:2], net)
    cb.restore_aligned(crops, net)
    tl, ta = [], []
    for _ in range(rounds):
        t, ref = wall_ms(lambda: per_face_loop(crops, net))
        tl.append(t)
        t, got = wall_ms(lambda: cb.restore_aligned(crops, net, max_batch=32))
        ta.append(t)
    same = all(a.dtype == b.dtype and np.array_equal(a, b) for a, b in zip(got, ref))
    assert same, 'restore_aligned differs from the per-crop loop'
    tl, ta = float(np.median(tl)), float(np.median(ta))
    print(f'(2) 64 crops of 256x256, 32 gray: per-crop loop {tl:.0f} ms = {64e3 / tl:.1f} faces/s | restore_aligned '
          f'(max_batch 32) {ta:.0f} ms = {64e3 / ta:.1f} faces/s | {tl / ta:.2f}x | equal per crop', flush=True)


def bench_gray(iters):
    rng = np.random.default_rng(3)
    frames = torch.from_numpy(rng.integers(0, 256, (8, 1080, 1920, 3), dtype=np.uint8)).to(DEV)
    frames[1::2] = frames[1::2, :, :, :1]
    old = lambda: [torch_is_gray(f) for f in frames]       # noqa: E731
    new = lambda: _device_is_gray(frames)                  # noqa: E731
    assert old() == new() == [False, True] * 4
    to, tn = [], []
    for _ in range(iters):
        to.append(wall_ms(old)[0])
        tn.append(wall_ms(new)[0])
    to, tn = float(np.median(to)), float(np.median(tn))
    print(f'(3) gray test of 8 frames 1080x1920: torch reductions {to:.2f} ms | cfb_is_gray_u8 {tn:.3f} ms | {to / tn:.1f}x',
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    print(card(), flush=True)
    bench_inpaint(args.iters)
    bench_aligned(args.rounds)
    bench_gray(args.iters)


if __name__ == '__main__':
    main()
