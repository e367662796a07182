"""Parse-mask timing on one GPU: 512x512 uint8 faces to 0/255 masks with ParseNet(512, 512, 19) (seeded weights, committed
faces), three paths at batch 8 and 32:
  (a) the unfused chain: cfb_u8_to_input -> ParseNet.forward (logits and out_img) -> face_parse_mask;
  (b) ParseNet.masks_u8 in fp32;
  (c) ParseNet.masks_u8 in fp16.
Device events, 3 warm-ups, median of --iters calls.  (a) and (b) must be byte-equal; the class-flip share of (c) against (b)
is reported.

--model bisenet compares the two parsers in one process, masks per second at each batch:
  ParseNet.masks_u8 in fp32 and fp16; BiSeNet(19).masks_u8 (seeded weights, oracle/bisenet_oracle.py); and the reference
  BiSeNet's computation on cuDNN -- oracle.bisenet_oracle.forward (the reference's ops, bit-identical to the reference class
  on the CPU) on CUDA tensors, with cudnn.allow_tf32 at its default (True) and False -- followed by face_parse_mask.  BiSeNet's
  masks_u8 must be byte-equal to cfb_u8_to_input + BiSeNet.forward + face_parse_mask.

    python tools/parse_masks_bench.py [--iters 20] [--batches 8,32] [--model parsenet|bisenet]
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import codeformer_b200 as cb                                   # noqa: E402
from codeformer_b200 import parsing as P                       # noqa: E402
from codeformer_b200 import pasteback as PB                    # noqa: E402
from tools.detection_bench import card                          # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')


def events(fn, iters, warmup=3):
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


def chain(net, faces):
    """(a): what parse_masks did for every parser before masks_u8 (a wrapper parser still takes it)."""
    return PB.parse_masks(faces, lambda x: net(x))


def bisenet_compare(parsenet, base, batches, iters, dev):
    from oracle import bisenet_oracle as BO
    sd = BO.random_bisenet_state_dict(1)
    bise = cb.BiSeNet(num_class=19)
    bise.load_state_dict(sd, strict=True)
    bise = bise.to(dev).eval()
    sd_dev = {k: v.to(dev) for k, v in sd.items()}

    def cudnn(faces, tf32):
        torch.backends.cudnn.allow_tf32 = tf32
        return PB.parse_masks(faces, lambda x: BO.forward(sd_dev, x))

    tf32_default = torch.backends.cudnn.allow_tf32
    for b in batches:
        faces = torch.from_numpy(np.ascontiguousarray(np.stack([np.roll(base[i % 4], 37 * (i // 4), axis=1)
                                                                for i in range(b)]))).to(dev)
        mask = bise.masks_u8(faces)[1]
        assert torch.equal(mask, PB.parse_masks(faces, lambda x: bise(x))), 'BiSeNet masks_u8 differs from the unfused chain'
        flip = float((cudnn(faces, False) != mask).float().mean()) * 100
        t = {}
        parsenet.set_precision('fp32')
        t['ParseNet masks_u8 fp32'] = events(lambda: parsenet.masks_u8(faces), iters)
        parsenet.set_precision('fp16')
        t['ParseNet masks_u8 fp16'] = events(lambda: parsenet.masks_u8(faces), iters)
        parsenet.set_precision('fp32')
        t['BiSeNet masks_u8'] = events(lambda: bise.masks_u8(faces), iters)
        t['BiSeNet reference on cuDNN (tf32 default)'] = events(lambda: cudnn(faces, tf32_default), iters)
        t['BiSeNet reference on cuDNN (allow_tf32=False)'] = events(lambda: cudnn(faces, False), iters)
        torch.backends.cudnn.allow_tf32 = tf32_default
        print(f'B={b}: ' + ' | '.join(f'{k} {v:.2f} ms = {b * 1e3 / v:.0f} masks/s' for k, v in t.items()) +
              f' | BiSeNet masks_u8 == unfused chain byte for byte; {flip:.3f} % of mask pixels differ from cuDNN fp32', flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--batches', default='8,32')
    ap.add_argument('--model', choices=('parsenet', 'bisenet'), default='parsenet')
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    dev = 'cuda:0'
    if args.model == 'bisenet':
        print(card(), '| ParseNet(512, 512, 19) and BiSeNet(19), seeded weights, 512x512 faces')
        net = P.ParseNet(in_size=512, out_size=512, parsing_ch=19)
        net.load_state_dict(P.random_parsenet_state_dict(P.parsenet_spec(512, 512, 32, 64, 19, 10, (32, 256)), 41), strict=True)
        base = np.load(os.path.join(GOLDEN, 'faces.npz'))['faces'][..., ::-1]
        bisenet_compare(net.to(dev).eval(), base, [int(v) for v in args.batches.split(',')], args.iters, dev)
        return
    print(card(), '| ParseNet(512, 512, 19), seeded weights, 512x512 faces')
    net = P.ParseNet(in_size=512, out_size=512, parsing_ch=19)
    net.load_state_dict(P.random_parsenet_state_dict(P.parsenet_spec(512, 512, 32, 64, 19, 10, (32, 256)), 41), strict=True)
    net = net.to(dev).eval()
    base = np.load(os.path.join(GOLDEN, 'faces.npz'))['faces'][..., ::-1]
    for b in (int(v) for v in args.batches.split(',')):
        faces = torch.from_numpy(np.ascontiguousarray(np.stack([np.roll(base[i % 4], 37 * (i // 4), axis=1)
                                                                for i in range(b)]))).to(dev)
        net.set_precision('fp32')
        ref = chain(net, faces)
        cls32, m32 = net.masks_u8(faces)
        assert torch.equal(ref, m32), '(a) and (b) differ'
        ta = events(lambda: chain(net, faces), args.iters)
        tb = events(lambda: net.masks_u8(faces), args.iters)
        net.set_precision('fp16')
        cls16, m16 = net.masks_u8(faces)
        torch.cuda.synchronize()
        cb.check_async_status()
        tc = events(lambda: net.masks_u8(faces), args.iters)
        flip = float((cls16 != cls32).float().mean()) * 100
        mflip = float((m16 != m32).float().mean()) * 100
        print(f'B={b}: (a) chain {ta:.2f} ms = {b * 1e3 / ta:.0f} faces/s | (b) masks_u8 fp32 {tb:.2f} ms = {b * 1e3 / tb:.0f} '
              f'faces/s ({ta / tb:.2f}x) | (c) masks_u8 fp16 {tc:.2f} ms = {b * 1e3 / tc:.0f} faces/s ({ta / tc:.2f}x of a, '
              f'{tb / tc:.2f}x of b) | (a) == (b) byte for byte | fp16: {flip:.3f} % of pixels change class, {mflip:.3f} % '
              'change mask value', flush=True)
    net.set_precision('fp32')


if __name__ == '__main__':
    main()
