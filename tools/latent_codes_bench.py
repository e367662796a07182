"""Timing of the latent-code path (VQAutoEncoder.latent_codes_u8 / generate_latent_gt) and of code_scores on one GPU.
Device events around warmed-up calls (medians of --iters), host wall clocks where the timed loop synchronises; the card, its
power limit and clocks printed first, in the same run.

  latent codes  ms per 512 x 512 face for the codes of a face and of its mirror (generate_latent_gt.py's 'orig' and 'hflip'):
                latent_codes_u8(hflip=True) at B = 32 and 64 (one encoder pass at 2B, uint8 in), against
                (a) the script's loop with the drop-ins: one face per call, vqgan.encoder + vqgan.quantize, indices to the host
                    (the fp32 input conversion is done on the device beforehand and not timed), and
                (b) VQAutoEncoder.forward at batch 2B on the fp32 inputs, which decodes and throws the decode away
  code scores   ms for 32 faces: the code_only pass from uint8 faces (cfb_codeformer_code_only_u8), the cfb_code_scores
                kernel alone, and code_scores() end to end (both, the layout copy and the status check's synchronise)

    python tools/latent_codes_bench.py [--iters 5]
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import codeformer_b200 as cb                                   # noqa: E402
from codeformer_b200 import _lib                               # noqa: E402
from codeformer_b200 import spec as S                          # noqa: E402
from tools.arcface_bench import event_ms, faces                # noqa: E402
from tools.detection_bench import card                         # noqa: E402


def fp32_chain(u8):
    """img2tensor(img / 255., bgr2rgb=True, float32=True) + normalize(0.5, 0.5) on the device (untimed set-up)."""
    x = (u8.double() / 255.).float()[..., [2, 1, 0]].permute(0, 3, 1, 2).contiguous()
    return (x - 0.5) / 0.5


def release(net):
    """Drop the module's cached workspaces: at B = 64 the encoder-only and the full forward's do not fit on one card together."""
    net._cfb_ws.clear()
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    print(card(), flush=True)
    vq = cb.VQAutoEncoder(512, 64, [1, 2, 2, 4, 4, 8], 'nearest', 2, [16], 1024)
    vq.load_state_dict(S.random_state_dict(S.vqae_spec(), 2), strict=True)
    vq = vq.cuda().eval()
    for B in (32, 64):
        u8 = faces(B)
        x2 = torch.cat([fp32_chain(u8), fp32_chain(u8.flip(2))])            # orig then hflip, as 2B fp32 faces
        fused = event_ms(lambda: vq.latent_codes_u8(u8, hflip=True), args.iters)
        release(vq)

        def script_loop():
            for i in range(2 * B):
                z = vq.encoder(x2[i:i + 1])
                _, _, log = vq.quantize(z)
                log['min_encoding_indices'].view(16, 16).cpu()
        script_loop()
        torch.cuda.synchronize()
        ts = []
        for _ in range(max(1, args.iters // 2)):
            t0 = time.perf_counter()
            script_loop()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        loop = float(np.median(ts))
        full = event_ms(lambda: vq(x2, return_min_encodings=False), args.iters)
        release(vq)
        print(f'latent codes B={B} (+ mirror): latent_codes_u8 {fused / B:.3f} ms per face; script loop with the drop-ins '
              f'{loop / B:.3f} ms per face ({loop / fused:.1f}x); VQAutoEncoder.forward at {2 * B} {full / B:.3f} ms per face '
              f'({full / fused:.1f}x)', flush=True)
        del x2

    net = cb.CodeFormer()
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    net = net.cuda().eval()
    lib = _lib.load()
    B = 32
    u8 = faces(B)
    gt = vq.latent_codes_u8(u8)
    net._prepare(u8.device)
    ws = net._cfb_workspace(u8.device, B)
    logits = torch.empty((B, 256, 1024), device='cuda')
    lq = torch.empty((B, 256, 16, 16), device='cuda')
    top = torch.empty((B, 256), dtype=torch.int64, device='cuda')
    feat = torch.empty((B, 256, 256), device='cuda')
    out = torch.empty((B, 3), dtype=torch.float64, device='cuda')
    E = net.quantize.embedding.weight.detach().contiguous()

    def code_only():
        _lib.check(lib.cfb_codeformer_code_only_u8(net._net, _lib.ptr(u8), _lib.ptr(logits), _lib.ptr(lq), _lib.ptr(top), B,
                                                   _lib.ptr(ws), ws.numel(), _lib.stream()), 'cfb_codeformer_code_only_u8')
    code_only()
    _lib.check(lib.cfb_nchw_to_nhwc(_lib.ptr(lq), _lib.ptr(feat), B, 256, 256, _lib.stream()), 'cfb_nchw_to_nhwc')

    def scores():
        _lib.check(lib.cfb_code_scores(_lib.ptr(logits), _lib.ptr(top), _lib.ptr(gt), _lib.ptr(feat), _lib.ptr(E), B, 256, 1024,
                                       256, _lib.ptr(out), _lib.stream()), 'cfb_code_scores')
    t_pass = event_ms(code_only, args.iters)
    t_kernel = event_ms(scores, args.iters * 4)
    t_total = event_ms(lambda: cb.code_scores(net, u8, gt), args.iters)
    print(f'code scores B={B}: code_only pass {t_pass:.3f} ms, cfb_code_scores kernel {t_kernel:.3f} ms '
          f'({100 * t_kernel / t_pass:.1f}% of the pass), code_scores() end to end {t_total:.3f} ms', flush=True)


if __name__ == '__main__':
    main()
