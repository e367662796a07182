"""Images/s and faces/s of ``restore_images`` (batched whole-image mode) against the per-image loop of the existing
drop-ins, on frame batches at 1080x1920 and 640x853 with 1 and 3 faces per frame, plus the stage shares of the batched
path (resize, detect, warp, CodeFormer, parse, paste).

Weights are seeded random (the numbers are about time, not quality).  The detector is RetinaFace-ResNet50 run in full;
only its candidate rows are replaced by k fixed, well separated faces per frame so that every frame holds exactly k faces.

--parser bisenet runs the paste-back's parse step with BiSeNet(19) (seeded weights, oracle/bisenet_oracle.py) instead of
ParseNet, in both paths.

    python tools/wholeimage_bench.py [--frames 8] [--reps 3] [--json out.json] [--parser parsenet|bisenet]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import codeformer_b200 as cb                      # noqa: E402
from codeformer_b200 import pasteback as PB       # noqa: E402
from codeformer_b200 import wholeimage as WI      # noqa: E402


class FixedFaces(cb.RetinaFace):
    """RetinaFace whose candidates are k fixed faces per image (the network still runs)."""
    k = 1

    def candidates(self, loc, conf, landms, h, w, conf_threshold=0.8):
        super().candidates(loc, conf, landms, h, w, conf_threshold)
        rows = []
        for j in range(self.k):
            s = min(h, w) / 4.0
            cx, cy = w * (j + 1) / (self.k + 1), h / 2.0
            lm = np.array(WI.FACE_TEMPLATE) / 512.0 * s + np.array([cx - s / 2, cy - s / 2])
            rows.append(np.concatenate([[cx - s / 2, cy - s / 2, cx + s / 2, cy + s / 2, 0.99], lm.reshape(-1)]))
        r = torch.tensor(np.array(rows, np.float32))
        return [r.to(loc.device) for _ in range(loc.shape[0])]


def nets(k, parser_name='parsenet'):
    from codeformer_b200 import spec as S
    from codeformer_b200.detection import random_retinaface_state_dict
    from codeformer_b200.parsing import parsenet_spec, random_parsenet_state_dict
    net = cb.ARCH_REGISTRY.get('CodeFormer')(dim_embd=512, codebook_size=1024, n_head=8, n_layers=9,
                                             connect_list=['32', '64', '128', '256']).cuda().eval()
    net.load_state_dict(S.random_state_dict(S.codeformer_spec(), 1), strict=True)
    det = FixedFaces().cuda()
    det.load_state_dict(random_retinaface_state_dict(1), strict=True)
    det.k = k
    parser = cb.init_parsing_model(parser_name, device='cpu')
    if parser_name == 'bisenet':
        from oracle.bisenet_oracle import random_bisenet_state_dict
        parser.load_state_dict(random_bisenet_state_dict(1), strict=True)
    else:
        parser.load_state_dict(random_parsenet_state_dict(parsenet_spec(512, 512, 32, 64, 19, 10, (32, 256)), 41), strict=False)
    return net, det.eval(), parser.cuda().eval()


def per_image_loop(imgs, net, det, parser, upscale=2):
    """The reference loop body per image with the existing drop-ins (detect_faces, align_warp_face, restore_faces,
    paste_faces_to_input_image); the detector's resize on the host (cv2), as the reference helper does it."""
    import cv2
    from types import SimpleNamespace
    out = []
    for img in imgs:
        helper = SimpleNamespace(upscale_factor=upscale, face_size=(512, 512), face_template=WI.FACE_TEMPLATE, pad_blur=False,
                                 all_landmarks_5=[], affine_matrices=[], cropped_faces=[], inverse_affine_matrices=[],
                                 use_parse=True, face_parse=parser, input_img=img)
        h, w = img.shape[:2]
        scale = 640 / min(h, w)
        dimg = cv2.resize(img, (int(w * scale), int(h * scale)), interpolation=cv2.INTER_AREA if scale < 1 else cv2.INTER_LINEAR)
        with torch.no_grad():
            b = det.detect_faces(dimg)
        helper.all_landmarks_5 = WI._landmarks(b, scale, h, w, False, 5)
        PB.align_warp_face(helper)
        with torch.no_grad():
            helper.restored_faces = net.restore_faces(helper.cropped_faces, w=0.5, adain=True)
        for a in helper.affine_matrices:
            inv = cv2.invertAffineTransform(a)
            inv *= upscale
            helper.inverse_affine_matrices.append(inv)
        out.append(PB.paste_faces_to_input_image(helper))
    return out


def stages(imgs, net, det, parser, upscale=2, max_batch=32):
    """The batched path stage by stage, each followed by a synchronisation: seconds per stage for the whole batch."""
    import cv2
    t = {}

    def mark(name, t0):
        torch.cuda.synchronize()
        t[name] = t.get(name, 0.0) + time.perf_counter() - t0
        return time.perf_counter()
    t0 = time.perf_counter()
    x = torch.from_numpy(np.stack(imgs)).cuda()
    h, w = x.shape[1:3]
    t0 = mark('upload', t0)
    scale = 640 / min(h, w)
    dh, dw = int(h * scale), int(w * scale)
    xd = PB.resize_area(x, (dw, dh)) if scale < 1 else PB.resize_linear(x, (dw, dh))
    t0 = mark('resize', t0)
    with torch.no_grad():
        dets = WI._detect(det, xd)
    lms = [WI._landmarks(d, scale, h, w, False, 5) for d in dets]
    aff, owner = [], []
    for k, lm in enumerate(lms):
        for L in lm:
            aff.append(cv2.estimateAffinePartial2D(L, WI.FACE_TEMPLATE, method=cv2.LMEDS)[0])
            owner.append(k)
    t0 = mark('detect', t0)
    crops = PB.warp_faces_multi(x, aff, owner)
    t0 = mark('warp', t0)
    with torch.no_grad():
        restored = torch.cat([net.forward_u8(crops[lo:lo + max_batch], w=0.5) for lo in range(0, crops.shape[0], max_batch)])
    t0 = mark('codeformer', t0)
    with torch.no_grad():
        masks = torch.cat([PB.parse_masks(restored[lo:lo + max_batch], parser) for lo in range(0, restored.shape[0], max_batch)])
    t0 = mark('parse', t0)
    invs = [cv2.invertAffineTransform(a) * upscale for a in aff]
    PB.adjust_inverse_affines(invs, upscale, False)
    canv = PB.resize_linear(x, (int(w * upscale), int(h * upscale)))
    out, _ = PB._paste_multi(canv, restored, invs, owner, upscale, masks)
    out.cpu()
    mark('paste', t0)
    return t


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    best = 1e30
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=8)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--json', default=None)
    ap.add_argument('--parser', choices=('parsenet', 'bisenet'), default='parsenet')
    a = ap.parse_args()
    from oracle.pasteback_oracle import synthetic_background
    rows = []
    print(f'parser: {a.parser}')
    print(f'{"frame":>10} {"faces":>5} {"loop img/s":>10} {"batch img/s":>11} {"loop face/s":>11} {"batch face/s":>12} '
          f'{"speed-up":>8}  stage shares (batched)', flush=True)
    for h, w in [(1080, 1920), (640, 853)]:
        imgs = [synthetic_background(h, w, s) for s in range(a.frames)]
        for k in (1, 3):
            net, det, parser = nets(k, a.parser)
            t_loop = timed(lambda: per_image_loop(imgs, net, det, parser), a.reps)
            t_batch = timed(lambda: cb.restore_images(imgs, net, det, parser=parser), a.reps)
            st = stages(imgs, net, det, parser)
            tot = sum(st.values())
            shares = {n: round(v / tot, 3) for n, v in st.items()}
            n = a.frames
            row = dict(parser=a.parser, frame=f'{h}x{w}', faces_per_frame=k, frames=n, loop_s=t_loop, batch_s=t_batch,
                       loop_img_s=n / t_loop, batch_img_s=n / t_batch, loop_face_s=n * k / t_loop,
                       batch_face_s=n * k / t_batch, speedup=t_loop / t_batch, stage_shares=shares)
            rows.append(row)
            print(f'{row["frame"]:>10} {k:>5} {row["loop_img_s"]:>10.2f} {row["batch_img_s"]:>11.2f} {row["loop_face_s"]:>11.2f} '
                  f'{row["batch_face_s"]:>12.2f} {row["speedup"]:>7.2f}x  '
                  + ' '.join(f'{n_}={v:.0%}' for n_, v in shares.items()), flush=True)
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
