"""Generate tests/golden/pasteback.npz from the UNMODIFIED reference (build container only).

TEST INFRASTRUCTURE.  Run:  PYTHONDONTWRITEBYTECODE=1 python oracle/gen_golden_pasteback.py
Needs /root/reference and cv2.  ``FaceRestoreHelper.align_warp_face`` / ``get_inverse_affine`` /
``paste_faces_to_input_image`` (facelib/utils/face_restoration_helper.py) run as written on an instance made with
``__new__`` (the constructor downloads detector weights); the imports the helper module needs only for detection and
downloads are stubbed.  ``face_parse`` is the reference ParseNet with the seeded parameters of parsenet.npz (seed 41).
The input is a composite of the committed faces.npz placed with known similarity transforms on a smooth seeded
background, with the template landmarks mapped by those transforms (no detector).

Cases
  P1  upscale 2, use_parse, background resized, 3 faces: 0 and 1 overlap (blend order matters), 2 is clipped by the border
  P2  upscale 1, use_parse False, a normal face and a tiny one (w_edge == 0)
  P3  upscale 2, use_parse, a given upsample_img and a face upsampler stub (np.repeat x2), so the faces are 1024 wide
The input image and P3's upsample_img are not stored: oracle.pasteback_oracle.synthetic_input / synthetic_upsample rebuild
them bit for bit (integer background, cv2-exact warps) from the stored placement matrices.  Stored per case: the uint8 result
as its difference to the background (mod 256), w_edge per face, the inverse affines as get_inverse_affine leaves them, the
parse masks (packed bits), the oracle's ambiguous pixels (pre-cast fraction < 1e-3 or > 1 - 1e-3, packed; no test needs them
any more: the oracle equals the reference everywhere) and seeded samples of the
oracle's pre-cast canvas (float32, at O.sample_index).  Crops: the SHA-256 of face 2 of P1 (clipped by the border) in the
three border modes.
"""
import hashlib
import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim                      # noqa: E402
from oracle import pasteback_oracle as O         # noqa: E402
from oracle.gen_golden import load_ref_parsenet  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden')
TEMPLATE = np.array([[192.98138, 239.94708], [318.90277, 240.1936], [256.63416, 314.01935],
                     [201.26117, 371.41043], [313.08905, 371.15118]])
H, W = 192, 256
# case -> (upscale, use_parse, faces.npz index, (scale, degrees, cx, cy)) per face
CASES = {
    'P1': (2, True, [(0, (0.20, 12.0, 85.0, 95.0)), (1, (0.19, -20.0, 140.0, 110.0)), (2, (0.17, 7.0, 240.0, 60.0))]),
    'P2': (1, False, [(3, (0.24, -8.0, 120.0, 100.0)), (0, (0.03, 15.0, 210.0, 160.0))]),
    'P3': (2, True, [(1, (0.20, 18.0, 80.0, 90.0)), (2, (0.18, -12.0, 175.0, 120.0))]),
}


def similarity(scale, deg, cx, cy):
    """face (512 x 512) -> image: rotate by deg about the face centre, scale, centre at (cx, cy)."""
    a = np.deg2rad(deg)
    c, s = np.cos(a) * scale, np.sin(a) * scale
    return np.array([[c, -s, cx - (c * 256 - s * 256)], [s, c, cy - (s * 256 + c * 256)]])


def compose(faces_bgr, placements, seed):
    """The input image (O.synthetic_input, which the tests rebuild from the stored matrices) and its landmarks; checks
    that cv2 composes the same image."""
    import cv2
    Ts = [(idx, similarity(*p)) for idx, p in placements]
    img = O.synthetic_input(faces_bgr, Ts, H, W, seed)
    ref = O.synthetic_background(H, W, seed)
    for idx, T in Ts:
        m = cv2.warpAffine(np.ones((512, 512), np.float32), T, (W, H)) > 0.5
        ref[m] = cv2.warpAffine(faces_bgr[idx], T, (W, H))[m]
    assert np.array_equal(img, ref)
    return img, [np.c_[TEMPLATE, np.ones(5)] @ T.T for _, T in Ts], np.stack([T for _, T in Ts])


def load_helper_class():
    """The UNMODIFIED FaceRestoreHelper; its detection / download imports are stubbed (never called here)."""
    ref_shim.load()
    sys.path.insert(0, ref_shim.REF_ROOT)
    stubs = {'facelib': None, 'facelib.detection': {'init_detection_model': None},
             'facelib.parsing': {'init_parsing_model': None}, 'basicsr.utils': None,
             'basicsr.utils.download_util': {'load_file_from_url': None}, 'basicsr.utils.misc': {'get_device': None}}
    for name, attrs in stubs.items():
        if name in sys.modules:
            continue
        m = types.ModuleType(name)
        if attrs is None:
            m.__path__ = [os.path.join(ref_shim.REF_ROOT, *name.split('.'))]
        else:
            m.__dict__.update(attrs)
        sys.modules[name] = m
    spec = importlib.util.spec_from_file_location('ref_face_restoration_helper', os.path.join(
        ref_shim.REF_ROOT, 'facelib', 'utils', 'face_restoration_helper.py'))
    mod = importlib.util.module_from_spec(spec)
    sys.dont_write_bytecode = True
    spec.loader.exec_module(mod)
    return mod.FaceRestoreHelper, mod


def make_helper(cls, img, lms, upscale, use_parse, parse_net):
    h = cls.__new__(cls)
    h.template_3points, h.upscale_factor, h.crop_ratio = False, upscale, (1, 1)
    h.face_size, h.det_model, h.face_template = (512, 512), 'retinaface_resnet50', TEMPLATE * 1.0
    h.save_ext, h.pad_blur, h.device, h.use_parse, h.face_parse, h.is_gray = 'png', False, torch.device('cpu'), use_parse, parse_net, False
    h.all_landmarks_5, h.det_faces, h.affine_matrices, h.inverse_affine_matrices = list(lms), [], [], []
    h.cropped_faces, h.restored_faces, h.pad_input_imgs = [], [], []
    h.input_img = img
    return h


class RepeatUpsampler:
    """Face upsampler stub (RealESRGANer.enhance signature): nearest x2 by np.repeat."""

    def enhance(self, img, outscale=2):
        return np.repeat(np.repeat(img, 2, axis=0), 2, axis=1), None


def parse_mask_ref(mod, net, face):
    """The reference's parse mask computation (face_restoration_helper.py:459-470), batch 1."""
    import cv2
    from torchvision.transforms.functional import normalize
    x = cv2.resize(face, (512, 512), interpolation=cv2.INTER_LINEAR)
    x = mod.img2tensor(x.astype('float32') / 255., bgr2rgb=True, float32=True)
    normalize(x, (0.5, 0.5, 0.5), (0.5, 0.5, 0.5), inplace=True)
    with torch.no_grad():
        out = net(x[None])[0].argmax(dim=1).squeeze().numpy()
    return O.MASK_COLORMAP[out]


def main():
    torch.set_grad_enabled(False)
    cls, mod = load_helper_class()
    from oracle.gen_golden import parsenet_inputs
    sd, _ = parsenet_inputs()
    net = load_ref_parsenet()(in_size=512, out_size=512, parsing_ch=19).eval()
    net.load_state_dict(sd, strict=True)
    faces_bgr = np.ascontiguousarray(np.load(os.path.join(OUT, 'faces.npz'))['faces'][..., ::-1])
    out = {}
    for ci, (case, (up, use_parse, placement)) in enumerate(CASES.items()):
        img, lms, Ts = compose(faces_bgr, placement, 3 + ci)
        helper = make_helper(cls, img, lms, up, use_parse, net)
        helper.align_warp_face()
        helper.get_inverse_affine()
        inv0 = np.stack([m.copy() for m in helper.inverse_affine_matrices])
        idx = [p[0] for p in placement]
        restored = [faces_bgr[i].copy() for i in idx]
        helper.restored_faces = [r.copy() for r in restored]
        upsampler = RepeatUpsampler() if case == 'P3' else None
        up_img = None
        if case == 'P3':
            up_img = O.synthetic_upsample(img, up)
        res = helper.paste_faces_to_input_image(upsample_img=None if up_img is None else up_img.copy(), face_upsampler=upsampler)
        faces_in = [upsampler.enhance(r, up)[0] for r in restored] if upsampler else restored
        masks = np.stack([parse_mask_ref(mod, net, f) for f in faces_in]) if use_parse else None
        canvas, info = O.paste_faces(img, restored, [m.copy() for m in inv0], up, masks, up_img,
                                     face_upsampler=(lambda f: upsampler.enhance(f, up)[0]) if upsampler else None, return_info=True)
        # the oracle restates cv2's blur and resize arithmetic, so the two are equal; the ambiguous band is still stored
        frac = canvas - np.floor(canvas)
        ambig = (frac < 1e-3) | (frac > 1 - 1e-3)
        diff = O.to_u8(canvas).astype(np.int16) - res
        assert not diff.any(), f'{case}: oracle != reference'
        bg = O.resize_linear_u8(img, (W * up, H * up)) if up_img is None else up_img
        out[f'{case}_input'] = np.array([H, W, 3 + ci])          # h, w, background seed
        out[f'{case}_T'] = Ts
        out[f'{case}_delta'] = res - bg                           # uint8 wrap-around; 0 wherever a face did not change it
        out[f'{case}_faces'] = np.array(idx)
        out[f'{case}_inv'] = inv0
        out[f'{case}_w_edge'] = np.array([d['w_edge'] for d in info])
        out[f'{case}_ambig'] = np.packbits(ambig)
        if masks is not None:
            out[f'{case}_parse'] = np.packbits(masks > 0)
        out[f'{case}_sample_val'] = canvas.reshape(-1)[O.sample_index(canvas.size)].astype(np.float32)
        print(case, 'w_edge', out[f'{case}_w_edge'], 'areas', [round(float(d['area']), 3) for d in info])
        if case == 'P1':
            for mode in ('constant', 'reflect101', 'reflect'):
                h2 = make_helper(cls, img, lms[2:3], up, use_parse, net)
                h2.align_warp_face(border_mode=mode)
                out[f'crop_{mode}_sha256'] = np.array(hashlib.sha256(np.ascontiguousarray(h2.cropped_faces[0]).tobytes()).hexdigest())
            out['crop_affine'] = h2.affine_matrices[0]
    np.savez_compressed(os.path.join(OUT, 'pasteback.npz'), **out)


if __name__ == '__main__':
    main()
