"""Seeded whole-image scenes for the paste-back sweep (tests/test_gpu_paste_sweep.py and its CPU twin
tests/test_paste_sweep_cpu.py), and the reference's paste written out with cv2 (``cv2_paste``).

A scene is the input of paste_faces_to_input_image: an input image, restored faces with the inverse affines
``get_inverse_affine`` leaves (face -> output canvas), the upscale, optional parse masks (0/255 MASK_COLORMAP images) and an
optional upsample_img.  Together the scenes cover w_edge 0 (the 3x3 second erosion) to 50, any rotation, faces partly and
wholly off the canvas and overlapping, upscale 1 / 1.5 / 2 / 3 / 4, a face upsampler (1024-wide faces), an upsample_img at
the output size and at another size, uint8 and float64 faces, and parse masks with solid regions and holes."""
import os
from types import SimpleNamespace

import numpy as np

from oracle import gray_oracle as G
from oracle import pasteback_oracle as O
from oracle.resize_lanczos4_oracle import resize_lanczos4_u8

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
UPSCALES = (1, 1.5, 2, 3, 4)
# w_edge of the first face of scene i, within 1: int(sqrt(area)) // 20 for a face about `side` canvas pixels wide
W_EDGES = (0, 1, 2, 3, 4, 5, 6, 7, 9, 12, 14, 16, 19, 21, 24, 27, 29, 33, 38, 44, 50, 0, 2, 8, 11, 17, 25, 30, 35, 41)
N_SCENES = len(W_EDGES)


def _faces():
    return np.ascontiguousarray(np.load(os.path.join(GOLD, 'faces.npz'))['faces'][..., ::-1])


def parse_mask(rng):
    """A 512 x 512 0/255 parse mask: a solid ellipse (the face) with solid holes (eyes, mouth) and a blocky noisy margin."""
    y, x = np.mgrid[0:512, 0:512].astype(np.float64)
    cy, cx = rng.uniform(200, 310, 2)
    ry, rx = rng.uniform(150, 260), rng.uniform(120, 230)
    m = ((y - cy) / ry) ** 2 + ((x - cx) / rx) ** 2 < 1
    for _ in range(int(rng.integers(1, 5))):
        hy, hx = rng.integers(60, 450, 2)
        hh, hw = rng.integers(8, 70, 2)
        m[hy:hy + hh, hx:hx + hw] = False
    blocks = rng.random((16, 16)) < 0.15
    m ^= np.repeat(np.repeat(blocks, 32, 0), 32, 1) & (rng.random((512, 512)) < 0.9)
    return m.astype(np.uint8) * np.uint8(255)


def _similarity(rng, side, cx, cy):
    """face (S x S, S = 512) -> canvas: any rotation, a face `side` canvas pixels wide centred at (cx, cy)."""
    a = rng.uniform(-np.pi, np.pi)
    s = side / 512.
    c, si = np.cos(a) * s, np.sin(a) * s
    return np.array([[c, -si, cx - (c * 256 - si * 256)], [si, c, cy - (si * 256 + c * 256)]])


def scene(i):
    """Scene i of the sweep (deterministic)."""
    rng = np.random.default_rng(1000 + i)
    up = UPSCALES[i % len(UPSCALES)]
    w_edge = W_EDGES[i]
    side = 24 + 20 * w_edge if w_edge else 14           # the face's side on the canvas
    f64 = i % 7 == 3
    upsampled = not f64 and i % 6 == 4 and up == 2       # a face upsampler: the faces are 1024 wide
    # the canvas holds the first face with some margin; small faces get a canvas of at least ~120 pixels
    h_up, w_up = (max(int(side * rng.uniform(1.1, 1.6)), 120) + int(rng.integers(0, 16)) for _ in range(2))
    h, w = max(int(h_up / up), 2), max(int(w_up / up), 2)
    h_up, w_up = int(h * up), int(w * up)
    faces = _faces()
    n = 1 + i % 3
    idx = [int(v) for v in rng.integers(0, len(faces), n)]
    Ts = [_similarity(rng, side, w_up * rng.uniform(0.4, 0.6), h_up * rng.uniform(0.4, 0.6))]
    for j in range(1, n):
        kind = (i + j) % 4
        s2 = side * rng.uniform(0.5, 1.2)
        if kind == 0:        # overlapping the first face
            c = (Ts[0][0, 2] + Ts[0][0, 0] * 256 + Ts[0][0, 1] * 256 + side * 0.3, Ts[0][1, 2] + Ts[0][1, 0] * 256 + Ts[0][1, 1] * 256)
        elif kind == 1:      # partly off the canvas
            c = (rng.choice([0., w_up]) + rng.uniform(-s2 / 4, s2 / 4), rng.uniform(0, h_up))
        elif kind == 2:      # wholly off it
            c = (-s2 * 2 if rng.random() < 0.5 else w_up + s2 * 2, rng.uniform(-s2, h_up + s2))
        else:                # anywhere
            c = (rng.uniform(0, w_up), rng.uniform(0, h_up))
        Ts.append(_similarity(rng, s2, *c))
    img = O.synthetic_background(h, w, i)
    fs = [faces[k] for k in idx]
    if f64:
        fs = [f.astype(np.float64) * rng.uniform(0.6, 0.95) + rng.uniform(3, 20) for f in fs]
    elif upsampled:
        fs = [np.repeat(np.repeat(f, 2, 0), 2, 1) for f in fs]
    invs = [T.copy() for T in Ts]                    # get_inverse_affine's matrices: the 512-wide face -> the canvas
    masks = np.stack([parse_mask(rng) for _ in range(n)]) if i % 4 != 1 else None
    upsample = None
    if i % 5 == 2:
        upsample = O.synthetic_upsample(img, int(np.ceil(up)))[:h_up, :w_up] if up == int(up) else None
    elif i % 5 == 4:        # another size than the output: INTER_LANCZOS4 to it
        upsample = O.synthetic_background(int(h_up * 0.8) + 3, int(w_up * 0.7) + 5, i + 7)
    return SimpleNamespace(i=i, img=img, faces=np.stack(fs), invs=invs, upscale=up, masks=masks, upsample=upsample,
                           upsampled=upsampled, f64=f64, out_size=(w_up, h_up))


def adjusted(sc):
    """The scene's inverse affines after paste_faces_to_input_image's own adjustment (face_restoration_helper.py:388-399)."""
    inv = [m.copy() for m in sc.invs]
    for m in inv:
        if sc.upsampled:
            m /= sc.upscale
            m[:, 2] *= sc.upscale
        else:
            m[:, 2] += 0.5 * sc.upscale if sc.upscale > 1 else 0
    return inv


def background(sc, lanczos):
    """The canvas the faces go into: INTER_LINEAR of the input, or upsample_img (INTER_LANCZOS4 to the output size)."""
    if sc.upsample is None:
        return O.resize_linear_u8(sc.img, sc.out_size)
    if sc.upsample.shape[:2] == sc.out_size[::-1]:
        return sc.upsample
    return lanczos(sc.upsample, sc.out_size)


def oracle_paste(sc, return_info=False):
    """The scene through the CPU oracle: (final image, float canvas, per-face info or None)."""
    bg = background(sc, resize_lanczos4_u8)
    if sc.f64:
        canvas = G.paste_faces_f64(sc.img, list(sc.faces), [m.copy() for m in sc.invs], sc.upscale, sc.masks, bg)
        return G.final_cast(canvas), canvas, None
    canvas, info = O.paste_faces(sc.img, list(sc.faces), [m.copy() for m in sc.invs], sc.upscale, sc.masks, bg,
                                 face_upsampler=(lambda f: f) if sc.upsampled else None, return_info=True)
    return O.to_u8(canvas), canvas, info


def cv2_paste(cv2, sc):
    """paste_faces_to_input_image:372-499 written out with cv2 (the parsing network's output given as masks).  Returns
    (final image, float canvas)."""
    up = sc.upscale
    w_up, h_up = sc.out_size
    if sc.upsample is None:
        canvas = cv2.resize(sc.img, (w_up, h_up), interpolation=cv2.INTER_LINEAR)
    else:
        canvas = cv2.resize(sc.upsample, (w_up, h_up), interpolation=cv2.INTER_LANCZOS4)
    for i, (face, inv) in enumerate(zip(sc.faces, adjusted(sc))):
        fs = face.shape[:2]
        inv_restored = cv2.warpAffine(face, inv, (w_up, h_up))
        inv_mask = cv2.warpAffine(np.ones(fs, np.float32), inv, (w_up, h_up))
        inv_mask_erosion = cv2.erode(inv_mask, np.ones((int(2 * up), int(2 * up)), np.uint8))
        pasted_face = inv_mask_erosion[:, :, None] * inv_restored
        total_face_area = np.sum(inv_mask_erosion)
        w_edge = int(total_face_area ** 0.5) // 20
        inv_mask_center = cv2.erode(inv_mask_erosion, np.ones((w_edge * 2, w_edge * 2), np.uint8))
        inv_soft_mask = cv2.GaussianBlur(inv_mask_center, (w_edge * 2 + 1, w_edge * 2 + 1), 0)[:, :, None]
        if sc.masks is not None:
            pm = cv2.GaussianBlur(sc.masks[i].astype(np.float64), (101, 101), 11)
            pm = cv2.GaussianBlur(pm, (101, 101), 11)
            pm[:10, :] = 0
            pm[-10:, :] = 0
            pm[:, :10] = 0
            pm[:, -10:] = 0
            pm = pm / 255.
            pm = cv2.resize(pm, fs)
            pm = cv2.warpAffine(pm, inv, (w_up, h_up), flags=3)[:, :, None]
            fuse = (pm < inv_soft_mask).astype('int')
            inv_soft_mask = pm * fuse + inv_soft_mask * (1 - fuse)
        canvas = inv_soft_mask * pasted_face + (1 - inv_soft_mask) * canvas
    out = canvas.astype(np.uint16) if np.max(canvas) > 256 else canvas.astype(np.uint8)
    return out, canvas


def general_affine(rng, kind, sw, sh, ow, oh):
    """A 2 x 3 matrix source -> output of the given kind: 'shear', 'flip' (negative determinant), 'scale' (0.05 .. 8) or
    'singular' (determinant about 1e-3, so the inverse maps the output to source coordinates beyond int16)."""
    a, b = rng.uniform(-np.pi, np.pi, 2)
    R = lambda t: np.array([[np.cos(t), -np.sin(t)], [np.sin(t), np.cos(t)]])
    if kind == 'shear':
        L = R(a) @ np.array([[1., rng.uniform(-1.5, 1.5)], [0., 1.]]) @ np.diag(rng.uniform(0.3, 3, 2)) @ R(b)
    elif kind == 'flip':
        L = R(a) @ np.diag([-rng.uniform(0.3, 3), rng.uniform(0.3, 3)]) @ R(b)
    elif kind == 'scale':
        L = R(a) @ np.diag(np.exp(rng.uniform(np.log(0.05), np.log(8), 2)))
    else:
        u = rng.uniform(0.5, 2)
        L = R(a) @ np.array([[u, u], [u, u * (1 + 1e-3 * rng.choice([-1, 1]))]])
    c_src = np.array([sw / 2, sh / 2])
    t = np.array([ow / 2, oh / 2]) + rng.uniform(-0.3, 0.3, 2) * [ow, oh] - L @ c_src
    return np.c_[L, t]
