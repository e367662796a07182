"""Whole-image mode on the GPU: the face crop warp and the paste-back of restored faces.

Mirrors ``FaceRestoreHelper.align_warp_face`` and ``paste_faces_to_input_image``
(/root/reference/facelib/utils/face_restoration_helper.py:319-349, 372-516) with cv2's arithmetic on the device
(``cfb_warp_affine_u8`` / ``cfb_resize_linear_u8`` / ``cfb_paste_faces``, csrc/pasteback.cu).

Two levels:
  * device level -- ``warp_faces`` returns CUDA uint8 crops [N,S,S,3] that feed ``CodeFormer.forward_u8`` directly, and
    ``paste_faces`` returns the CUDA uint8 image [h_up,w_up,3];
  * drop-in level -- ``align_warp_face(face_helper)`` and ``paste_faces_to_input_image(face_helper, ...)`` take a
    ``FaceRestoreHelper`` instance and do what its methods of the same name do, so the calling script stays as it is.

The package does not import cv2.  Only the drop-in ``align_warp_face`` imports it, lazily, for
``cv2.estimateAffinePartial2D(..., LMEDS)`` (as the reference helper does).  No CPU fallback: CPU tensors raise.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from .parsing import face_parse_mask

BORDER_MODES = {'constant': 0, 'reflect': 2, 'reflect101': 4}
PARSE_SIZE = 512


def invert_affine(M):
    """``cv2.invertAffineTransform`` in double (warpAffine's own inversion)."""
    M = np.asarray(M, np.float64).reshape(2, 3)
    D = M[0, 0] * M[1, 1] - M[0, 1] * M[1, 0]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22, A12, A21 = M[1, 1] * D, M[0, 0] * D, -M[0, 1] * D, -M[1, 0] * D
    return np.array([[A11, A12, -A11 * M[0, 2] - A12 * M[1, 2]], [A21, A22, -A21 * M[0, 2] - A22 * M[1, 2]]], np.float64)


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _check_image(x, name, ndim=3):
    if not torch.is_tensor(x) or not x.is_cuda:
        raise RuntimeError(f'{name}: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
    if x.dtype != torch.uint8:
        raise NotImplementedError(f'{name}: only 8-bit images are supported, got {x.dtype}')
    if x.dim() != ndim or x.shape[-1] != 3:
        raise NotImplementedError(f'{name}: only 3-channel HWC images are supported, got shape {tuple(x.shape)}')
    return x.contiguous()


def _matrices(ms, n=None):
    a = np.ascontiguousarray(np.asarray([np.asarray(m, np.float64).reshape(2, 3) for m in ms], np.float64).reshape(-1, 6))
    if n is not None and a.shape[0] != n:
        raise RuntimeError(f'expected {n} affine matrices, got {a.shape[0]}')
    return a


def warp_faces(img, affines, face_size=512, border_mode='constant', border_value=(135, 133, 132)):
    """``cv2.warpAffine(img, M, (face_size, face_size), borderMode=..., borderValue=...)`` for every M:
    img CUDA uint8 [h,w,3] -> CUDA uint8 [N,face_size,face_size,3]."""
    img = _check_image(img, 'warp_faces')
    if border_mode not in BORDER_MODES:
        raise ValueError(f"border_mode must be one of {sorted(BORDER_MODES)}, got {border_mode!r}")
    m = _matrices(affines)
    n = m.shape[0]
    h, w = img.shape[:2]
    out = torch.empty((n, face_size, face_size, 3), dtype=torch.uint8, device=img.device)
    bv = [int(v) for v in border_value]
    with torch.cuda.device(img.device):
        _lib.check(_lib.load().cfb_warp_affine_u8(_lib.ptr(img), h, w, m.ctypes.data_as(ctypes.c_void_p), n, _lib.ptr(out),
                                                  face_size, face_size, BORDER_MODES[border_mode], bv[0], bv[1], bv[2],
                                                  _stream(img.device)), 'cfb_warp_affine_u8')
    return out


def resize_linear(img, size):
    """``cv2.resize(img, size, interpolation=INTER_LINEAR)`` (size = (w, h)) on CUDA uint8 [h,w,3] or [N,h,w,3]."""
    batched = img.dim() == 4
    img = _check_image(img, 'resize_linear', 4 if batched else 3)
    x = img if batched else img[None]
    n, h, w = x.shape[:3]
    out = torch.empty((n, size[1], size[0], 3), dtype=torch.uint8, device=img.device)
    with torch.cuda.device(img.device):
        _lib.check(_lib.load().cfb_resize_linear_u8(_lib.ptr(x), n, h, w, _lib.ptr(out), size[1], size[0], _stream(img.device)),
                   'cfb_resize_linear_u8')
    return out if batched else out[0]


def resize_area(img, size):
    """``cv2.resize(img, size, interpolation=INTER_AREA)`` (size = (w, h), shrinking only) on CUDA uint8 [h,w,3] or
    [N,h,w,3] (``cfb_resize_area_u8``)."""
    batched = img.dim() == 4
    img = _check_image(img, 'resize_area', 4 if batched else 3)
    x = img if batched else img[None]
    n, h, w = x.shape[:3]
    if size[0] > w or size[1] > h:
        raise NotImplementedError(f'resize_area shrinks only ({w}x{h} -> {size[0]}x{size[1]}); use resize_linear to enlarge')
    out = torch.empty((n, size[1], size[0], 3), dtype=torch.uint8, device=img.device)
    with torch.cuda.device(img.device):
        _lib.check(_lib.load().cfb_resize_area_u8(_lib.ptr(x), n, h, w, _lib.ptr(out), size[1], size[0], _stream(img.device)),
                   'cfb_resize_area_u8')
    return out if batched else out[0]


def resize_linear_factor(img, f):
    """``cv2.resize(img, (0, 0), fx=f, fy=f, interpolation=INTER_LINEAR)`` for f >= 1 on CUDA uint8 [h,w,3] or [N,h,w,3]:
    the output is (round(h f), round(w f)) and the taps follow f itself (``cfb_resize_linear_scale_u8``)."""
    batched = img.dim() == 4
    img = _check_image(img, 'resize_linear_factor', 4 if batched else 3)
    x = img if batched else img[None]
    n, h, w = x.shape[:3]
    oh, ow = int(np.rint(h * f)), int(np.rint(w * f))
    out = torch.empty((n, oh, ow, 3), dtype=torch.uint8, device=img.device)
    with torch.cuda.device(img.device):
        _lib.check(_lib.load().cfb_resize_linear_scale_u8(_lib.ptr(x), n, h, w, _lib.ptr(out), oh, ow, float(f), float(f),
                                                          _stream(img.device)), 'cfb_resize_linear_scale_u8')
    return out if batched else out[0]


def _index(img_index, n, n_img):
    idx = np.ascontiguousarray(np.asarray(img_index, np.int32).reshape(-1))
    if idx.shape[0] != n:
        raise RuntimeError(f'expected {n} image indices, got {idx.shape[0]}')
    if n and (idx.min() < 0 or idx.max() >= n_img):
        raise RuntimeError(f'image index out of range [0, {n_img})')
    return idx


def warp_faces_multi(imgs, affines, img_index, face_size=512, border_mode='constant', border_value=(135, 133, 132)):
    """``warp_faces`` across images in one launch: imgs CUDA uint8 [B,h,w,3], crop i = ``cv2.warpAffine(imgs[img_index[i]],
    affines[i], ...)`` -> CUDA uint8 [N,face_size,face_size,3]."""
    imgs = _check_image(imgs, 'warp_faces_multi', 4)
    if border_mode not in BORDER_MODES:
        raise ValueError(f"border_mode must be one of {sorted(BORDER_MODES)}, got {border_mode!r}")
    m = _matrices(affines) if len(affines) else np.zeros((0, 6), np.float64)
    n = m.shape[0]
    B, h, w = imgs.shape[:3]
    idx = _index(img_index, n, B)
    out = torch.empty((n, face_size, face_size, 3), dtype=torch.uint8, device=imgs.device)
    bv = [int(v) for v in border_value]
    with torch.cuda.device(imgs.device):
        _lib.check(_lib.load().cfb_warp_affine_multi_u8(_lib.ptr(imgs), B, h, w, m.ctypes.data_as(ctypes.c_void_p),
                                                        idx.ctypes.data_as(ctypes.c_void_p), n, _lib.ptr(out), face_size,
                                                        face_size, BORDER_MODES[border_mode], bv[0], bv[1], bv[2],
                                                        _stream(imgs.device)), 'cfb_warp_affine_multi_u8')
    return out


def _paste_multi(canvases, restored, inverse_affines, img_index, upscale, masks):
    """The paste over several canvases [B,h_up,w_up,3] (the backgrounds, already at the output size) with matrices already
    adjusted; face i goes into canvas img_index[i].  Returns (CUDA uint8 [B,h_up,w_up,3], w_edge per face)."""
    canvases = _check_image(canvases, 'paste_faces_multi', 4).clone()
    restored = _check_image(restored, 'paste_faces_multi: restored faces', 4)
    n, S = restored.shape[0], restored.shape[1]
    if restored.shape[2] != S:
        raise RuntimeError(f'paste_faces_multi: restored faces must be square, got {tuple(restored.shape)}')
    B, h_up, w_up = canvases.shape[:3]
    m = _matrices(inverse_affines, n) if n else np.zeros((0, 6), np.float64)
    idx = _index(img_index, n, B)
    if masks is not None:
        if not (torch.is_tensor(masks) and masks.is_cuda and masks.dtype == torch.uint8 and tuple(masks.shape) == (n, PARSE_SIZE, PARSE_SIZE)):
            raise RuntimeError(f'paste_faces_multi: parse masks must be CUDA uint8 [{n},512,512]')
        masks = masks.contiguous()
    lib = _lib.load()
    dev = canvases.device
    mp = m.ctypes.data_as(ctypes.c_void_p)
    need = lib.cfb_paste_faces_multi_workspace_bytes(B, h_up, w_up, n, S, int(masks is not None), mp)
    if need < 0:
        _lib.check(1, 'cfb_paste_faces_multi_workspace_bytes')
    ws = torch.empty(int(need), dtype=torch.uint8, device=dev)
    w_edge = np.zeros(max(n, 1), np.int32)
    with torch.cuda.device(dev):
        _lib.check(lib.cfb_paste_faces_multi(_lib.ptr(canvases), B, h_up, w_up, _lib.ptr(restored), n, S, _lib.ptr(masks), mp,
                                             idx.ctypes.data_as(ctypes.c_void_p), float(upscale),
                                             w_edge.ctypes.data_as(ctypes.c_void_p), _lib.ptr(ws), ws.numel(), _stream(dev)),
                   'cfb_paste_faces_multi')
    return canvases, w_edge[:n]


def paste_faces_multi(imgs, restored, inverse_affines, img_index, upscale, face_parse=None, upsample_imgs=None,
                      face_size=512, masks=None):
    """``paste_faces`` across images: imgs CUDA uint8 [B,h,w,3] (equal-size input images), restored [N,S,S,3], face i
    belonging to image img_index[i]; ``upsample_imgs`` (optional, CUDA uint8 [B,h_up,w_up,3]) replaces the resized
    backgrounds.  Each output image equals ``paste_faces`` of that image and its own faces.  -> CUDA uint8
    [B,h_up,w_up,3]."""
    imgs = _check_image(imgs, 'paste_faces_multi', 4)
    if restored.dim() != 4:
        raise RuntimeError('paste_faces_multi: restored faces must be [N,S,S,3]')
    S = restored.shape[1]
    if S not in (face_size, face_size * upscale):
        raise RuntimeError(f'paste_faces_multi: restored faces are {S} wide; expected {face_size} or {face_size} * upscale')
    B, h, w = imgs.shape[:3]
    h_up, w_up = int(h * upscale), int(w * upscale)
    if upsample_imgs is None:
        canvases = resize_linear(imgs, (w_up, h_up))
    else:
        canvases = _check_image(upsample_imgs, 'paste_faces_multi: upsample_imgs', 4)
        if tuple(canvases.shape[:3]) != (B, h_up, w_up):
            raise NotImplementedError(f'paste_faces_multi: upsample_imgs must be [{B},{h_up},{w_up},3], got {tuple(canvases.shape)}')
    inv = adjust_inverse_affines([np.array(m, np.float64).reshape(2, 3) for m in inverse_affines], upscale,
                                 S != face_size)
    if face_parse is not None and masks is None and restored.shape[0] > 0:
        masks = parse_masks(_check_image(restored, 'paste_faces_multi: restored faces', 4), face_parse)
    return _paste_multi(canvases, restored, inv, img_index, upscale, masks)[0]


def adjust_inverse_affines(inverse_affines, upscale, upsampled):
    """The reference's in-place adjustment before the warp (face_restoration_helper.py:388-399): with a face upsampler
    ``/= upscale`` and ``[:, 2] *= upscale``; otherwise ``[:, 2] += 0.5 * upscale`` when upscale > 1."""
    for inv in inverse_affines:
        if upsampled:
            inv /= upscale
            inv[:, 2] *= upscale
        else:
            inv[:, 2] += 0.5 * upscale if upscale > 1 else 0
    return inverse_affines


def parse_masks(restored, face_parse):
    """The parse masks of paste_faces_to_input_image:458-468 for all faces at once: resize to 512 (INTER_LINEAR),
    img2tensor + normalize, ``face_parse(x)[0]``, argmax + MASK_COLORMAP.  -> CUDA uint8 [N,512,512] (0/255)."""
    faces = restored if restored.shape[1] == PARSE_SIZE else resize_linear(restored, (PARSE_SIZE, PARSE_SIZE))
    n = faces.shape[0]
    x = torch.empty((n, 3, PARSE_SIZE, PARSE_SIZE), dtype=torch.float32, device=faces.device)
    with torch.cuda.device(faces.device):
        _lib.check(_lib.load().cfb_u8_to_input(_lib.ptr(faces.contiguous()), _lib.ptr(x), n, PARSE_SIZE * PARSE_SIZE,
                                               _stream(faces.device)), 'cfb_u8_to_input')
    with torch.no_grad():
        logits = face_parse(x)[0]
    return face_parse_mask(logits)[1]


def _paste(img, restored, inverse_affines, upscale, face_size, masks, upsample_img, debug=False):
    """The paste itself, with matrices already adjusted.  Returns (CUDA uint8 image, w_edge per face[, f32 canvas])."""
    img = _check_image(img, 'paste_faces')
    restored = _check_image(restored, 'paste_faces: restored faces', 4)
    n, S = restored.shape[0], restored.shape[1]
    if restored.shape[2] != S:
        raise RuntimeError(f'paste_faces: restored faces must be square, got {tuple(restored.shape)}')
    h, w = img.shape[:2]
    h_up, w_up = int(h * upscale), int(w * upscale)
    if upsample_img is None:
        canvas = resize_linear(img, (w_up, h_up))
    else:
        upsample_img = _check_image(upsample_img, 'paste_faces: upsample_img')
        if tuple(upsample_img.shape[:2]) != (h_up, w_up):
            raise NotImplementedError(f'paste_faces: upsample_img must be {h_up}x{w_up} (the image times upscale), got '
                                      f'{tuple(upsample_img.shape[:2])}; resize it first')
        canvas = upsample_img.clone()
    m = _matrices(inverse_affines, n)
    if masks is not None:
        if not (torch.is_tensor(masks) and masks.is_cuda and masks.dtype == torch.uint8 and tuple(masks.shape) == (n, PARSE_SIZE, PARSE_SIZE)):
            raise RuntimeError(f'paste_faces: parse masks must be CUDA uint8 [{n},512,512]')
        masks = masks.contiguous()
    lib = _lib.load()
    dev = img.device
    need = lib.cfb_paste_faces_workspace_bytes(h_up, w_up, n, S, int(masks is not None), m.ctypes.data_as(ctypes.c_void_p))
    if need < 0:
        _lib.check(1, 'cfb_paste_faces_workspace_bytes')
    ws = torch.empty(int(need), dtype=torch.uint8, device=dev)
    w_edge = np.zeros(max(n, 1), np.int32)
    dbg = torch.empty((h_up, w_up, 3), dtype=torch.float32, device=dev) if debug else None
    with torch.cuda.device(dev):
        _lib.check(lib.cfb_paste_faces(_lib.ptr(canvas), h_up, w_up, _lib.ptr(restored), n, S, _lib.ptr(masks),
                                       m.ctypes.data_as(ctypes.c_void_p), float(upscale), _lib.ptr(dbg),
                                       w_edge.ctypes.data_as(ctypes.c_void_p), _lib.ptr(ws), ws.numel(), _stream(dev)),
                   'cfb_paste_faces')
    return (canvas, w_edge[:n], dbg) if debug else (canvas, w_edge[:n])


def paste_faces(img, restored, inverse_affines, upscale, face_parse=None, upsample_img=None, face_size=512, masks=None):
    """Device-level paste_faces_to_input_image: img CUDA uint8 [h,w,3] (the input image), restored CUDA uint8 [N,S,S,3]
    with S = face_size, or S = face_size * upscale for faces that went through a face upsampler, inverse_affines as
    ``get_inverse_affine`` leaves them (not modified here).  ``face_parse`` (a module mapping [N,3,512,512] CUDA to a
    tuple whose first entry is the logits, e.g. ``init_parsing_model()``) selects use_parse; ``masks`` (CUDA uint8
    [N,512,512], 0/255) gives the parse masks directly instead.  Returns CUDA uint8 [h_up,w_up,3]."""
    if restored.dim() != 4:
        raise RuntimeError('paste_faces: restored faces must be [N,S,S,3]')
    S = restored.shape[1]
    if S == face_size:
        upsampled = False
    elif S == face_size * upscale:
        upsampled = True
    else:
        raise RuntimeError(f'paste_faces: restored faces are {S} wide; expected {face_size} or {face_size} * upscale')
    inv = adjust_inverse_affines([np.array(m, np.float64).reshape(2, 3) for m in inverse_affines], upscale, upsampled)
    if face_parse is not None and masks is None:
        masks = parse_masks(_check_image(restored, 'paste_faces: restored faces', 4), face_parse)
    return _paste(img, restored, inv, upscale, S, masks, upsample_img)[0]


# ---- drop-in level ------------------------------------------------------------------------------------------------
def _host_image(img, name):
    img = np.asarray(img)
    if img.dtype != np.uint8:
        raise NotImplementedError(f'{name}: only 8-bit images are supported, got {img.dtype}')
    if img.ndim != 3 or img.shape[2] != 3:
        raise NotImplementedError(f'{name}: only 3-channel BGR images are supported (gray and alpha stay caller-side), '
                                  f'got shape {img.shape}')
    return img


def _to_device(x, dev, name):
    if torch.is_tensor(x):
        if not x.is_cuda:
            raise RuntimeError(f'{name}: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
        return x
    return torch.from_numpy(np.ascontiguousarray(_host_image(x, name))).to(dev)


def align_warp_face(face_helper, border_mode='constant', device='cuda'):
    """``FaceRestoreHelper.align_warp_face`` (face_restoration_helper.py:319-349) with the crops warped on the GPU.
    Appends to ``affine_matrices`` / ``cropped_faces`` (host uint8, as the reference) and returns the crops as CUDA uint8
    [N,S,S,3] for ``forward_u8``."""
    import cv2    # estimateAffinePartial2D(LMEDS) stays on the host, as in the reference
    if getattr(face_helper, 'pad_blur', False):
        raise NotImplementedError('align_warp_face: pad_blur stays caller-side')
    img = _to_device(face_helper.input_img, device, 'align_warp_face')
    size = tuple(face_helper.face_size)
    if size[0] != size[1]:
        raise NotImplementedError('align_warp_face: only square face sizes are supported')
    affines = [cv2.estimateAffinePartial2D(lm, face_helper.face_template, method=cv2.LMEDS)[0]
               for lm in face_helper.all_landmarks_5]
    face_helper.affine_matrices.extend(affines)
    if not affines:
        return torch.empty((0, size[1], size[0], 3), dtype=torch.uint8, device=img.device)
    crops = warp_faces(img, affines, size[0], border_mode)
    face_helper.cropped_faces.extend(list(crops.cpu().numpy()))
    return crops


def paste_faces_to_input_image(face_helper, upsample_img=None, draw_box=False, face_upsampler=None, device='cuda'):
    """``FaceRestoreHelper.paste_faces_to_input_image`` (face_restoration_helper.py:372-516) on the GPU; returns the host
    uint8 image as the reference does.  ``face_helper.face_parse`` is used when ``use_parse`` (any module mapping
    [N,3,512,512] CUDA to logits first, e.g. ``init_parsing_model()``); ``face_upsampler`` is duck-typed
    (``.enhance(face, outscale=...)[0]``).  The inverse affine matrices are adjusted in place, as the reference does."""
    if draw_box:
        raise NotImplementedError('paste_faces_to_input_image: draw_box (a debug overlay) is not supported')
    img = _to_device(face_helper.input_img, device, 'paste_faces_to_input_image')
    upscale = face_helper.upscale_factor
    fs = tuple(face_helper.face_size)
    if fs[0] != fs[1]:
        raise NotImplementedError('paste_faces_to_input_image: only square face sizes are supported')
    if len(face_helper.restored_faces) != len(face_helper.inverse_affine_matrices):
        raise AssertionError('length of restored_faces and affine_matrices are different.')
    h, w = img.shape[:2]
    h_up, w_up = int(h * upscale), int(w * upscale)
    if upsample_img is not None:
        up = np.asarray(upsample_img) if not torch.is_tensor(upsample_img) else upsample_img
        if tuple(up.shape[:2]) != (h_up, w_up):
            raise NotImplementedError(f'paste_faces_to_input_image: upsample_img must be {h_up}x{w_up}, got {tuple(up.shape[:2])}')
        upsample_img = _to_device(up, img.device, 'paste_faces_to_input_image: upsample_img')
    faces = list(face_helper.restored_faces)
    if face_upsampler is not None:
        faces = [face_upsampler.enhance(f if not torch.is_tensor(f) else f.cpu().numpy(), outscale=upscale)[0] for f in faces]
        size = fs[0] * upscale
    else:
        size = fs[0]
    adjust_inverse_affines(face_helper.inverse_affine_matrices, upscale, face_upsampler is not None)
    if faces:
        restored = torch.stack([_to_device(f, img.device, 'restored face') for f in faces]).contiguous()
    else:
        restored = torch.empty((0, size, size, 3), dtype=torch.uint8, device=img.device)
    if restored.shape[1] != size:
        raise RuntimeError(f'paste_faces_to_input_image: restored faces are {restored.shape[1]} wide, expected {size}')
    masks = None
    if face_helper.use_parse and restored.shape[0] > 0:
        masks = parse_masks(restored, face_helper.face_parse)
    out, _ = _paste(img, restored, face_helper.inverse_affine_matrices, upscale, size, masks, upsample_img)
    return out.cpu().numpy()
