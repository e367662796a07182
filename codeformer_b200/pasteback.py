"""Whole-image mode on the GPU: the face crop warp and the paste-back of restored faces.

Mirrors ``FaceRestoreHelper.align_warp_face`` and ``paste_faces_to_input_image``
(/root/reference/facelib/utils/face_restoration_helper.py:319-349, 372-516) with cv2's arithmetic on the device
(``cfb_warp_affine_u8`` / ``cfb_resize_linear_u8`` / ``cfb_paste_faces``, csrc/pasteback.cu).  Gray images: the helper's
``add_restored_face`` leaves float64 faces (``gray_adain_faces`` / ``add_restored_face`` here), which the paste functions take
as CUDA float64 tensors (``cfb_paste_faces_f64``).  An upsampled background of another size is resized with cv2's
INTER_LANCZOS4 (``resize_lanczos4``), as the reference does.

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
from .parsing import ParseNet, face_parse_mask

BORDER_MODES = {'constant': 0, 'reflect': 2, 'reflect101': 4}
PARSE_SIZE = 512


def invert_affine(M):
    """``cv2.invertAffineTransform`` in double (warpAffine's own inversion)."""
    M = np.asarray(M, np.float64).reshape(2, 3)
    D = M[0, 0] * M[1, 1] - M[0, 1] * M[1, 0]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22, A12, A21 = M[1, 1] * D, M[0, 0] * D, -M[0, 1] * D, -M[1, 0] * D
    return np.array([[A11, A12, -A11 * M[0, 2] - A12 * M[1, 2]], [A21, A22, -A21 * M[0, 2] - A22 * M[1, 2]]], np.float64)


def _check_image(x, name, ndim=3, dtype=torch.uint8):
    if not torch.is_tensor(x) or not x.is_cuda:
        raise RuntimeError(f'{name}: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
    if x.dtype != dtype:
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
                                                  _lib.stream(img.device)), 'cfb_warp_affine_u8')
    return out


def resize_linear(img, size):
    """``cv2.resize(img, size, interpolation=INTER_LINEAR)`` (size = (w, h)) on CUDA uint8 [h,w,3] or [N,h,w,3]."""
    batched = img.dim() == 4
    img = _check_image(img, 'resize_linear', 4 if batched else 3)
    x = img if batched else img[None]
    n, h, w = x.shape[:3]
    out = torch.empty((n, size[1], size[0], 3), dtype=torch.uint8, device=img.device)
    with torch.cuda.device(img.device):
        _lib.check(_lib.load().cfb_resize_linear_u8(_lib.ptr(x), n, h, w, _lib.ptr(out), size[1], size[0], _lib.stream(img.device)),
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
        _lib.check(_lib.load().cfb_resize_area_u8(_lib.ptr(x), n, h, w, _lib.ptr(out), size[1], size[0], _lib.stream(img.device)),
                   'cfb_resize_area_u8')
    return out if batched else out[0]


def resize_lanczos4(img, size):
    """``cv2.resize(img, size, interpolation=INTER_LANCZOS4)`` (size = (w, h), enlarging or shrinking, byte for byte) on CUDA
    uint8 or uint16 [h,w,3] or [N,h,w,3] (``cfb_resize_lanczos4_u8`` / ``cfb_resize_lanczos4_u16``: cv2's int16 taps for 8-bit
    images, its float32 path for 16-bit ones); an [N,...] call is one launch and equals N single calls."""
    batched = img.dim() == 4
    wide = torch.is_tensor(img) and img.dtype == torch.uint16
    # a 16-bit image is checked and made contiguous as int16, the same bytes (torch's uint16 has few kernels)
    img = _check_image(img.view(torch.int16) if wide else img, 'resize_lanczos4', 4 if batched else 3,
                       torch.int16 if wide else torch.uint8)
    x = img if batched else img[None]
    n, h, w = x.shape[:3]
    out = torch.empty((n, size[1], size[0], 3), dtype=torch.uint16 if wide else torch.uint8, device=img.device)
    fn = 'cfb_resize_lanczos4_u16' if wide else 'cfb_resize_lanczos4_u8'
    with torch.cuda.device(img.device):
        _lib.check(getattr(_lib.load(), fn)(_lib.ptr(x), n, h, w, _lib.ptr(out), size[1], size[0], _lib.stream(img.device)), fn)
    return out if batched else out[0]


def gray_adain_faces(restored, cropped, with_stats=False):
    """``add_restored_face`` on a gray image (face_restoration_helper.py:364-369) for N faces at once:
    ``adain_npy(bgr2gray(restored[i]), cropped[i])``, CUDA uint8 [N,S,S,3] twice -> CUDA float64 [N,S,S,3]; with ``with_stats``
    also CUDA float64 [N,4,3]: content mean, content std, style mean, style std per channel.  The statistics are two-pass
    float64 sums in a fixed order: within 1e-13 relative of the exact statistics and 1e-10 of numpy's (whose own float64 sums
    carry a few 1e-12), identical on every run and for a face alone or inside a batch.  The result goes to ``paste_faces`` / ``paste_faces_multi`` as it is.
    ``CodeFormer.restore_faces`` does not call this; ``restore_aligned`` (the ``--has_aligned`` loop) does for gray crops."""
    restored = _check_image(restored, 'gray_adain_faces: restored faces', 4)
    cropped = _check_image(cropped, 'gray_adain_faces: cropped faces', 4)
    if restored.shape != cropped.shape or restored.shape[1] != restored.shape[2] or restored.device != cropped.device:
        raise RuntimeError(f'gray_adain_faces: expected two [N,S,S,3] tensors on one device, got {tuple(restored.shape)} and '
                           f'{tuple(cropped.shape)}')
    n, S = restored.shape[:2]
    out = torch.empty((n, S, S, 3), dtype=torch.float64, device=restored.device)
    stats = torch.empty((n, 4, 3), dtype=torch.float64, device=restored.device)
    with torch.cuda.device(restored.device):
        _lib.check(_lib.load().cfb_gray_adain_faces(_lib.ptr(restored), _lib.ptr(cropped), n, S, _lib.ptr(out), _lib.ptr(stats),
                                                    _lib.stream(restored.device)), 'cfb_gray_adain_faces')
    return (out, stats) if with_stats else out


def _check_faces(x, name):
    """Restored faces: CUDA uint8 [N,S,S,3], or float64 for the faces of a gray image."""
    if torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float64 and x.dim() == 4 and x.shape[-1] == 3:
        return x.contiguous()
    return _check_image(x, name, 4)


def _canvas(img, upsample_img, size, name):
    """The background at the output size (w_up, h_up): INTER_LINEAR of the input, or the upsampled image through
    INTER_LANCZOS4 (face_restoration_helper.py:376-381; a copy when it already has that size)."""
    batched = img.dim() == 4
    if upsample_img is None:
        return resize_linear(img, size)
    up = _check_image(upsample_img, f'{name}: upsample_img', 4 if batched else 3)
    if batched and up.shape[0] != img.shape[0]:
        raise RuntimeError(f'{name}: {up.shape[0]} upsampled images for {img.shape[0]} images')
    return resize_lanczos4(up, size)


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
                                                          _lib.stream(img.device)), 'cfb_resize_linear_scale_u8')
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
                                                        _lib.stream(imgs.device)), 'cfb_warp_affine_multi_u8')
    return out


def _paste_multi(canvases, restored, inverse_affines, img_index, upscale, masks, wide=None):
    """The paste over several canvases [B,h_up,w_up,3] (the backgrounds, already at the output size) with matrices already
    adjusted; face i goes into canvas img_index[i].  Returns (CUDA uint8 [B,h_up,w_up,3], w_edge per face).  float64 faces
    (gray images) go through ``cfb_paste_faces_f64``; ``wide`` (a dict) then receives, per image whose canvas exceeds 256, the
    CUDA uint16 image the reference returns for it (face_restoration_helper.py:496-499)."""
    canvases = _check_image(canvases, 'paste_faces_multi', 4).clone()
    restored = _check_faces(restored, 'paste_faces_multi: restored faces')
    f64 = restored.dtype == torch.float64
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
    need = (lib.cfb_paste_faces_f64_workspace_bytes if f64 else lib.cfb_paste_faces_multi_workspace_bytes)(
        B, h_up, w_up, n, S, int(masks is not None), mp)
    if need < 0:
        _lib.check(1, 'cfb_paste_faces_multi_workspace_bytes')
    ws = torch.empty(int(need), dtype=torch.uint8, device=dev)
    w_edge = np.zeros(max(n, 1), np.int32)
    if f64:
        u16 = torch.empty(canvases.shape, dtype=torch.uint16, device=dev)
        is_wide = np.zeros(B, np.int32)
        with torch.cuda.device(dev):
            _lib.check(lib.cfb_paste_faces_f64(_lib.ptr(canvases), B, h_up, w_up, _lib.ptr(restored), n, S, _lib.ptr(masks), mp,
                                               idx.ctypes.data_as(ctypes.c_void_p), float(upscale), _lib.ptr(u16),
                                               is_wide.ctypes.data_as(ctypes.c_void_p), w_edge.ctypes.data_as(ctypes.c_void_p),
                                               _lib.ptr(ws), ws.numel(), _lib.stream(dev)), 'cfb_paste_faces_f64')
        if wide is not None:
            wide.update({int(k): u16[k] for k in np.nonzero(is_wide)[0]})
        return canvases, w_edge[:n]
    with torch.cuda.device(dev):
        _lib.check(lib.cfb_paste_faces_multi(_lib.ptr(canvases), B, h_up, w_up, _lib.ptr(restored), n, S, _lib.ptr(masks), mp,
                                             idx.ctypes.data_as(ctypes.c_void_p), float(upscale),
                                             w_edge.ctypes.data_as(ctypes.c_void_p), _lib.ptr(ws), ws.numel(), _lib.stream(dev)),
                   'cfb_paste_faces_multi')
    return canvases, w_edge[:n]


def paste_faces_multi(imgs, restored, inverse_affines, img_index, upscale, face_parse=None, upsample_imgs=None,
                      face_size=512, masks=None, wide=None):
    """``paste_faces`` across images: imgs CUDA uint8 [B,h,w,3] (equal-size input images), restored [N,S,S,3], face i
    belonging to image img_index[i]; ``upsample_imgs`` (optional, CUDA uint8 [B,h_up,w_up,3]) replaces the resized
    backgrounds (resized with INTER_LANCZOS4 when their size is not the output's).  ``restored`` may be CUDA float64 (the
    faces of gray images, ``gray_adain_faces``); ``wide`` (a dict) then receives the uint16 image of every image whose canvas
    exceeds 256, as ``_paste_multi`` describes.  Each output image equals ``paste_faces`` of that image and its own faces.
    -> CUDA uint8 [B,h_up,w_up,3]."""
    imgs = _check_image(imgs, 'paste_faces_multi', 4)
    if restored.dim() != 4:
        raise RuntimeError('paste_faces_multi: restored faces must be [N,S,S,3]')
    S = restored.shape[1]
    if S not in (face_size, face_size * upscale):
        raise RuntimeError(f'paste_faces_multi: restored faces are {S} wide; expected {face_size} or {face_size} * upscale')
    B, h, w = imgs.shape[:3]
    h_up, w_up = int(h * upscale), int(w * upscale)
    canvases = _canvas(imgs, upsample_imgs, (w_up, h_up), 'paste_faces_multi')
    inv = adjust_inverse_affines([np.array(m, np.float64).reshape(2, 3) for m in inverse_affines], upscale,
                                 S != face_size)
    if face_parse is not None and masks is None and restored.shape[0] > 0:
        masks = parse_masks(_check_faces(restored, 'paste_faces_multi: restored faces'), face_parse)
    return _paste_multi(canvases, restored, inv, img_index, upscale, masks, wide)[0]


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
    img2tensor + normalize, ``face_parse(x)[0]``, argmax + MASK_COLORMAP.  -> CUDA uint8 [N,512,512] (0/255).  float64 faces
    (gray images) are 512 wide -- a face upsampler returns uint8 -- and convert with ``cfb_f64_to_input``.  uint8 faces and
    this package's ``ParseNet`` take ``ParseNet.masks_u8`` (same bytes, no fp32 tensor in between); in its fp16 precision
    the status word is checked after the parse, so an fp16 range overflow raises instead of giving masks."""
    f64 = restored.dtype == torch.float64
    if f64 and restored.shape[1] != PARSE_SIZE:
        raise NotImplementedError(f'parse_masks: float64 faces must be {PARSE_SIZE} wide, got {restored.shape[1]}')
    faces = restored if restored.shape[1] == PARSE_SIZE else resize_linear(restored, (PARSE_SIZE, PARSE_SIZE))
    if not f64 and isinstance(face_parse, ParseNet):
        mask = face_parse.masks_u8(faces)[1]
        if face_parse.precision == 'fp16':
            torch.cuda.current_stream(faces.device).synchronize()
            _lib.check(_lib.load().cfb_check_async_status(), 'parse_masks')
        return mask
    n = faces.shape[0]
    x = torch.empty((n, 3, PARSE_SIZE, PARSE_SIZE), dtype=torch.float32, device=faces.device)
    lib = _lib.load()
    with torch.cuda.device(faces.device):
        _lib.check((lib.cfb_f64_to_input if f64 else lib.cfb_u8_to_input)(_lib.ptr(faces.contiguous()), _lib.ptr(x), n,
                                                                         PARSE_SIZE * PARSE_SIZE, _lib.stream(faces.device)),
                   'cfb_f64_to_input' if f64 else 'cfb_u8_to_input')
    with torch.no_grad():
        logits = face_parse(x)[0]
    return face_parse_mask(logits)[1]


def _paste(img, restored, inverse_affines, upscale, face_size, masks, upsample_img, debug=False):
    """The paste itself, with matrices already adjusted.  Returns (CUDA uint8 image, w_edge per face[, f32 canvas]); for
    float64 faces whose canvas exceeds 256 the image is the uint16 one the reference returns."""
    img = _check_image(img, 'paste_faces')
    restored = _check_faces(restored, 'paste_faces: restored faces')
    n, S = restored.shape[0], restored.shape[1]
    if restored.shape[2] != S:
        raise RuntimeError(f'paste_faces: restored faces must be square, got {tuple(restored.shape)}')
    h, w = img.shape[:2]
    h_up, w_up = int(h * upscale), int(w * upscale)
    canvas = _canvas(img, upsample_img, (w_up, h_up), 'paste_faces')
    if restored.dtype == torch.float64:
        if debug:
            raise NotImplementedError('paste_faces: the debug canvas is built for uint8 faces')
        wide = {}
        out, w_edge = _paste_multi(canvas[None], restored, inverse_affines, [0] * n, upscale, masks, wide)
        return wide.get(0, out[0]), w_edge
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
                                       w_edge.ctypes.data_as(ctypes.c_void_p), _lib.ptr(ws), ws.numel(), _lib.stream(dev)),
                   'cfb_paste_faces')
    return (canvas, w_edge[:n], dbg) if debug else (canvas, w_edge[:n])


def paste_faces(img, restored, inverse_affines, upscale, face_parse=None, upsample_img=None, face_size=512, masks=None):
    """Device-level paste_faces_to_input_image: img CUDA uint8 [h,w,3] (the input image), restored CUDA uint8 [N,S,S,3]
    with S = face_size, or S = face_size * upscale for faces that went through a face upsampler, inverse_affines as
    ``get_inverse_affine`` leaves them (not modified here).  ``restored`` may be CUDA float64 (a gray image's faces from
    ``gray_adain_faces``; S = face_size), in which case the result is uint16 when the canvas exceeds 256, as in the reference.
    ``upsample_img`` of another size than the output is resized with INTER_LANCZOS4.  ``face_parse`` (a module mapping [N,3,512,512] CUDA to a
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
        masks = parse_masks(_check_faces(restored, 'paste_faces: restored faces'), face_parse)
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


def _to_device(x, dev, name, f64_ok=False):
    if torch.is_tensor(x):
        if not x.is_cuda:
            raise RuntimeError(f'{name}: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
        return x
    if f64_ok and np.asarray(x).dtype == np.float64 and np.asarray(x).ndim == 3 and np.asarray(x).shape[2] == 3:
        return torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    return torch.from_numpy(np.ascontiguousarray(_host_image(x, name))).to(dev)


def add_restored_face(face_helper, restored_face, input_face=None, device='cuda'):
    """``FaceRestoreHelper.add_restored_face`` (face_restoration_helper.py:364-369) with the gray branch on the GPU: when
    ``face_helper.is_gray`` and ``input_face`` is given, appends ``adain_npy(bgr2gray(restored_face), input_face)`` (host
    float64, as the reference; ``gray_adain_faces``), otherwise the face as it is.  Faces are host uint8 arrays or CUDA uint8
    tensors [S,S,3].  Without ``input_face`` a gray helper appends the plain float64 luminance, computed on the host as the
    reference does (the command-line loop always passes the cropped face)."""
    if not getattr(face_helper, 'is_gray', False):
        face_helper.restored_faces.append(restored_face)
        return
    if input_face is None:
        f = restored_face.cpu().numpy() if torch.is_tensor(restored_face) else np.asarray(restored_face)
        gray = 0.2989 * f[:, :, 2] + 0.5870 * f[:, :, 1] + 0.1140 * f[:, :, 0]
        face_helper.restored_faces.append(gray[:, :, np.newaxis].repeat(3, axis=2))
        return
    r = _to_device(restored_face, device, 'add_restored_face')
    c = _to_device(input_face, r.device, 'add_restored_face: input face')
    face_helper.restored_faces.append(gray_adain_faces(r[None], c[None])[0].cpu().numpy())


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


def paste_faces_to_input_image(face_helper, upsample_img=None, draw_box=False, face_upsampler=None, device='cuda',
                               lanczos=False):
    """``FaceRestoreHelper.paste_faces_to_input_image`` (face_restoration_helper.py:372-516) on the GPU; returns the host
    uint8 image as the reference does.  ``face_helper.face_parse`` is used when ``use_parse`` (any module mapping
    [N,3,512,512] CUDA to logits first, e.g. ``init_parsing_model()``); ``face_upsampler`` is duck-typed
    (``.enhance(face, outscale=...)[0]``).  The inverse affine matrices are adjusted in place, as the reference does.
    ``restored_faces`` may be float64 (a gray image, ``add_restored_face``): the result is then uint16 when the canvas exceeds
    256, as in the reference; a face upsampler gets such faces on the host and returns uint8.  With ``lanczos=True`` an
    ``upsample_img`` of another size than the output is resized with INTER_LANCZOS4 on the device, as the reference does
    (:381); without it such an image is refused, which catches a background made for another ``upscale``."""
    if draw_box:
        raise NotImplementedError('paste_faces_to_input_image: draw_box (a debug overlay) is not supported')
    img = _to_device(face_helper.input_img, device, 'paste_faces_to_input_image')
    upscale = face_helper.upscale_factor
    fs = tuple(face_helper.face_size)
    if fs[0] != fs[1]:
        raise NotImplementedError('paste_faces_to_input_image: only square face sizes are supported')
    if len(face_helper.restored_faces) != len(face_helper.inverse_affine_matrices):
        raise AssertionError('length of restored_faces and affine_matrices are different.')
    if upsample_img is not None:
        h_up, w_up = int(img.shape[0] * upscale), int(img.shape[1] * upscale)
        if tuple(upsample_img.shape[:2]) != (h_up, w_up) and not lanczos:
            raise NotImplementedError(f'paste_faces_to_input_image: upsample_img is {tuple(upsample_img.shape[:2])}, the output '
                                      f'{h_up}x{w_up}; pass lanczos=True for the reference\'s INTER_LANCZOS4 resize')
        upsample_img = _to_device(upsample_img, img.device, 'paste_faces_to_input_image: upsample_img')
    faces = list(face_helper.restored_faces)
    if face_upsampler is not None:
        faces = [face_upsampler.enhance(f if not torch.is_tensor(f) else f.cpu().numpy(), outscale=upscale)[0] for f in faces]
        size = fs[0] * upscale
    else:
        size = fs[0]
    adjust_inverse_affines(face_helper.inverse_affine_matrices, upscale, face_upsampler is not None)
    if faces:
        restored = [_to_device(f, img.device, 'restored face', f64_ok=True) for f in faces]
        if len({f.dtype for f in restored}) > 1:
            raise RuntimeError('paste_faces_to_input_image: restored faces mix uint8 and float64')
        restored = torch.stack(restored).contiguous()
    else:
        restored = torch.empty((0, size, size, 3), dtype=torch.uint8, device=img.device)
    if restored.shape[1] != size:
        raise RuntimeError(f'paste_faces_to_input_image: restored faces are {restored.shape[1]} wide, expected {size}')
    masks = None
    if face_helper.use_parse and restored.shape[0] > 0:
        masks = parse_masks(restored, face_helper.face_parse)
    out, _ = _paste(img, restored, face_helper.inverse_affine_matrices, upscale, size, masks, upsample_img)
    return out.cpu().numpy()
