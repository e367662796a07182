"""Whole-image restoration over batches of images or video frames.

``restore_images`` gives, for every image, exactly what the per-image loop of inference_codeformer.py:178-229 gives with
``FaceRestoreHelper(upscale, face_size=512, crop_ratio=(1, 1), det_model, save_ext='png', use_parse=parser is not None)``
and this package's drop-ins: read_image (with its INTER_LINEAR enlargement of images whose short side is below 512),
``get_face_landmarks_5(only_center_face, resize=640, eye_dist_threshold=5)``, ``align_warp_face``, CodeFormer with
``adain=True``, ``add_restored_face``, the optional background upsampler, ``get_inverse_affine`` and
``paste_faces_to_input_image``.  It runs them across images instead of one image at a time:

  * images of equal size are stacked and go through the resizes and the detector as one batch (the detector's resize to
    a short side of 640 is ``cfb_resize_area_u8`` when it shrinks, cv2's INTER_AREA);
  * the crops of all images of a chunk are warped in one launch (``cfb_warp_affine_multi_u8``) and restored by
    ``CodeFormer.forward_u8`` in batches of at most ``max_batch`` faces; the parse masks are batched the same way;
  * the paste-back runs once per chunk of images (``cfb_paste_faces_multi``), one read-back of the erosion areas.

  * a ``codeformer_b200.RealESRGANer`` background / face upsampler whose scale is ``upscale`` runs once per chunk on the
    device (``enhance_batch``): the chunk's images, then its restored faces (the colour faces as uint8, the gray images'
    float64 faces as a second batch), each as one batch of tiles.  With another scale
    it is called per image / per face through ``enhance(img, outscale=upscale)``, which runs the network and cv2's
    INTER_LANCZOS4 on the device.  A background whose size is not the output's (``read_image`` enlarged the image, or any
    other upsampler's result) goes through INTER_LANCZOS4 on the device (``resize_lanczos4``), as the reference's paste does;
  * gray images (``is_gray``) take the gray branch of ``add_restored_face`` for their own faces: one ``gray_adain_faces``
    call over the chunk's gray faces, then the float64 paste (``cfb_paste_faces_f64``) over the gray images' canvases after
    the uint8 paste of the colour images' faces.  A chunk may mix gray and colour images; the colour ones are untouched.

``restore_images_sweep`` gives ``restore_images`` at several fidelity weights from one pass of everything that does not
depend on ``w``: detection, the crop warp and the background run once per chunk, each face's encoder and Transformer once
(``CodeFormer.forward_u8_sweep``); the decoder, the gray colour transfer, the face upsampler, the masks and the paste per weight.

``restore_aligned`` is the ``--has_aligned`` loop of the same script (:180-213) over already aligned crops of any size: the
INTER_LINEAR resize to 512x512, the gray test of all crops in one launch (``cfb_is_gray_u8``), CodeFormer in batches and the
gray crops' colour transfer, all on the device.

What stays on the host, as in the reference: the NMS and the landmark filter, ``get_center_face``,
``cv2.estimateAffinePartial2D(LMEDS)`` (cv2 is imported lazily, as ``align_warp_face`` does), and the ``enhance`` of any
other upsampler, per image.  Every result is per image: batching and chunking do not change any byte.
"""
import numpy as np
import torch

from . import _lib
from .arch import fidelity_weights, sweep_chunks, sweep_weights
from .detection import RetinaFace, cuda_u8_image
from .detection import finish_detections as retinaface_finish
from .upsampler import RealESRGANer
from .pasteback import (_paste_multi, adjust_inverse_affines, gray_adain_faces, parse_masks, resize_area, resize_lanczos4,
                        resize_linear, resize_linear_factor, warp_faces_multi)
from .yolov5face import YoloDetector, _resize_u8, letterbox_geometry
from .yolov5face import finish_detections as yolo_finish

FACE_SIZE = 512
# FaceRestoreHelper's 5-point template for face_size 512, crop_ratio (1, 1)
FACE_TEMPLATE = np.array([[192.98138, 239.94708], [318.90277, 240.1936], [256.63416, 314.01935],
                          [201.26117, 371.41043], [313.08905, 371.15118]]) * (FACE_SIZE / 512.0)


def is_gray(img, threshold=10):
    """facelib's ``is_gray`` on a host uint8 BGR image: the mean variance of the channel differences is <= threshold."""
    c = [np.asarray(img[:, :, i], dtype=np.int16) for i in range(3)]
    diff = ((c[0] - c[1]).var() + (c[1] - c[2]).var() + (c[2] - c[0]).var()) / 3.0
    return bool(diff <= threshold)


def _gray_sums(x):
    """``cfb_is_gray_u8``: CUDA uint8 [N,h,w,3] -> host int64 [N,6], {Σd1, Σd2, Σd3, Σd1², Σd2², Σd3²} of the channel
    differences d1 = B-G, d2 = G-R, d3 = R-B of each image: one launch, one read-back."""
    x = x.contiguous()
    n, h, w = x.shape[:3]
    sums = torch.empty((n, 6), dtype=torch.int64, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().cfb_is_gray_u8(_lib.ptr(x), n, h, w, _lib.ptr(sums), _lib.stream(x.device)), 'cfb_is_gray_u8')
    return sums.cpu().numpy()


def _device_is_gray(imgs, threshold=10):
    """``is_gray`` of a CUDA image [h,w,3] (a bool) or of a batch [N,h,w,3] (a list of N) from exact integer moments (the
    variances numpy computes, up to its rounding)."""
    batched = imgs.dim() == 4
    x = imgs if batched else imgs[None]
    n = x.shape[1] * x.shape[2]
    flags = []
    for row in _gray_sums(x):
        total = 0.0
        for k in range(3):
            s, s2 = int(row[k]), int(row[3 + k])
            total += (n * s2 - s * s) / (n * n)
        flags.append(bool(total / 3.0 <= threshold))
    return flags if batched else flags[0]


def get_center_face(det_faces, h=0, w=0):
    """facelib's ``get_center_face`` (face_restoration_helper.py:40-52) with the image centre."""
    center = np.array([w / 2, h / 2])
    dist = [np.linalg.norm(np.array([(f[0] + f[2]) / 2, (f[1] + f[3]) / 2]) - center) for f in det_faces]
    idx = dist.index(min(dist))
    return det_faces[idx], idx


def _detect(detector, x):
    """``detect_faces`` of each image of x (CUDA uint8 [B,h,w,3]) with the detector's defaults, one forward for the batch:
    a list of B host arrays (or None), as ``detect_faces`` returns them."""
    B, h, w = x.shape[:3]
    if isinstance(detector, RetinaFace):
        loc, conf, landms = detector.forward_u8(x)
        cands = detector.candidates(loc, conf, landms, h, w, 0.8)
        return [retinaface_finish(c.cpu().numpy(), 0.8, 0.4) for c in cands]
    if isinstance(detector, YoloDetector):
        first, second, (H, W), (top, left) = letterbox_geometry(h, w, detector.target_size)
        if first is not None:
            x = _resize_u8(x, *first)
        if second is not None:
            x = _resize_u8(x, *second)
        pred, _ = detector.detector.forward_u8(x, (H, W), (top, left), raw=False)
        cands = detector.detector.candidates(pred, H, W, 0.7)
        return [yolo_finish([c], (H, W), [(h, w, 3)], 0.7, 0.5, detector.min_face) for c in cands]
    raise NotImplementedError(f'restore_images: detector {type(detector).__name__} is not built; use '
                              'init_detection_model("retinaface_resnet50") or init_detection_model("YOLOv5l")')


def _landmarks(bboxes, scale, h, w, only_center_face, eye_dist_threshold):
    """The host part of ``get_face_landmarks_5`` after ``detect_faces``: rescale, eye-distance filter, centre face."""
    if bboxes is None or bboxes.shape[0] == 0:
        return []
    bboxes = bboxes / scale
    lms, det_faces = [], []
    for bbox in bboxes:
        eye_dist = np.linalg.norm([bbox[6] - bbox[8], bbox[7] - bbox[9]])
        if eye_dist_threshold is not None and eye_dist < eye_dist_threshold:
            continue
        lms.append(np.array([[bbox[i], bbox[i + 1]] for i in range(5, 15, 2)]))
        det_faces.append(bbox[0:5])
    if not det_faces:
        return []
    if only_center_face:
        _, idx = get_center_face(det_faces, h, w)
        lms = [lms[idx]]
    return lms


def _chunks(images, max_batch):
    """Indices of the images grouped by size (first appearance order), each group cut into runs of <= max_batch."""
    groups = {}
    for i, im in enumerate(images):
        groups.setdefault(tuple(im.shape), []).append(i)
    out = []
    for idx in groups.values():
        out += [idx[k:k + max_batch] for k in range(0, len(idx), max_batch)]
    return out


def _as_input(img, dev, name='restore_images'):
    """-> (CUDA uint8 [h,w,3], host array or None, came from the host)."""
    if isinstance(img, np.ndarray):
        if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
            raise NotImplementedError(f'{name} takes uint8 HWC BGR images with 3 channels (gray, alpha and 16-bit '
                                      f'images stay caller-side), got {img.dtype} {img.shape}')
        return cuda_u8_image(img, dev, name), img, True
    if torch.is_tensor(img):
        if not img.is_cuda:
            raise RuntimeError(f'{name}: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
        return cuda_u8_image(img, dev, name).contiguous(), None, False
    raise NotImplementedError(f'{name} takes numpy arrays or CUDA tensors, got {type(img).__name__}')


def _restore(net, crops, w, max_batch, errors, adain=True, name='restore_images'):
    """CodeFormer over the crops in batches of <= max_batch (``w``: a float, or a float32 tensor of one weight per crop); a
    failed batch gives its input faces back (the reference's per-face fallback, inference_codeformer.py:208-210)."""
    out = torch.empty_like(crops)
    dev = crops.device
    for lo in range(0, crops.shape[0], max_batch):
        hi = min(crops.shape[0], lo + max_batch)
        try:
            res = net.forward_u8(crops[lo:hi], w=w[lo:hi] if torch.is_tensor(w) else w, adain=adain)
            torch.cuda.current_stream(dev).synchronize()
            _lib.check(_lib.load().cfb_check_async_status(), name)
            out[lo:hi] = res
        except RuntimeError as err:
            errors.append((lo, str(err)))
            out[lo:hi] = crops[lo:hi]
    return out


def _on_device(upsampler, upscale):
    """The upsampler runs through ``enhance_batch``: this package's RealESRGANer over its 3-channel RRDBNet at its own scale."""
    return isinstance(upsampler, RealESRGANer) and upsampler._device_path() and upscale == float(upsampler.scale)


def _restore_sweep(net, crops, ws, max_batch, errors, name='restore_images_sweep'):
    """CodeFormer over the crops at each weight of ``ws`` (a float32 tensor [K]): ``forward_u8_sweep`` over chunks of
    ``max(1, max_batch // K)`` crops.  Returns K tensors like ``crops``; a failed chunk gives its input faces back in every
    variant (the reference's per-face fallback, inference_codeformer.py:208-210)."""
    outs = [torch.empty_like(crops) for _ in range(ws.shape[0])]
    dev = crops.device
    for lo, hi in sweep_chunks(crops.shape[0], ws.shape[0], max_batch):
        try:
            res = net.forward_u8_sweep(crops[lo:hi], ws, adain=True)
            torch.cuda.current_stream(dev).synchronize()
            _lib.check(_lib.load().cfb_check_async_status(), name)
            for k, o in enumerate(outs):
                o[lo:hi] = res[:, k]
        except RuntimeError as err:
            errors.append((lo, str(err)))
            for o in outs:
                o[lo:hi] = crops[lo:hi]
    return outs


def _net_device(net, name):
    dev = next(net.parameters()).device
    if dev.type != 'cuda':
        raise RuntimeError(f'{name}: the network is not on a CUDA device; there is no CPU fallback')
    return dev


def _restore_pipeline(inputs, detector, parser, restore, upscale, only_center_face, detection_resize, eye_dist_threshold,
                      bg_upsampler, face_upsampler, max_batch, dev):
    """The body of ``restore_images`` with its CodeFormer stage as a parameter: ``restore(crops, idx, owner)`` gives the
    restored faces of a chunk's crops as a list of V variants (V = 1 for ``restore_images``, one per weight for a sweep).  The
    gray test, resizes, detection, landmark fits, crop warp, background and inverse affines run once per chunk; the gray
    colour transfer, the face upsampler, the parse masks and the paste run per variant, each variant pasted on the one
    background.  Returns (results[v][i], crops_out[i], faces_out[v][i])."""
    import cv2    # estimateAffinePartial2D(LMEDS) / invertAffineTransform stay on the host, as in the reference
    n_img = len(inputs)
    results, crops_out, faces_out = None, [None] * n_img, None
    for idx in _chunks([t for t, _, _ in inputs], max_batch):
        x = torch.stack([inputs[i][0] for i in idx])
        h0, w0 = x.shape[1:3]
        # read_image: gray test, then an INTER_LINEAR enlargement (fx = fy) when the short side is below 512
        gray = [is_gray(inputs[i][1]) if inputs[i][2] else None for i in idx]
        on_dev = [k for k, i in enumerate(idx) if not inputs[i][2]]
        if on_dev:                                          # the CUDA images of the chunk in one launch
            for k, g in zip(on_dev, _device_is_gray(x if len(on_dev) == len(idx) else x[on_dev])):
                gray[k] = g
        if min(h0, w0) < 512:
            x = resize_linear_factor(x, 512.0 / min(h0, w0))
        h, wd = x.shape[1:3]
        # get_face_landmarks_5(resize=640): INTER_AREA when shrinking, INTER_LINEAR otherwise
        scale = detection_resize / min(h, wd)
        dh, dw = int(h * scale), int(wd * scale)
        xd = resize_area(x, (dw, dh)) if scale < 1 else resize_linear(x, (dw, dh))
        with torch.no_grad():
            dets = _detect(detector, xd)
        lms = [_landmarks(d, scale, h, wd, only_center_face, eye_dist_threshold) for d in dets]
        affines, owner = [], []
        for k, lm in enumerate(lms):
            for landmark in lm:
                affines.append(cv2.estimateAffinePartial2D(landmark, FACE_TEMPLATE, method=cv2.LMEDS)[0])
                owner.append(k)
        crops = warp_faces_multi(x, affines, owner, FACE_SIZE)
        with torch.no_grad():
            restored_v = restore(crops, idx, owner)
        if results is None:
            results = [[None] * n_img for _ in restored_v]
            faces_out = [[None] * n_img for _ in restored_v]
        owner = np.asarray(owner, np.int64)
        # add_restored_face: the faces of gray images become adain_npy(bgr2gray(restored), cropped), float64
        is_g = np.asarray([gray[k] for k in owner], bool)
        gsel, csel = np.nonzero(is_g)[0], np.nonzero(~is_g)[0]
        gt, ct = torch.from_numpy(gsel).to(dev), torch.from_numpy(csel).to(dev)
        variants = []
        for restored in restored_v:
            gray_faces = gray_adain_faces(restored[gt], crops[gt]) if len(gsel) else None
            S = FACE_SIZE
            if face_upsampler is not None and len(affines):
                S = int(FACE_SIZE * upscale)
                up = torch.empty((len(affines), S, S, 3), dtype=torch.uint8, device=dev)

                def no_16bit(wide):
                    if any(wide):
                        raise NotImplementedError('restore_images: the face upsampler returned a 16-bit face (a gray face above '
                                                  '256 is 16-bit to RealESRGANer.enhance); 16-bit faces are not pasted')

                def host_faces(faces):
                    res = [np.asarray(face_upsampler.enhance(f, outscale=upscale)[0]) for f in faces]
                    no_16bit([r.dtype != np.uint8 for r in res])
                    if any(r.shape != (S, S, 3) for r in res):
                        raise RuntimeError(f'restore_images: the face upsampler returned {res[0].shape[:2]}, expected {S}x{S}')
                    return torch.from_numpy(np.ascontiguousarray(np.stack(res))).to(dev)
                if len(csel):
                    if _on_device(face_upsampler, upscale):
                        up[ct] = face_upsampler.enhance_batch(restored[ct], outscale=upscale)
                    else:
                        up[ct] = host_faces(restored[ct].cpu().numpy())
                if len(gsel):          # the float64 faces come back uint8, as enhance returns them in the reference
                    if _on_device(face_upsampler, upscale):
                        res = face_upsampler.enhance_batch(gray_faces, outscale=upscale)
                        no_16bit([r.dtype != torch.uint8 for r in res])
                        up[gt] = torch.stack(res)
                    else:
                        up[gt] = host_faces(gray_faces.cpu().numpy())
                restored, gray_faces = up, None
            variants.append((restored, gray_faces))
        h_up, w_up = int(h * upscale), int(wd * upscale)
        if bg_upsampler is not None and _on_device(bg_upsampler, upscale):
            canvases = bg_upsampler.enhance_batch(torch.stack([inputs[i][0] for i in idx]), outscale=upscale)
        elif bg_upsampler is not None:
            bgs = []
            for i in idx:
                src = inputs[i][1] if inputs[i][2] else inputs[i][0].cpu().numpy()
                bg = np.asarray(bg_upsampler.enhance(src, outscale=upscale)[0])
                if bg.dtype != np.uint8 or bg.ndim != 3 or bg.shape[2] != 3:
                    raise NotImplementedError(f'restore_images: the background upsampler returned {bg.dtype} {bg.shape}; only '
                                              'uint8 BGR backgrounds are pasted')
                bgs.append(torch.from_numpy(np.ascontiguousarray(bg)))
            canvases = torch.stack(bgs).to(dev)
        else:
            canvases = resize_linear(x, (w_up, h_up))
        if tuple(canvases.shape[1:3]) != (h_up, w_up):      # paste_faces_to_input_image: INTER_LANCZOS4 to the output size
            canvases = resize_lanczos4(canvases, (w_up, h_up))
        invs = []
        for a in affines:
            inv = cv2.invertAffineTransform(a)
            inv *= upscale
            invs.append(inv)
        adjust_inverse_affines(invs, upscale, face_upsampler is not None)

        def masks_of(faces):
            if parser is None or faces.shape[0] == 0:
                return None
            with torch.no_grad():
                return torch.cat([parse_masks(faces[lo:lo + max_batch], parser) for lo in range(0, faces.shape[0], max_batch)])
        for v, (restored, gray_faces) in enumerate(variants):      # _paste_multi pastes on a copy of the canvases
            wide = {}
            if gray_faces is None:
                out, _ = _paste_multi(canvases, restored, invs, owner, upscale, masks_of(restored))
            else:
                # the uint8 paste for the colour images' faces, then the float64 paste over the gray images' canvases alone
                out, _ = _paste_multi(canvases, restored[ct], [invs[j] for j in csel], owner[csel], upscale,
                                      masks_of(restored[ct]))
                gk = np.unique(owner[gsel])
                gkt = torch.from_numpy(gk).to(dev)
                gw = {}
                out_g, _ = _paste_multi(out[gkt], gray_faces, [invs[j] for j in gsel], np.searchsorted(gk, owner[gsel]),
                                        upscale, masks_of(gray_faces), gw)
                out[gkt] = out_g
                wide = {int(gk[k]): val for k, val in gw.items()}
            for k, i in enumerate(idx):
                sel = torch.from_numpy(np.nonzero(owner == k)[0]).to(dev)
                res = wide.get(k, out[k])
                faces = restored[sel]
                if gray_faces is not None and gray[k]:
                    faces = gray_faces[torch.from_numpy(np.searchsorted(gsel, np.nonzero(owner == k)[0])).to(dev)]
                if inputs[i][2]:
                    results[v][i] = res.cpu().numpy()
                    if v == 0:
                        crops_out[i] = crops[sel].cpu().numpy()
                    faces_out[v][i] = faces.cpu().numpy()
                else:
                    results[v][i] = res
                    if v == 0:
                        crops_out[i] = crops[sel]
                    faces_out[v][i] = faces
    return results, crops_out, faces_out


def restore_images(images, net, detector, parser=None, w=0.5, upscale=2, only_center_face=False, detection_resize=640,
                   eye_dist_threshold=5, bg_upsampler=None, face_upsampler=None, max_batch=32, return_faces=False):
    """Restore whole images in batches.  ``images``: a list of uint8 HWC BGR numpy arrays or CUDA tensors.  ``net``: a
    ``CodeFormer``; ``detector``: ``init_detection_model('retinaface_resnet50' | 'YOLOv5l')``; ``parser``: a ParseNet
    (``init_parsing_model()``) or None for use_parse=False.  ``bg_upsampler`` / ``face_upsampler``: objects with
    ``enhance(img, outscale=upscale)`` (``RealESRGANer``).  A ``codeformer_b200.RealESRGANer`` over ``RRDBNet`` with
    ``scale == upscale`` runs on the device, once per chunk of images for the backgrounds and once for the restored faces
    (``enhance_batch``); any other upsampler is called per image / per face through ``enhance`` (for this package's
    RealESRGANer at another scale that call runs the network and the INTER_LANCZOS4 resize on the device).  The float64 faces
    of gray images go with the colour ones: one ``enhance_batch`` of the chunk's gray faces on the device, or ``enhance`` per
    face; they come back uint8 as in the reference (a face above 256 is 16-bit to ``enhance``: NotImplementedError).

    Returns the restored images (host uint8 arrays for host inputs, CUDA tensors for CUDA inputs); with ``return_faces``
    also, per image, the cropped faces [n,512,512,3] and the restored faces as they were pasted (float64 for a gray image
    without a face upsampler, as the reference's ``restored_faces`` holds them).  A gray image whose pasted canvas exceeds
    256 comes back uint16, as in the reference.  Each image equals the
    reference loop body on that image alone, whatever ``max_batch`` is.  ``self.last_restore_errors`` of the reference's
    fallback is ``restore_images.last_errors``: (face offset, message) of each CodeFormer batch that fell back.

    ``w``: one fidelity weight, or one per image (``fidelity_weights`` over the images): every face of image i is restored
    with ``w[i]``, and faces of images with different weights still share CodeFormer batches."""
    images = list(images)
    dev = _net_device(net, 'restore_images')
    w = fidelity_weights(w, len(images), dev)
    if torch.is_tensor(w):
        w = w.cpu()                                    # picked per face on the host, moved with each chunk's faces
    max_batch = max(1, int(max_batch))
    inputs = [_as_input(im, dev) for im in images]
    errors = []

    def restore(crops, idx, owner):
        wf = w[torch.as_tensor(np.asarray(idx, np.int64)[np.asarray(owner, np.int64)])].to(dev) if torch.is_tensor(w) else w
        return [_restore(net, crops, wf, max_batch, errors)]
    results, crops_out, faces_out = _restore_pipeline(inputs, detector, parser, restore, upscale, only_center_face,
                                                      detection_resize, eye_dist_threshold, bg_upsampler, face_upsampler,
                                                      max_batch, dev)
    results, faces_out = (results or [[]])[0], (faces_out or [[]])[0]
    restore_images.last_errors = errors
    if return_faces:
        return results, crops_out, faces_out
    return results


restore_images.last_errors = []


def restore_images_sweep(images, net, detector, ws, parser=None, upscale=2, only_center_face=False, detection_resize=640,
                         eye_dist_threshold=5, bg_upsampler=None, face_upsampler=None, max_batch=32, return_faces=False):
    """``restore_images`` at several fidelity weights: ``results[k][i]`` equals ``restore_images(images, ..., w=ws[k])[i]``,
    byte for byte and in dtype.  ``ws``: K >= 1 weights (``sweep_weights``), shared by all images.

    Per chunk of images the gray test, the resizes, detection, the landmark fits, the crop warp and the background
    upsample run once, and every face's encoder and Transformer run once (``CodeFormer.forward_u8_sweep`` over batches of
    ``max(1, max_batch // K)`` faces).  Per weight: the gray colour transfer, the face upsampler, the parse masks (of the
    restored faces) and the paste, each on the image's one background.  With ``return_faces`` also the cropped faces per
    image (``crops[i]``) and the restored faces per weight (``faces[k][i]``).  A CodeFormer batch that fails gives its input
    faces back in every variant; ``restore_images_sweep.last_errors`` lists (face offset, message) of each."""
    images = list(images)
    dev = _net_device(net, 'restore_images_sweep')
    ws = sweep_weights(ws, dev).to(dev)
    max_batch = max(1, int(max_batch))
    inputs = [_as_input(im, dev, 'restore_images_sweep') for im in images]
    errors = []
    results, crops_out, faces_out = _restore_pipeline(
        inputs, detector, parser, lambda crops, idx, owner: _restore_sweep(net, crops, ws, max_batch, errors), upscale,
        only_center_face, detection_resize, eye_dist_threshold, bg_upsampler, face_upsampler, max_batch, dev)
    if results is None:                                # no images
        results = faces_out = [[] for _ in range(ws.shape[0])]
    restore_images_sweep.last_errors = errors
    if return_faces:
        return results, crops_out, faces_out
    return results


restore_images_sweep.last_errors = []


def restore_aligned(faces, net, w=0.5, adain=True, max_batch=32, return_crops=False):
    """The ``--has_aligned`` loop of inference_codeformer.py:180-213 over already cropped and aligned faces.  ``faces``: a
    list of uint8 HWC BGR crops of any size (numpy arrays or CUDA tensors); ``net``: a ``CodeFormer``.  Per crop, as the
    reference does for one: ``cv2.resize(img, (512, 512), INTER_LINEAR)`` (``resize_linear``, one launch per crop size),
    ``is_gray(img, threshold=10)`` of the resized crop, CodeFormer with ``w`` / ``adain`` (``forward_u8`` over all crops in
    batches of ``max_batch``; a failed batch gives its input crops back, as the reference's per-face fallback does, and
    ``restore_aligned.last_errors`` lists (crop offset, message) of each) and ``add_restored_face``: the gray crops become
    ``adain_npy(bgr2gray(restored), cropped)`` in float64 (``gray_adain_faces``).  ``w``: one fidelity weight, or one per
    crop (``fidelity_weights``).

    The gray test runs on the device for all crops at once (``cfb_is_gray_u8``): exact integer moments, so it decides as the
    reference's numpy variances do except for a crop whose score is within numpy's rounding of the threshold.

    Returns, per crop, what the reference's ``face_helper.restored_faces`` holds: uint8 [512,512,3], or float64 for a gray
    crop; host arrays for host inputs and CUDA tensors for CUDA inputs.  With ``return_crops`` also the resized crops
    (CUDA uint8 [N,512,512,3]) and the gray flags.  Results do not depend on ``max_batch``."""
    faces = list(faces)
    dev = next(net.parameters()).device
    if dev.type != 'cuda':
        raise RuntimeError('restore_aligned: the network is not on a CUDA device; there is no CPU fallback')
    max_batch = max(1, int(max_batch))
    w = fidelity_weights(w, len(faces), dev)
    if torch.is_tensor(w):
        w = w.to(dev)
    inputs = [_as_input(f, dev, 'restore_aligned') for f in faces]
    n = len(inputs)
    crops = torch.empty((n, FACE_SIZE, FACE_SIZE, 3), dtype=torch.uint8, device=dev)
    groups = {}
    for i, (t, _, _) in enumerate(inputs):
        groups.setdefault(tuple(t.shape), []).append(i)
    for shape, idx in groups.items():
        x = torch.stack([inputs[i][0] for i in idx])
        if shape[:2] != (FACE_SIZE, FACE_SIZE):        # cv2.resize to the same size is a copy
            x = resize_linear(x, (FACE_SIZE, FACE_SIZE))
        crops[torch.tensor(idx, device=dev)] = x
    gray = _device_is_gray(crops) if n else []
    errors = []
    with torch.no_grad():
        restored = _restore(net, crops, w, max_batch, errors, adain=adain, name='restore_aligned')
    gsel = np.nonzero(np.asarray(gray, bool))[0]
    gray_faces = None
    if len(gsel):
        gt = torch.from_numpy(gsel).to(dev)
        gray_faces = gray_adain_faces(restored[gt], crops[gt])
    pos = {int(i): k for k, i in enumerate(gsel)}
    results = []
    for i in range(n):
        face = gray_faces[pos[i]] if i in pos else restored[i]
        results.append(face.cpu().numpy() if inputs[i][2] else face)
    restore_aligned.last_errors = errors
    if return_crops:
        return results, crops, gray
    return results


restore_aligned.last_errors = []
