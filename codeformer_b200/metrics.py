"""Restoration metrics on the GPU: basicsr's PSNR and SSIM (basicsr/metrics/psnr_ssim.py, metric_util.py), the measures
CodeFormer's fidelity trade-off is reported with, for restored faces, fidelity sweeps and whole images.

``calculate_psnr`` / ``calculate_ssim`` are drop-ins with the reference's signature and values; ``psnr_ssim`` scores batches,
sweeps and lists of images in one launch per group of equal shape and dtype.  Semantics (cfb_psnr_ssim in include/cfb200.h):
float64 arithmetic, ``crop_border`` pixels dropped from each edge, ``test_y_channel`` as the reference's ``to_y_channel``
(channel 0 blue), PSNR peak 255 for every dtype, SSIM with the 11-tap Gaussian window (sigma 1.5) over the valid region.
Deliberate differences from the reference, which returns NaN with a warning or fails inside cv2 in these cases:
  * a negative ``crop_border``, or a cropped image without pixels (PSNR) or with a side under 11 (SSIM): ``ValueError``;
  * dtypes other than uint8, uint16, float32 and float64: ``NotImplementedError`` (two different supported dtypes are
    compared as float64, which holds all their values exactly);
  * CPU torch tensors: ``RuntimeError`` (numpy arrays are copied to the current CUDA device);
  * on the Y path, the squared differences are float32 as in the reference, but PSNR averages them in float64.
"""
import numpy as np
import torch

from . import _lib

_KIND = {torch.uint8: 0, torch.uint16: 1, torch.float32: 2, torch.float64: 3}
_NP_DTYPES = (np.uint8, np.uint16, np.float32, np.float64)
_SSIM_MIN_SIDE = 11
_MAX_PAIRS = 65535          # pairs per launch (cfb_psnr_ssim)


def _device_image(img, fn, device):
    """A numpy array or CUDA tensor of a supported dtype -> CUDA tensor (numpy arrays are copied to ``device``)."""
    if isinstance(img, np.ndarray):
        if img.dtype not in _NP_DTYPES:
            raise NotImplementedError(f'{fn}: dtype {img.dtype} is not supported (uint8, uint16, float32, float64)')
        return torch.from_numpy(np.ascontiguousarray(img)).to(device)
    if not torch.is_tensor(img):
        raise TypeError(f'{fn}: expected a numpy array or a CUDA tensor, got {type(img).__name__}')
    if not img.is_cuda:
        raise RuntimeError(f'{fn}: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
    if img.dtype not in _KIND:
        raise NotImplementedError(f'{fn}: dtype {img.dtype} is not supported (uint8, uint16, float32, float64)')
    return img


def _device_of(*imgs):
    for img in imgs:
        if torch.is_tensor(img) and img.is_cuda:
            return img.device
    return torch.device('cuda', torch.cuda.current_device())


def _same_dtype(a, b):
    return (a, b) if a.dtype == b.dtype else (a.to(torch.float64), b.to(torch.float64))


def _check_crop(h, w, crop_border, min_side, fn):
    if crop_border < 0:
        raise ValueError(f'{fn}: crop_border must be >= 0, got {crop_border}')
    if h - 2 * crop_border < min_side or w - 2 * crop_border < min_side:
        raise ValueError(f'{fn}: a {h}x{w} image with crop_border {crop_border} leaves less than {min_side} pixel(s) per side')


def _launch(a, b, k, crop_border, test_y_channel, psnr_mode, want_ssim):
    """cfb_psnr_ssim over a [P,H,W,C] against b [P/k,H,W,C] (contiguous, one dtype, one device) -> float64 [P] tensors."""
    lib = _lib.load()
    P, H, W, C = a.shape
    dev = a.device
    psnr = torch.empty(P, dtype=torch.float64, device=dev) if psnr_mode else None
    ssim = torch.empty(P, dtype=torch.float64, device=dev) if want_ssim else None
    if k > _MAX_PAIRS:
        raise ValueError(f'psnr_ssim: at most {_MAX_PAIRS} candidates per image')
    step = _MAX_PAIRS // k * k
    with torch.cuda.device(dev):
        for i in range(0, P, step):
            n = min(step, P - i)
            need = lib.cfb_psnr_ssim_workspace_bytes(n, H, W, C, crop_border, int(test_y_channel))
            if need < 0:
                _lib.check(1, 'cfb_psnr_ssim_workspace_bytes')
            ws = torch.empty(max(int(need), 1), dtype=torch.uint8, device=dev)
            _lib.check(lib.cfb_psnr_ssim(_lib.ptr(a[i:i + n]), _lib.ptr(b[i // k:(i + n) // k]), _KIND[a.dtype], n, k, H, W, C,
                                         crop_border, int(test_y_channel), psnr_mode, int(want_ssim),
                                         None if psnr is None else _lib.ptr(psnr[i:i + n]),
                                         None if ssim is None else _lib.ptr(ssim[i:i + n]), _lib.ptr(ws), ws.numel(),
                                         _lib.stream(dev)), 'cfb_psnr_ssim')
    return psnr, ssim


def _drop_in_pair(img1, img2, crop_border, input_order, min_side, fn):
    """The reference's argument handling (shape assert, input_order, reorder_image) -> two [1,H,W,C] device tensors."""
    assert img1.shape == img2.shape, f'Image shapes are different: {tuple(img1.shape)}, {tuple(img2.shape)}.'
    if input_order not in ('HWC', 'CHW'):
        raise ValueError(f'Wrong input_order {input_order}. Supported input_orders are "HWC" and "CHW"')
    if len(img1.shape) not in (2, 3):
        raise ValueError(f'{fn}: expected a 2-D or 3-D image, got shape {tuple(img1.shape)}')
    crop_border = int(crop_border)
    dev = _device_of(img1, img2)
    out = []
    for img in (img1, img2):
        if len(img.shape) == 3 and input_order == 'CHW':      # numpy arrays are reordered on the host, before the copy
            img = img.transpose(1, 2, 0) if isinstance(img, np.ndarray) else img.permute(1, 2, 0)
        out.append(_hwc(_device_image(img, fn, dev)))
    a, b = out
    if a.device != b.device:
        raise RuntimeError(f'{fn}: the two images are on different devices ({a.device}, {b.device})')
    _check_crop(a.shape[0], a.shape[1], crop_border, min_side, fn)
    a, b = _same_dtype(a, b)
    return a.contiguous()[None], b.contiguous()[None], crop_border


def calculate_psnr(img1, img2, crop_border, input_order='HWC', test_y_channel=False):
    """PSNR (dB) of two images, as ``basicsr.metrics.calculate_psnr``: ``inf`` for identical images, peak 255.

    img1 / img2: numpy arrays or CUDA tensors, HWC, CHW (``input_order``) or 2-D.  The mean squared error is computed on the
    device -- exactly, for integer images without ``test_y_channel`` -- and the final ``log10`` in numpy, so that result equals
    the reference's bit for bit."""
    a, b, crop = _drop_in_pair(img1, img2, crop_border, input_order, 1, 'calculate_psnr')
    mse, _ = _launch(a, b, 1, crop, test_y_channel, 2, False)
    mse = np.float64(mse.item())
    if mse == 0:
        return float('inf')
    return 20. * np.log10(255. / np.sqrt(mse))


def calculate_ssim(img1, img2, crop_border, input_order='HWC', test_y_channel=False):
    """SSIM of two images, as ``basicsr.metrics.calculate_ssim``: the mean over channels of the mean SSIM map.  Arguments as
    ``calculate_psnr``; the cropped image needs at least 11 x 11 pixels."""
    a, b, crop = _drop_in_pair(img1, img2, crop_border, input_order, _SSIM_MIN_SIDE, 'calculate_ssim')
    _, ssim = _launch(a, b, 1, crop, test_y_channel, 0, True)
    return np.float64(ssim.item())


def _hwc(t):
    return t[..., None] if t.dim() == 2 else t


def _psnr_ssim_lists(restored, gt, crop_border, test_y_channel):
    fn = 'psnr_ssim'
    sweep = len(restored) > 0 and isinstance(restored[0], (list, tuple))
    rows = list(restored) if sweep else [restored]
    if not isinstance(gt, (list, tuple)) or any(len(r) != len(gt) for r in rows):
        raise ValueError(f'{fn}: restored must be a list of len(gt) images, or a list of such lists')
    dev = _device_of(*gt, *[x for r in rows for x in r])
    gts = [_hwc(_device_image(g, fn, dev)) for g in gt]
    psnr = torch.empty((len(rows), len(gt)), dtype=torch.float64, device=dev)
    ssim = torch.empty_like(psnr)
    groups = {}
    for k, row in enumerate(rows):
        for i, img in enumerate(row):
            r = _hwc(_device_image(img, fn, dev))
            if r.dim() != 3 or tuple(r.shape) != tuple(gts[i].shape):
                raise ValueError(f'{fn}: restored image {i} has shape {tuple(r.shape)}, its ground truth {tuple(gts[i].shape)}')
            _check_crop(r.shape[0], r.shape[1], crop_border, _SSIM_MIN_SIDE, fn)
            r, g = _same_dtype(r, gts[i])
            groups.setdefault((tuple(r.shape), r.dtype), []).append((k, i, r, g))
    for members in groups.values():            # one launch per shape and dtype
        a = torch.stack([m[2] for m in members])
        b = torch.stack([m[3] for m in members])
        p, s = _launch(a, b, 1, crop_border, test_y_channel, 1, True)
        ks = torch.tensor([m[0] for m in members], device=dev)
        idx = torch.tensor([m[1] for m in members], device=dev)
        psnr[ks, idx] = p
        ssim[ks, idx] = s
    return (psnr, ssim) if sweep else (psnr[0], ssim[0])


def psnr_ssim(restored, gt, crop_border=0, test_y_channel=False):
    """PSNR (dB) and SSIM of restored images against their ground truth, as float64 CUDA tensors ``(psnr, ssim)``.

    * ``restored`` [B,H,W,C] against ``gt`` [B,H,W,C]: [B] each;
    * a fidelity sweep ``restored`` [B,K,H,W,C] (``CodeFormer.forward_u8_sweep``) against ``gt`` [B,H,W,C]: [B,K], the shape
      ``identity_similarity`` returns; the ground truth is read once per face, not copied K times;
    * lists of HWC or 2-D images of any sizes and dtypes (``restore_images`` results): ``restored`` a list of N images
      against ``gt`` a list of N gives [N]; a list of K such lists (``restore_images_sweep`` results, ``restored[k][i]``)
      gives [K,N].  One launch per group of equal shape and dtype.

    Images are numpy arrays or CUDA tensors.  Each value equals ``calculate_psnr`` / ``calculate_ssim`` of the pair, up to
    the rounding of the device ``log10`` (PSNR) and of the order of the sums (SSIM); it does not depend on the batch."""
    if isinstance(restored, (list, tuple)):
        return _psnr_ssim_lists(restored, gt, int(crop_border), test_y_channel)
    fn = 'psnr_ssim'
    dev = _device_of(restored, gt)
    a, b = _device_image(restored, fn, dev), _device_image(gt, fn, dev)
    if b.dim() != 4 or a.dim() not in (4, 5) or a.shape[0] != b.shape[0] or tuple(a.shape[-3:]) != tuple(b.shape[1:]):
        raise ValueError(f'{fn}: expected restored [B,H,W,C] or [B,K,H,W,C] and gt [B,H,W,C], got {tuple(a.shape)} and '
                         f'{tuple(b.shape)}')
    crop_border = int(crop_border)
    B, H, W, C = b.shape
    _check_crop(H, W, crop_border, _SSIM_MIN_SIDE, fn)
    K = a.shape[1] if a.dim() == 5 else 1
    a, b = _same_dtype(a, b)
    psnr, ssim = _launch(a.reshape(B * K, H, W, C).contiguous(), b.contiguous(), K, crop_border, test_y_channel, 1, True)
    shape = (B, K) if a.dim() == 5 else (B,)
    return psnr.view(shape), ssim.view(shape)
