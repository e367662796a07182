"""RRDBNet + RealESRGANer on libcfb200 (SURVEY.md section 8 row f4).

Mirrors, for the caller,
    RRDBNet(num_in_ch, num_out_ch, scale, num_feat, num_block, num_grow_ch)   /root/reference/basicsr/archs/rrdbnet_arch.py:67-120
    RealESRGANer(scale, model_path, model, tile, tile_pad, pre_pad, half).enhance(img, outscale)
                                                                               /root/reference/basicsr/utils/realesrgan_utils.py:14-250
as they are built by ``set_realesrgan()`` (/root/reference/inference_codeformer.py:36-61) and called on the background image
and on restored faces.  The network's arithmetic is ``cfb_rrdb_forward`` (CUDA, include/cfb200.h); this module owns the
parameters (same state-dict keys, strict load of a reference checkpoint) and the image plumbing around the model call --
colour handling, reflect pre/mod padding, the tile loop -- written against torch tensors on the device.  No CPU fallback.
"""
import ctypes
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from . import spec as S
from .native import NativeNet, Precision
from .registry import ARCH_REGISTRY


def _rrdbnet_init(name, shape, g):
    """Kaiming-normal * 0.1 weights and zero biases, like default_init_weights (arch_util.py:18-36)."""
    if name.endswith('.weight'):
        fan_in = shape[1] * shape[2] * shape[3]
        return nn.Parameter(torch.randn(shape, generator=g) * math.sqrt(2.0 / fan_in) * 0.1)
    return nn.Parameter(torch.zeros(shape))


@ARCH_REGISTRY.register()
class RRDBNet(Precision, NativeNet):
    """Parameters of the reference's RRDBNet (identical ``state_dict``) with ``forward`` on the wgmma conv engine.
    ``set_precision('fp16')`` is what the reference computes with ``half=True``; conv_first and conv_last stay fp32 in both
    precisions."""

    train = nn.Module.train          # no BatchNorm: training mode changes nothing here

    def __init__(self, num_in_ch, num_out_ch, scale=4, num_feat=64, num_block=23, num_grow_ch=32):
        if num_feat != 64 or num_grow_ch != 32:
            raise NotImplementedError('codeformer_b200 builds RRDBNet for num_feat=64, num_grow_ch=32 (the RealESRGAN models)')
        super().__init__('rrdb', (num_in_ch, num_out_ch, scale, num_feat, num_block, num_grow_ch),
                         S.rrdbnet_spec(num_in_ch, num_out_ch, scale, num_feat, num_block, num_grow_ch), _rrdbnet_init)
        self.scale, self.num_in_ch, self.num_out_ch = scale, num_in_ch, num_out_ch
        self.num_feat, self.num_block, self.num_grow_ch = num_feat, num_block, num_grow_ch

    def forward(self, x):
        """x [B, num_in_ch, H, W] fp32 CUDA -> [B, num_out_ch, H*scale, W*scale] (rrdbnet_arch.py:103-119)."""
        if not (torch.is_tensor(x) and x.is_cuda):
            raise RuntimeError('RRDBNet.forward: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
        if x.dtype != torch.float32:
            raise RuntimeError(f'RRDBNet.forward: expected float32, got {x.dtype} (the H100 path computes in split-fp16 x3 with '
                               'fp32 accumulation; .half() models are not needed)')
        if x.dim() != 4 or x.shape[1] != self.num_in_ch:
            raise RuntimeError(f'RRDBNet.forward: expected [B,{self.num_in_ch},H,W], got {tuple(x.shape)}')
        us = 2 if self.scale == 2 else (4 if self.scale == 1 else 1)
        B, _, H, W = x.shape
        if H % us or W % us:
            raise AssertionError('pixel_unshuffle needs H and W divisible by the factor (arch_util.py:202)')
        lib = _lib.load()
        x = x.contiguous()
        dev = x.device
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            out = torch.empty((B, self.num_out_ch, H // us * 4, W // us * 4), dtype=torch.float32, device=dev)
            ws = self._workspace(B, H, W, dev)
            _lib.check(lib.cfb_rrdb_forward(self._net, _lib.ptr(x), _lib.ptr(out), B, H, W, _lib.ptr(ws), ws.numel(),
                                            _lib.stream(dev)), 'cfb_rrdb_forward')
        return out


    def forward_u8_tiles(self, images, pre_pad, tiles, tile_h, tile_w, out):
        """One forward at batch ``len(tiles)`` of equal tile_h x tile_w tiles read from ``images`` (CUDA uint8 [B,H,W,3] BGR)
        and cropped into ``out`` (CUDA uint8 [B,H*scale,W*scale,3] BGR): ``cfb_rrdb_forward_u8_tiles`` (include/cfb200.h),
        rows of ``tiles`` = (image, in_y, in_x, crop_y, crop_x, crop_h, crop_w, out_y, out_x).  Used by
        ``RealESRGANer.enhance_batch``, which makes the table."""
        B, H, W, _ = images.shape
        rows = np.ascontiguousarray(np.asarray(tiles, dtype=np.int32).reshape(-1, 9))
        lib = _lib.load()
        dev = images.device
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            ws = self._workspace(rows.shape[0], tile_h, tile_w, dev)
            _lib.check(lib.cfb_rrdb_forward_u8_tiles(self._net, _lib.ptr(images), B, H, W, pre_pad,
                                                     rows.ctypes.data_as(ctypes.c_void_p), rows.shape[0], tile_h, tile_w,
                                                     _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream(dev)),
                       'cfb_rrdb_forward_u8_tiles')
        return out

    # element kinds of cfb_rrdb_forward_tiles (CFB_IMG_* of include/cfb200.h)
    IMAGE_KINDS = {torch.uint8: 0, torch.uint16: 1, torch.float32: 2, torch.float64: 3}

    def forward_tiles(self, images, pre_pad, tiles, tile_h, tile_w, out, max_range):
        """``forward_u8_tiles`` for CUDA uint8 / uint16 / float32 / float64 images [B,H,W,3] into a CUDA uint8 or uint16 ``out``
        ([B,H*scale,W*scale,3]) with the reference's per-image ``max_range`` (``cfb_rrdb_forward_tiles``): the call fills
        ``max_range`` (CUDA int32 [B]) with 255 or 65535 per image before the forward, on the device."""
        B, H, W, _ = images.shape
        rows = np.ascontiguousarray(np.asarray(tiles, dtype=np.int32).reshape(-1, 9))
        lib = _lib.load()
        dev = images.device
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            ws = self._workspace(rows.shape[0], tile_h, tile_w, dev)
            _lib.check(lib.cfb_rrdb_forward_tiles(self._net, _lib.ptr(images), self.IMAGE_KINDS[images.dtype], B, H, W, pre_pad,
                                                  rows.ctypes.data_as(ctypes.c_void_p), rows.shape[0], tile_h, tile_w,
                                                  _lib.ptr(out), self.IMAGE_KINDS[out.dtype], _lib.ptr(max_range), _lib.ptr(ws),
                                                  ws.numel(), _lib.stream(dev)), 'cfb_rrdb_forward_tiles')
        return out


def unshuffle_factor(scale):
    """pixel_unshuffle factor of RRDBNet's input, which is also pre_process's mod_scale (1: no mod pad)."""
    return 2 if scale == 2 else (4 if scale == 1 else 1)


def reflect_pad_index(n, pre_pad, scale):
    """Source index of every row (or column) of pre_process's padded image: F.pad(.., (0, pre_pad), 'reflect') of n rows, then
    the reflect pad to the pixel-unshuffle multiple.  The uint8 input conv of ``cfb_rrdb_forward_u8_tiles`` composes the same
    two maps per pixel."""
    def tail(i, m):
        return np.where(i < m, i, 2 * (m - 1) - i)
    m = unshuffle_factor(scale)
    p = n + pre_pad
    i = np.arange(p + (m - p % m) % m)
    return tail(tail(i, p), n)


class RealESRGANer:
    """The reference's helper around the upsampling network (realesrgan_utils.py:14-250): ``enhance(img)`` takes an HWC
    uint8 / uint16 / float BGR (or gray, or BGRA) image and returns ``(upsampled image, mode)``.  ``model`` is any module mapping
    [1,3,h,w] -> [1,3,h*scale,w*scale] on ``device`` (``codeformer_b200.RRDBNet`` in production; the tests also pass CPU
    stand-ins to compare the tiling against the reference's).  ``precision`` (not in the reference): ``None`` leaves the model
    as it is, a string is passed to ``model.set_precision`` -- the reference's ``half=use_half`` maps to
    ``precision='fp16' if use_half else None``."""

    def __init__(self, scale, model_path=None, model=None, tile=0, tile_pad=10, pre_pad=10, half=False, device=None, gpu_id=None,
                 precision=None):
        self.scale, self.tile_size, self.tile_pad, self.pre_pad = scale, tile, tile_pad, pre_pad
        self.mod_scale = None
        self.half = False          # accepted for signature parity and ignored; fp16 operands are opted into with `precision`
        if device is None:
            device = torch.device('cuda', gpu_id if gpu_id is not None else torch.cuda.current_device())
        self.device = torch.device(device)
        if model_path is not None:                                  # realesrgan_utils.py:59-66
            loadnet = torch.load(model_path, map_location=torch.device('cpu'))
            model.load_state_dict(loadnet['params_ema' if 'params_ema' in loadnet else 'params'], strict=True)
        model.eval()
        if precision is not None:
            model.set_precision(precision)
        self.model = model.to(self.device)

    def pre_process(self, img):
        """HWC float image -> [1,C,H,W] on the device, reflect pre-pad, reflect pad to the pixel-unshuffle multiple (:71-94)."""
        t = torch.from_numpy(np.ascontiguousarray(np.transpose(img, (2, 0, 1)))).float()
        self.img = t.unsqueeze(0).to(self.device)
        if self.pre_pad != 0:
            self.img = F.pad(self.img, (0, self.pre_pad, 0, self.pre_pad), 'reflect')
        self.mod_scale = 2 if self.scale == 2 else (4 if self.scale == 1 else None)
        if self.mod_scale is not None:
            _, _, h, w = self.img.shape
            self.mod_pad_h = (self.mod_scale - h % self.mod_scale) % self.mod_scale
            self.mod_pad_w = (self.mod_scale - w % self.mod_scale) % self.mod_scale
            self.img = F.pad(self.img, (0, self.mod_pad_w, 0, self.mod_pad_h), 'reflect')

    def process(self):
        self.output = self.model(self.img)

    def tile_plan(self, height, width):
        """Tile rectangles of tile_process (:100-175): for every tile (input rect with padding, output rect, crop of the
        model output).  Pure function of the sizes -- tested on the CPU against the reference's loop."""
        plan = []
        ts, tp, sc = self.tile_size, self.tile_pad, self.scale
        for y in range(math.ceil(height / ts)):
            for x in range(math.ceil(width / ts)):
                x0, x1 = x * ts, min(x * ts + ts, width)
                y0, y1 = y * ts, min(y * ts + ts, height)
                px0, px1 = max(x0 - tp, 0), min(x1 + tp, width)
                py0, py1 = max(y0 - tp, 0), min(y1 + tp, height)
                plan.append({'in': (py0, py1, px0, px1), 'out': (y0 * sc, y1 * sc, x0 * sc, x1 * sc),
                             'crop': ((y0 - py0) * sc, (y0 - py0) * sc + (y1 - y0) * sc, (x0 - px0) * sc, (x0 - px0) * sc + (x1 - x0) * sc)})
        return plan

    # Default bound of enhance_batch's workspace: tiles of one shape go through one forward as long as its workspace
    # (cfb_rrdb_workspace_bytes) stays within this budget, and at least one tile always does.  A 480 x 480 tile at x2 takes
    # about 0.69 GB, so the default runs six of them per forward.  The network's workspace only grows.
    WORKSPACE_BUDGET = 4 << 30

    def tile_groups(self, batch, height, width, max_tiles=None, tile_bytes=None):
        """The forwards of ``enhance_batch`` for ``batch`` images of height x width: a list of (tile_h, tile_w, rows), rows =
        (image, in_y, in_x, crop_y, crop_x, crop_h, crop_w, out_y, out_x) of tiles of one input-window shape, from
        ``tile_plan`` over the padded image (``tile == 0``: the whole padded image as one tile).  Tiles that lie in the pads only
        are dropped: post_process discards their output.  Each shape is cut into runs of at most ``max_tiles`` tiles;
        ``max_tiles=None`` takes as many as ``WORKSPACE_BUDGET`` holds, from ``tile_bytes(n, tile_h, tile_w)`` (the workspace of
        an n-tile forward).  A pure function of the sizes."""
        sc = self.scale
        hp, wp = len(reflect_pad_index(height, self.pre_pad, sc)), len(reflect_pad_index(width, self.pre_pad, sc))
        if self.tile_size > 0:
            plan = self.tile_plan(hp, wp)
        else:
            plan = [{'in': (0, hp, 0, wp), 'out': (0, hp * sc, 0, wp * sc), 'crop': (0, hp * sc, 0, wp * sc)}]
        shapes = {}
        for b in range(batch):
            for t in plan:
                py0, py1, px0, px1 = t['in']
                oy0, _, ox0, _ = t['out']
                cy0, cy1, cx0, cx1 = t['crop']
                if oy0 >= height * sc or ox0 >= width * sc:
                    continue
                shapes.setdefault((py1 - py0, px1 - px0), []).append((b, py0, px0, cy0, cx0, cy1 - cy0, cx1 - cx0, oy0, ox0))
        out = []
        for (th, tw), rows in shapes.items():
            k = max_tiles
            if k is None:
                one = tile_bytes(1, th, tw)
                k = max(1, (self.WORKSPACE_BUDGET - one) // (tile_bytes(2, th, tw) - one) + 1)
            k = max(1, int(k))
            out += [(th, tw, rows[i:i + k]) for i in range(0, len(rows), k)]
        return out

    def _device_path(self, outscale=None):
        """enhance / enhance_batch run on the device: the model is this package's 3-channel RRDBNet (any ``outscale``)."""
        m = self.model
        return isinstance(m, RRDBNet) and m.num_in_ch == 3 and m.num_out_ch == 3

    @torch.no_grad()
    def enhance_batch(self, images, outscale=None, max_tiles=None, lanczos=False):
        """``enhance`` of every image of ``images`` (CUDA [B,H,W,3] BGR) on the device.  uint8 images give CUDA uint8
        [B,H*scale,W*scale,3]; uint16, float32 and float64 images give a list of B CUDA tensors [H*scale,W*scale,3], each
        uint16 where that image's float32 maximum exceeds 256 and uint8 otherwise, as ``enhance`` picks its dtype per image.
        Each image equals ``enhance(img)[0]`` byte for byte.  With ``lanczos=True`` an ``outscale`` other than ``scale`` resizes
        the network's output to (int(W*outscale), int(H*outscale)) with cv2's INTER_LANCZOS4 on the device
        (``resize_lanczos4``, realesrgan_utils.py:245-250), one launch per output dtype, as ``enhance`` does; without it such an
        ``outscale`` is refused, so that a caller who sized its buffers for ``scale`` never gets another size.  The tiles of all
        images are grouped by input-window shape (``tile_groups``) and every group runs as forwards of at most ``max_tiles``
        tiles (default: as many as ``WORKSPACE_BUDGET`` holds) that read the images and write the integer result directly
        (``cfb_rrdb_forward_u8_tiles``, ``cfb_rrdb_forward_tiles`` for the other dtypes).  Keeps no state on ``self``: threads
        may share one upsampler.

        Raises NotImplementedError for ``outscale`` other than None / ``scale`` without ``lanczos=True``, for images that are
        not uint8 / uint16 / float32 / float64 with 3 channels and for models other than a 3-channel
        ``codeformer_b200.RRDBNet``; ValueError for an ``outscale`` that is not positive; RuntimeError for CPU tensors and for
        pads not smaller than the dimension they reflect; AssertionError, as RRDBNet.forward, for tiles whose size is not a
        multiple of the pixel-unshuffle factor."""
        if outscale is not None and outscale != float(self.scale) and not lanczos:
            raise NotImplementedError(f'RealESRGANer.enhance_batch: outscale {outscale} != scale {self.scale} changes the output '
                                      'size; pass lanczos=True for the reference\'s INTER_LANCZOS4 resize')
        if outscale is not None and not outscale > 0:
            raise ValueError(f'RealESRGANer.enhance_batch: outscale must be positive, got {outscale}')
        if not self._device_path():
            raise NotImplementedError('RealESRGANer.enhance_batch: built for a codeformer_b200.RRDBNet with 3 input and 3 output '
                                      f'channels, got {type(self.model).__name__}')
        if not torch.is_tensor(images):
            raise NotImplementedError(f'RealESRGANer.enhance_batch takes a CUDA tensor, got {type(images).__name__}')
        if not images.is_cuda:
            raise RuntimeError('RealESRGANer.enhance_batch: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
        if images.dtype not in RRDBNet.IMAGE_KINDS or images.dim() != 4 or images.shape[3] != 3:
            raise NotImplementedError(f'RealESRGANer.enhance_batch takes uint8, uint16, float32 or float64 [B,H,W,3] BGR images '
                                      f'(gray and alpha images go through enhance), got {images.dtype} {tuple(images.shape)}')
        B, H, W, _ = images.shape
        sc = self.scale
        u8 = images.dtype == torch.uint8
        if outscale is not None and outscale != float(sc):
            from .pasteback import resize_lanczos4
            size = (int(W * outscale), int(H * outscale))
            if B == 0 or H == 0 or W == 0 or size[0] == 0 or size[1] == 0:
                out = torch.empty((B, size[1], size[0], 3), dtype=torch.uint8, device=images.device)
                return out if u8 else list(out)
            up = self.enhance_batch(images, max_tiles=max_tiles)
            if u8:
                return resize_lanczos4(up, size)
            res = [None] * B
            for dt in (torch.uint8, torch.uint16):          # one launch per output dtype; uint16 is stacked as int16
                sel = [i for i in range(B) if up[i].dtype == dt]
                if sel:
                    batch = torch.stack([up[i].view(torch.int16) if dt == torch.uint16 else up[i] for i in sel])
                    for i, r in zip(sel, resize_lanczos4(batch.view(dt), size)):
                        res[i] = r
            return res
        out = torch.empty((B, H * sc, W * sc, 3), dtype=torch.uint8 if u8 else torch.uint16, device=images.device)
        if B == 0 or H == 0 or W == 0:
            return out if u8 else list(out.view(torch.int16).to(torch.uint8))
        # made contiguous through an int16 view for uint16 (torch's uint16 has few kernels): the same bytes
        images = images.view(torch.int16).contiguous().view(torch.uint16) if images.dtype == torch.uint16 else images.contiguous()
        us = unshuffle_factor(sc)
        lib = _lib.load()
        max_range = None if u8 else torch.empty(B, dtype=torch.int32, device=images.device)

        def tile_bytes(n, th, tw):
            return lib.cfb_rrdb_workspace_bytes(self.model._handle(), n, th, tw)
        for th, tw, rows in self.tile_groups(B, H, W, max_tiles, tile_bytes):
            if th % us or tw % us:
                raise AssertionError('pixel_unshuffle needs H and W divisible by the factor (arch_util.py:202)')
            if u8:
                self.model.forward_u8_tiles(images, self.pre_pad, rows, th, tw, out)
            else:
                self.model.forward_tiles(images, self.pre_pad, rows, th, tw, out, max_range)
        if u8:
            return out
        wide = (max_range == 65535).tolist()                # the one read-back: each result's dtype
        narrow = None if all(wide) else out.view(torch.int16).to(torch.uint8)
        return [out[i] if wide[i] else narrow[i] for i in range(B)]

    def tile_process(self):
        b, c, height, width = self.img.shape
        self.output = self.img.new_zeros((b, c, height * self.scale, width * self.scale))
        for t in self.tile_plan(height, width):
            py0, py1, px0, px1 = t['in']
            tile = self.model(self.img[:, :, py0:py1, px0:px1].contiguous())
            oy0, oy1, ox0, ox1 = t['out']
            cy0, cy1, cx0, cx1 = t['crop']
            self.output[:, :, oy0:oy1, ox0:ox1] = tile[:, :, cy0:cy1, cx0:cx1]

    def post_process(self):
        if self.mod_scale is not None:                              # :177-186
            _, _, h, w = self.output.shape
            self.output = self.output[:, :, 0:h - self.mod_pad_h * self.scale, 0:w - self.mod_pad_w * self.scale]
        if self.pre_pad != 0:
            _, _, h, w = self.output.shape
            self.output = self.output[:, :, 0:h - self.pre_pad * self.scale, 0:w - self.pre_pad * self.scale]
        return self.output

    def _run(self, img_rgb):
        self.pre_process(img_rgb)
        if self.tile_size > 0:
            self.tile_process()
        else:
            self.process()
        out = self.post_process().squeeze(0).float().cpu().clamp_(0, 1).numpy()
        return np.transpose(out[[2, 1, 0], :, :], (1, 2, 0))          # RGB CHW -> BGR HWC (:209-210)

    @torch.no_grad()
    def enhance(self, img, outscale=None, alpha_upsampler='realesrgan'):
        """The reference's ``enhance``.  uint8, uint16, float32 and float64 3-channel images with this package's RRDBNet go
        through ``enhance_batch``, the INTER_LANCZOS4 resize of ``outscale != scale`` included (the same bytes and dtype);
        every other case (gray, alpha, other models) through pre_process / tile_process / post_process and cv2 on the host."""
        if (img.dtype in (np.uint8, np.uint16, np.float32, np.float64) and img.ndim == 3 and img.shape[2] == 3
                and self._device_path()):
            x = torch.from_numpy(np.ascontiguousarray(img)).to(self.device)
            return self.enhance_batch(x[None], outscale=outscale, lanczos=True)[0].cpu().numpy(), 'RGB'
        return self._enhance_host(img, outscale, alpha_upsampler)

    @torch.no_grad()
    def _enhance_host(self, img, outscale=None, alpha_upsampler='realesrgan'):
        """``enhance`` through pre_process / tile_process / post_process with cv2 on the host: every dtype and channel count
        the reference takes."""
        import cv2
        h_input, w_input = img.shape[0:2]
        img = img.astype(np.float32)
        max_range = 65535 if np.max(img) > 256 else 255              # :193-199
        img = img / max_range
        alpha = None
        if img.ndim == 2:
            img_mode, img = 'L', cv2.cvtColor(img, cv2.COLOR_GRAY2RGB)
        elif img.shape[2] == 4:
            img_mode, alpha = 'RGBA', img[:, :, 3]
            img = cv2.cvtColor(img[:, :, 0:3], cv2.COLOR_BGR2RGB)
            if alpha_upsampler == 'realesrgan':
                alpha = cv2.cvtColor(alpha, cv2.COLOR_GRAY2RGB)
        else:
            img_mode, img = 'RGB', cv2.cvtColor(img, cv2.COLOR_BGR2RGB)
        output_img = self._run(img)
        if img_mode == 'L':
            output_img = cv2.cvtColor(output_img, cv2.COLOR_BGR2GRAY)
        if img_mode == 'RGBA':                                        # :218-236
            if alpha_upsampler == 'realesrgan':
                output_alpha = cv2.cvtColor(self._run(alpha), cv2.COLOR_BGR2GRAY)
            else:
                h, w = alpha.shape[0:2]
                output_alpha = cv2.resize(alpha, (w * self.scale, h * self.scale), interpolation=cv2.INTER_LINEAR)
            output_img = cv2.cvtColor(output_img, cv2.COLOR_BGR2BGRA)
            output_img[:, :, 3] = output_alpha
        if max_range == 65535:
            output = (output_img * 65535.0).round().astype(np.uint16)
        else:
            output = (output_img * 255.0).round().astype(np.uint8)
        if outscale is not None and outscale != float(self.scale):
            output = cv2.resize(output, (int(w_input * outscale), int(h_input * outscale)), interpolation=cv2.INTER_LANCZOS4)
        return output, img_mode
