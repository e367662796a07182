"""YOLOv5l-face on libcfb200: the second large face detector of whole-image mode (``--detection_model YOLOv5l``).

Mirrors ``YoloDetector`` of the reference's facelib/detection/yolov5face/face_detector.py with the ``Model`` of
models/yolo.py built from models/yolov5l.yaml, as ``init_detection_model('YOLOv5l')`` (facelib/detection/__init__.py:49-71)
creates it: same ``state_dict`` (662 entries incl. the BatchNorm buffers and Detect's ``anchors`` / ``anchor_grid``, so
``yolov5l-face.pth`` loads strictly), same ``forward(x) -> (pred, [x_l])`` and ``detect_faces`` result.  The letterbox
resize, the network, the Detect decode and the objectness threshold run on the GPU (``cfb_yolov5face_*``); one small
device-to-host copy brings back the candidates, and the NMS, the coordinate scaling and the int conversion run on the host
as in the reference.  No CPU fallback; inference only.  The package imports neither torchvision, cv2 nor yaml.
"""
import math
import os
from collections import OrderedDict

import numpy as np
import torch

from . import _lib
from .detection import bn_net_init, cuda_u8_image, nms
from .native import NativeNet

# (layer, c1, c2, bottlenecks) of the C3 blocks of yolov5l.yaml; the backbone ones (1, 3, 5) have shortcuts
YOLOV5L_C3 = ((1, 64, 128, 3), (3, 256, 256, 9), (5, 512, 512, 9), (8, 1024, 1024, 3), (12, 1024, 512, 3), (16, 512, 256, 3),
              (19, 512, 512, 3), (22, 1024, 1024, 3))
# (layer, c1, c2, k) of the plain Conv layers (k = 3: stride 2)
YOLOV5L_CONV = ((2, 128, 256, 3), (4, 256, 512, 3), (6, 512, 1024, 3), (9, 1024, 512, 1), (13, 512, 256, 1), (17, 256, 256, 3),
                (20, 512, 512, 3))
ANCHORS = ((4, 5, 8, 10, 13, 16), (23, 29, 43, 55, 73, 105), (146, 217, 231, 300, 335, 433))    # pixels, per level
STRIDES = (8, 16, 32)
DETECT_CH = (256, 512, 1024)


def yolov5l_spec():
    """state_dict keys -> (shape, dtype) of the reference ``Model('yolov5l.yaml')``, in registration order."""
    spec = OrderedDict()

    def conv(p, c1, c2, k):
        spec[p + '.conv.weight'] = ((c2, c1, k, k), torch.float32)
        for name in ('weight', 'bias', 'running_mean', 'running_var'):
            spec[f'{p}.bn.{name}'] = ((c2,), torch.float32)
        spec[p + '.bn.num_batches_tracked'] = ((), torch.int64)

    conv('model.0.stem_1', 3, 64, 3)
    conv('model.0.stem_2a', 64, 32, 1)
    conv('model.0.stem_2b', 32, 64, 3)
    conv('model.0.stem_3', 128, 64, 1)
    c3 = {i: (c1, c2, n) for i, c1, c2, n in YOLOV5L_C3}
    plain = {i: (c1, c2, k) for i, c1, c2, k in YOLOV5L_CONV}
    for i in range(1, 23):
        p = f'model.{i}'
        if i in c3:
            c1, c2, n = c3[i]
            c_ = c2 // 2
            conv(p + '.cv1', c1, c_, 1)
            conv(p + '.cv2', c1, c_, 1)
            conv(p + '.cv3', 2 * c_, c2, 1)
            for j in range(n):
                conv(f'{p}.m.{j}.cv1', c_, c_, 1)
                conv(f'{p}.m.{j}.cv2', c_, c_, 3)
        elif i in plain:
            conv(p, *plain[i])
        elif i == 7:
            conv(p + '.cv1', 1024, 512, 1)
            conv(p + '.cv2', 2048, 1024, 1)
    spec['model.23.anchors'] = ((3, 3, 2), torch.float32)
    spec['model.23.anchor_grid'] = ((3, 1, 3, 1, 1, 2), torch.float32)
    for lv, c in enumerate(DETECT_CH):
        spec[f'model.23.m.{lv}.weight'] = ((48, c, 1, 1), torch.float32)
        spec[f'model.23.m.{lv}.bias'] = ((48,), torch.float32)
    return spec


def _anchor_buffers():
    a = torch.tensor(ANCHORS, dtype=torch.float32).view(3, 3, 2)
    return a / torch.tensor(STRIDES, dtype=torch.float32).view(3, 1, 1), a.clone().view(3, 1, 3, 1, 1, 2)


def random_yolov5l_state_dict(seed=1, obj_gain=12.0, obj_bias=(0.6, -4.0, -4.0), cls_bias=4.0):
    """Seeded parameters with activations of order 1 through the whole network: conv weights N(0, 1/fan_in), BatchNorm gamma
    U(0.5, 1) (U(0.1, 0.3) on the Bottleneck cv2 convs, whose outputs add up along the shortcut chains), running_var
    U(0.2, 0.4) (about the variance a conv of SiLU outputs has, so the image still shapes the deepest features), running_mean / beta 0.1 N; Detect's weights N(0, 1/fan_in), bias 0.1 N.  Detect's objectness and class
    rows (fields 4 and 15 of each anchor) get ``obj_gain`` times larger weights and ``obj_bias`` (per level) / ``cls_bias``
    more bias: the class score is then close to 1, and the objectness lets a few stride-8 predictions of a noise image clear
    the default 0.7 threshold.  (The stride-16 and -32 levels of this random network vary little across the image.)"""
    g = torch.Generator().manual_seed(seed)
    anchors, anchor_grid = _anchor_buffers()
    sd = OrderedDict()
    for name, (shape, dtype) in yolov5l_spec().items():
        if dtype == torch.int64:
            t = torch.tensor(100, dtype=torch.int64)
        elif name.endswith('anchors'):
            t = anchors.clone()
        elif name.endswith('anchor_grid'):
            t = anchor_grid.clone()
        elif len(shape) == 4:
            fan_in = shape[1] * shape[2] * shape[3]
            t = torch.randn(shape, generator=g) / fan_in ** 0.5
            if name.startswith('model.23.'):
                t.view(3, 16, -1)[:, [4, 15]] *= obj_gain
        elif name.endswith('running_var'):
            t = 0.2 + 0.2 * torch.rand(shape, generator=g)
        elif name.endswith('bn.weight'):
            lo, hi = (0.1, 0.3) if '.m.' in name and '.cv2.' in name else (0.5, 1.0)
            t = lo + (hi - lo) * torch.rand(shape, generator=g)
        else:
            t = 0.1 * torch.randn(shape, generator=g)
            if name.startswith('model.23.'):
                t.view(3, 16)[:, 4] += obj_bias[int(name.split('.')[3])]
                t.view(3, 16)[:, 15] += cls_bias
        sd[name] = t
    return sd


def predictions(h, w):
    """Number of Detect rows of an h x w input (h, w multiples of 32)."""
    return 3 * ((h // 8) * (w // 8) + (h // 16) * (w // 16) + (h // 32) * (w // 32))


def _xywh2xyxy(x):
    y = x.clone()
    y[:, 0] = x[:, 0] - x[:, 2] / 2
    y[:, 1] = x[:, 1] - x[:, 3] / 2
    y[:, 2] = x[:, 0] + x[:, 2] / 2
    y[:, 3] = x[:, 1] + x[:, 3] / 2
    return y


def _scale_coords(img1_shape, coords, img0_shape):
    """scale_coords (4 columns x1 y1 x2 y2) / scale_coords_landmarks (10 columns) of utils/general.py:42-63, 249-276: in
    place on float32 columns, gain and pad computed in float64."""
    gain = min(img1_shape[0] / img0_shape[0], img1_shape[1] / img0_shape[1])
    pad = (img1_shape[1] - img0_shape[1] * gain) / 2, (img1_shape[0] - img0_shape[0] * gain) / 2
    n = coords.shape[1]
    coords[:, list(range(0, n, 2))] -= pad[0]
    coords[:, list(range(1, n, 2))] -= pad[1]
    coords[:, :n] /= gain
    for c in range(n):
        coords[:, c].clamp_(0, img0_shape[1 - c % 2])
    return coords


def finish_detections(cands, img1_shape, img0_shapes, conf_thres, iou_thres, min_face):
    """The host steps of ``YoloDetector.detect_faces`` after the objectness threshold (face_detector.py:69-148 and
    non_max_suppression_face from ``x = x[xc[xi]]`` on), on CPU float32 tensors: per image the [k, 16] prediction rows
    whose objectness is > conf_thres, in prediction order.  ``img1_shape`` is the network input (H, W), ``img0_shapes`` the
    original image shapes.  Returns an int64 [n, 15] array (box, x1 again, 5 landmarks) over all images, or None."""
    bboxes, points = [], []
    for x, img_shape in zip(cands, img0_shapes):
        det = torch.zeros((0, 16))
        x = x.clone()
        if x.shape[0]:
            x[:, 15:] *= x[:, 4:5]
            box = _xywh2xyxy(x[:, :4])
            conf, j = x[:, 15:].max(1, keepdim=True)
            x = torch.cat((box, conf, x[:, 5:15], j.float()), 1)[conf.view(-1) > conf_thres]
            if x.shape[0]:
                boxes, scores = x[:, :4] + x[:, 15:16] * 4096, x[:, 4]
                keep = nms(torch.cat((boxes, scores[:, None]), 1).numpy(), iou_thres)
                det = x[torch.as_tensor(keep, dtype=torch.long)]
        image_height, image_width = img_shape[:2]
        gn = torch.tensor(img_shape)[[1, 0, 1, 0]]
        gn_lks = torch.tensor(img_shape)[[1, 0, 1, 0, 1, 0, 1, 0, 1, 0]]
        _scale_coords(img1_shape, det[:, :4], img_shape)          # the reference discards the .round() of both
        _scale_coords(img1_shape, det[:, 5:15], img_shape)
        for k in range(det.size()[0]):
            b = (det[k, :4].view(1, 4) / gn).view(-1).tolist()
            b = list(map(int, [b[0] * image_width, b[1] * image_height, b[2] * image_width, b[3] * image_height]))
            if b[3] - b[1] < min_face:
                continue
            lm = (det[k, 5:15].view(1, 10) / gn_lks).view(-1).tolist()
            lm = list(map(int, [v * image_width if i % 2 == 0 else v * image_height for i, v in enumerate(lm)]))
            bboxes.append(b)
            points.append(lm)
    if not points:
        return None
    bboxes = np.array(bboxes, dtype=np.int64).reshape(-1, 4)
    return np.concatenate((bboxes, bboxes[:, :1], np.array(points, dtype=np.int64).reshape(-1, 10)), axis=1)


def letterbox_geometry(h0, w0, target_size=None):
    """``_preprocess`` of one h0 x w0 image (face_detector.py:50-67, letterbox with auto=True): the target_size resize (or
    None), the letterbox resize (or None), the canvas (H, W) and the (top, left) offset of the image in it."""
    first = None
    h, w = h0, w0
    if target_size:
        r = target_size / min(h0, w0)
        if r < 1:
            first = (int(h0 * r), int(w0 * r))
            h, w = first
    imgsz = math.ceil(max(h, w) / 32) * 32
    r = min(imgsz / h, imgsz / w)
    nw, nh = int(round(w * r)), int(round(h * r))
    dw, dh = np.mod(imgsz - nw, 64) / 2, np.mod(imgsz - nh, 64) / 2
    second = (nh, nw) if (w, h) != (nw, nh) else None
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    return first, second, (nh + top + bottom, nw + left + right), (top, left)


def _yolov5l_init(name, entry, g):
    """The detectors' defaults (``bn_net_init``), plus Detect's anchor buffers."""
    leaf = name.rsplit('.', 1)[-1]
    if leaf in ('anchors', 'anchor_grid'):
        return _anchor_buffers()[0 if leaf == 'anchors' else 1].clone()
    return bn_net_init(name, entry, g)


class YOLOv5lFace(NativeNet):
    """Parameter holder with the reference ``Model('yolov5l.yaml')``'s ``state_dict``, ``stride`` and ``forward`` on the wgmma
    conv engine."""

    def __init__(self):
        super().__init__('yolov5face', (), yolov5l_spec(), _yolov5l_init)
        self.stride = torch.tensor([8., 16., 32.])
        self.yaml_file = 'yolov5l.yaml'
        self.eval()

    def _run(self, x, H, W, u8=None, raw=True):
        """x: fp32 NCHW [B,3,H,W], or uint8 BGR [B,h,w,3] with u8 = (top, left) inside the H x W canvas."""
        lib = _lib.load()
        dev = x.device
        B = x.shape[0]
        if H % 32 or W % 32 or H < 32 or W < 32:
            raise RuntimeError(f'YOLOv5lFace: H and W must be positive multiples of 32 (got {H}x{W})')
        P = predictions(H, W)
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            pred = torch.empty((B, P, 16), dtype=torch.float32, device=dev)
            raws = [torch.empty((B, 3, H // s, W // s, 16), dtype=torch.float32, device=dev) for s in STRIDES] if raw else []
            rp = [_lib.ptr(r) for r in raws] if raw else [None] * 3
            ws = self._workspace(B, H, W, dev)
            st = _lib.stream(dev)
            if u8 is None:
                _lib.check(lib.cfb_yolov5face_forward(self._net, _lib.ptr(x), _lib.ptr(pred), *rp, B, H, W, _lib.ptr(ws),
                                                      ws.numel(), st), 'cfb_yolov5face_forward')
            else:
                _lib.check(lib.cfb_yolov5face_forward_u8(self._net, _lib.ptr(x), x.shape[1], x.shape[2], u8[0], u8[1], _lib.ptr(pred),
                                                         *rp, B, H, W, _lib.ptr(ws), ws.numel(), st),
                           'cfb_yolov5face_forward_u8')
        return pred, raws

    def forward(self, x):
        """x [B,3,H,W] fp32 CUDA (RGB / 255, H and W multiples of 32) -> (pred [B,P,16], [x_l [B,3,H/s,W/s,16] for s = 8, 16,
        32]): Detect's inference output (yolo.py:52-86)."""
        if not (torch.is_tensor(x) and x.is_cuda):
            raise RuntimeError('YOLOv5lFace.forward: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
        if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != 3:
            raise RuntimeError(f'YOLOv5lFace.forward: expected float32 [B,3,H,W], got {x.dtype} {tuple(x.shape)}')
        return self._run(x.contiguous(), x.shape[2], x.shape[3])

    def forward_u8(self, images, canvas=None, offset=(0, 0), raw=True):
        """uint8 HWC BGR images [B,h,w,3] (CUDA) placed at ``offset`` = (top, left) of a ``canvas`` = (H, W) letterbox
        (default: the image itself) whose other pixels are 114 -> the ``forward`` outputs of that canvas in RGB / 255."""
        if not (torch.is_tensor(images) and images.is_cuda and images.dtype == torch.uint8 and images.dim() == 4 and images.shape[3] == 3):
            raise RuntimeError('YOLOv5lFace.forward_u8: expected a CUDA uint8 [B,H,W,3] tensor')
        H, W = canvas if canvas is not None else (images.shape[1], images.shape[2])
        return self._run(images.contiguous(), int(H), int(W), (int(offset[0]), int(offset[1])), raw)

    def candidates(self, pred, h, w, conf_thres=0.7):
        """Rows of ``pred`` whose objectness is > conf_thres, in prediction order: one CPU tensor per image (the
        ``x[xc[xi]]`` of non_max_suppression_face on the device)."""
        lib = _lib.load()
        B, P = pred.shape[0], pred.shape[1]
        if P != predictions(h, w):
            raise RuntimeError(f'candidates: {P} predictions do not belong to a {h}x{w} input')
        dev = pred.device
        with torch.cuda.device(dev):
            rows = torch.empty((B, P, 16), dtype=torch.float32, device=dev)
            counts = torch.empty((B,), dtype=torch.int32, device=dev)
            _lib.check(lib.cfb_yolov5face_candidates(_lib.ptr(pred.contiguous()), B, h, w, float(conf_thres), _lib.ptr(rows),
                                                     _lib.ptr(counts), _lib.stream(dev)),
                       'cfb_yolov5face_candidates')
            n = counts.cpu().tolist()
        return [rows[b, :n[b]].cpu() for b in range(B)]


def _resize_u8(x, h, w):
    """cv2.resize(INTER_LINEAR) of uint8 [B,h0,w0,3] CUDA images to h x w (cfb_resize_linear_u8)."""
    lib = _lib.load()
    out = torch.empty((x.shape[0], h, w, 3), dtype=torch.uint8, device=x.device)
    _lib.check(lib.cfb_resize_linear_u8(_lib.ptr(x), x.shape[0], x.shape[1], x.shape[2], _lib.ptr(out), h, w,
                                        _lib.stream(x.device)), 'cfb_resize_linear_u8')
    return out


class YoloDetector:
    """``YoloDetector`` (face_detector.py) for ``models/yolov5l.yaml``: ``.detector`` is a :class:`YOLOv5lFace`;
    ``detect_faces`` returns the reference's int64 [n, 15] array or None."""

    def __init__(self, config_name, min_face=10, target_size=None, device='cuda'):
        cfg = os.path.basename(str(config_name))
        if cfg != 'yolov5l.yaml':
            raise NotImplementedError(f'codeformer_b200 builds the YOLOv5l face detector (models/yolov5l.yaml), not {cfg!r}'
                                      + ('; YOLOv5n needs depthwise convs' if cfg == 'yolov5n.yaml' else ''))
        self.target_size = target_size
        self.min_face = min_face
        self.detector = YOLOv5lFace()
        self.device = device

    def detect_faces(self, imgs, conf_thres=0.7, iou_thres=0.5):
        """uint8 HWC BGR image, or list of equal-size images (numpy or CUDA tensors) -> int64 [n, 15] (box, x1, 5
        landmarks; all images' faces in order) or None."""
        images = imgs if isinstance(imgs, list) else [imgs]
        dev = next(self.detector.parameters()).device
        if dev.type != 'cuda':
            raise RuntimeError('YoloDetector.detect_faces: the detector is not on a CUDA device; there is no CPU fallback')
        batch = [cuda_u8_image(im, dev, 'YoloDetector.detect_faces', 'numpy arrays or CUDA tensors').to(dev) for im in images]
        shapes = [tuple(int(s) for s in im.shape) for im in batch]
        if len(set(shapes)) != 1:
            raise ValueError(f'detect_faces: the images of one call must have the same size, got {shapes}')
        h0, w0 = shapes[0][:2]
        first, second, (H, W), (top, left) = letterbox_geometry(h0, w0, self.target_size)
        x = torch.stack(batch)
        with torch.cuda.device(dev):
            if first is not None:
                x = _resize_u8(x, *first)
            if second is not None:
                x = _resize_u8(x, *second)
            pred, _ = self.detector.forward_u8(x, (H, W), (top, left), raw=False)
            cands = self.detector.candidates(pred, H, W, conf_thres)
        return finish_detections(cands, (H, W), shapes, conf_thres, iou_thres, self.min_face)
