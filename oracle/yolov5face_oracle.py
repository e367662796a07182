"""YOLOv5l-face restated op for op on the CPU in fp32 (torch), from a state dict.

Reference: facelib/detection/yolov5face/ of the reference tree: models/yolov5l.yaml (the layer list), models/common.py (Conv,
StemBlock, C3, Bottleneck, SPP), models/yolo.py (Detect, forward :52-86), face_detector.py (YoloDetector._preprocess,
detect_faces) and utils/datasets.py (letterbox).  The preprocessing uses pasteback_oracle's numpy restatement of cv2's
INTER_LINEAR resize, so no cv2 is needed; the host post-processing is the package's own finish_detections.
tests/test_oracle_yolov5face.py checks all of it bit for bit against the unmodified reference classes.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from codeformer_b200.yolov5face import STRIDES, YOLOV5L_C3, finish_detections
from oracle.pasteback_oracle import resize_linear_u8


def _conv(sd, p, x, stride=1):
    w = sd[p + '.conv.weight']
    y = F.conv2d(x, w, None, stride, w.shape[-1] // 2)
    y = F.batch_norm(y, sd[p + '.bn.running_mean'], sd[p + '.bn.running_var'], sd[p + '.bn.weight'], sd[p + '.bn.bias'], False,
                     0.03, 1e-5)
    return F.silu(y)


def _c3(sd, i, x):
    n = {li: nb for li, _, _, nb in YOLOV5L_C3}[i]
    p = f'model.{i}'
    y = _conv(sd, p + '.cv1', x)
    for j in range(n):
        t = _conv(sd, f'{p}.m.{j}.cv2', _conv(sd, f'{p}.m.{j}.cv1', y))
        y = y + t if i in (1, 3, 5) else t            # backbone C3s: shortcut (Bottleneck.add)
    return _conv(sd, p + '.cv3', torch.cat((y, _conv(sd, p + '.cv2', x)), 1))


def _up(x):
    return F.interpolate(x, scale_factor=2., mode='nearest')


def forward(sd, x):
    """x [B,3,H,W] fp32 (RGB / 255, H and W multiples of 32) -> (pred [B,P,16], [x_l [B,3,ny,nx,16]])."""
    s1 = _conv(sd, 'model.0.stem_1', x, 2)
    s2b = _conv(sd, 'model.0.stem_2b', _conv(sd, 'model.0.stem_2a', s1), 2)
    s2p = F.max_pool2d(s1, 2, 2, 0, ceil_mode=True)
    y = _conv(sd, 'model.0.stem_3', torch.cat((s2b, s2p), 1))
    y = _c3(sd, 1, y)
    x3 = _c3(sd, 3, _conv(sd, 'model.2', y, 2))
    x5 = _c3(sd, 5, _conv(sd, 'model.4', x3, 2))
    y = _conv(sd, 'model.7.cv1', _conv(sd, 'model.6', x5, 2))
    y = _conv(sd, 'model.7.cv2', torch.cat([y] + [F.max_pool2d(y, k, 1, k // 2) for k in (3, 5, 7)], 1))
    x9 = _conv(sd, 'model.9', _c3(sd, 8, y))
    x13 = _conv(sd, 'model.13', _c3(sd, 12, torch.cat((_up(x9), x5), 1)))
    p3 = _c3(sd, 16, torch.cat((_up(x13), x3), 1))
    p4 = _c3(sd, 19, torch.cat((_conv(sd, 'model.17', p3, 2), x13), 1))
    p5 = _c3(sd, 22, torch.cat((_conv(sd, 'model.20', p4, 2), x9), 1))
    z, raws = [], []
    for lv, f in enumerate((p3, p4, p5)):
        o = F.conv2d(f, sd[f'model.23.m.{lv}.weight'], sd[f'model.23.m.{lv}.bias'])
        bs, _, ny, nx = o.shape
        r = o.view(bs, 3, 16, ny, nx).permute(0, 1, 3, 4, 2).contiguous()
        raws.append(r)
        yy, xx = torch.meshgrid(torch.arange(ny, device=o.device), torch.arange(nx, device=o.device), indexing='ij')
        grid = torch.stack((xx, yy), 2).view(1, 1, ny, nx, 2).float()
        ag = sd['model.23.anchor_grid'][lv]
        s = STRIDES[lv]
        d = torch.zeros_like(r)
        sig = [0, 1, 2, 3, 4, 15]
        d[..., sig] = r[..., sig].sigmoid()
        d[..., 5:15] = r[..., 5:15]
        d[..., 0:2] = (d[..., 0:2] * 2.0 - 0.5 + grid) * s
        d[..., 2:4] = (d[..., 2:4] * 2) ** 2 * ag
        for k in range(5, 15, 2):
            d[..., k:k + 2] = d[..., k:k + 2] * ag + grid * s
        z.append(d.view(bs, -1, 16))
    return torch.cat(z, 1), raws


def preprocess(imgs, target_size=None):
    """YoloDetector._preprocess of BGR uint8 images (after detect_faces' BGR -> RGB): [B,3,H,W] fp32, RGB / 255."""
    out = []
    for img in imgs:
        img = np.ascontiguousarray(img[..., ::-1])
        h0, w0 = img.shape[:2]
        if target_size:
            r = target_size / min(h0, w0)
            if r < 1:
                img = resize_linear_u8(img, (int(w0 * r), int(h0 * r)))
        h, w = img.shape[:2]
        size = math.ceil(max(h, w) / 32) * 32
        r = min(size / h, size / w)
        nw, nh = int(round(w * r)), int(round(h * r))
        dw, dh = np.mod(size - nw, 64) / 2, np.mod(size - nh, 64) / 2
        if (w, h) != (nw, nh):
            img = resize_linear_u8(img, (nw, nh))
        top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
        left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
        canvas = np.full((nh + top + bottom, nw + left + right, 3), 114, np.uint8)
        canvas[top:top + nh, left:left + nw] = img
        out.append(canvas)
    x = torch.from_numpy(np.array(out).transpose(0, 3, 1, 2))
    return x.float() / 255.0


def candidates(pred, conf_thres):
    """Per image the prediction rows whose objectness is > conf_thres, in order (non_max_suppression_face's x[xc[xi]])."""
    return [p[p[:, 4] > conf_thres] for p in pred]


def detect_faces(sd, imgs, conf_thres=0.7, iou_thres=0.5, min_face=10, target_size=None):
    images = imgs if isinstance(imgs, list) else [imgs]
    x = preprocess(images, target_size)
    pred, _ = forward(sd, x)
    return finish_detections(candidates(pred, conf_thres), tuple(x.shape[2:]), [im.shape for im in images], conf_thres, iou_thres,
                             min_face)
