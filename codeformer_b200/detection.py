"""RetinaFace-ResNet50 on libcfb200: the face detector of whole-image mode (``detect -> align -> restore -> parse -> paste``).

Mirrors ``RetinaFace(network_name='resnet50')`` of /root/reference/facelib/detection/retinaface/retinaface.py as built by
``init_detection_model('retinaface_resnet50')`` (facelib/detection/__init__.py:24-44) and called by
``FaceRestoreHelper.get_face_landmarks_5`` as ``face_detector.detect_faces(img)``: same ``state_dict`` (456 entries incl. the
BatchNorm buffers, so ``detection_Resnet50_Final.pth`` loads strictly), same ``forward(x) -> (loc, conf, landms)`` and
``detect_faces`` result.  The network, the prior boxes, the decode and the score threshold run on the GPU
(``cfb_retinaface_*``); one small device-to-host copy brings back the candidates, and the sort and the NMS run on the host
as in the reference.  No CPU fallback; inference only.  The package imports neither torchvision nor cv2.
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .native import NativeNet

RESNET50_BLOCKS = (3, 4, 6, 3)


def retinaface_spec():
    """state_dict keys -> (shape, dtype) of the reference RetinaFace('resnet50'), in registration order."""
    spec = OrderedDict()

    def conv(name, cin, cout, k, bias=False):
        spec[name + '.weight'] = ((cout, cin, k, k), torch.float32)
        if bias:
            spec[name + '.bias'] = ((cout,), torch.float32)

    def bn(name, c):
        for k in ('weight', 'bias', 'running_mean', 'running_var'):
            spec[f'{name}.{k}'] = ((c,), torch.float32)
        spec[name + '.num_batches_tracked'] = ((), torch.int64)

    conv('body.conv1', 3, 64, 7)
    bn('body.bn1', 64)
    cin = 64
    for li, (nb, wd) in enumerate(zip(RESNET50_BLOCKS, (64, 128, 256, 512))):
        for b in range(nb):
            p = f'body.layer{li + 1}.{b}'
            conv(p + '.conv1', cin, wd, 1); bn(p + '.bn1', wd)
            conv(p + '.conv2', wd, wd, 3); bn(p + '.bn2', wd)
            conv(p + '.conv3', wd, 4 * wd, 1); bn(p + '.bn3', 4 * wd)
            if b == 0:
                conv(p + '.downsample.0', cin, 4 * wd, 1); bn(p + '.downsample.1', 4 * wd)
            cin = 4 * wd
    for k, c in enumerate((512, 1024, 2048)):
        conv(f'fpn.output{k + 1}.0', c, 256, 1); bn(f'fpn.output{k + 1}.1', 256)
    for m in ('merge1', 'merge2'):
        conv(f'fpn.{m}.0', 256, 256, 3); bn(f'fpn.{m}.1', 256)
    for s in (1, 2, 3):
        for name, ci, co in (('conv3X3', 256, 128), ('conv5X5_1', 256, 64), ('conv5X5_2', 64, 64), ('conv7X7_2', 64, 64),
                             ('conv7x7_3', 64, 64)):
            conv(f'ssh{s}.{name}.0', ci, co, 3); bn(f'ssh{s}.{name}.1', co)
    for head, co in (('ClassHead', 4), ('BboxHead', 8), ('LandmarkHead', 20)):
        for k in range(3):
            conv(f'{head}.{k}.conv1x1', 256, co, 1, bias=True)
    return spec


def random_retinaface_state_dict(seed=1, class_gain=8.0, class_bias=0.0):
    """Seeded parameters with activations of order 1 through the whole network: conv weights N(0, 1/fan_in) (the stem's
    /100: it reads the mean-subtracted image), BatchNorm gamma U(0.5, 1) (bn3 / downsample U(0.1, 0.3)), running_var
    U(0.5, 1.5), running_mean / beta 0.1 N.  The ClassHead weights are ``class_gain`` times larger and the face-class channel
    gets ``class_bias`` more bias than the background channel, so that a few percent of the priors of a noise image clear
    the default 0.8 threshold."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    for name, (shape, dtype) in retinaface_spec().items():
        if dtype == torch.int64:
            t = torch.tensor(100, dtype=torch.int64)
        elif len(shape) == 4:
            fan_in = shape[1] * shape[2] * shape[3]
            t = torch.randn(shape, generator=g) / fan_in ** 0.5
            if name == 'body.conv1.weight':
                t = t / 100.0
            elif name.startswith('ClassHead.'):
                t = t * class_gain
        elif name.endswith('running_var'):
            t = 0.5 + torch.rand(shape, generator=g)
        elif name.endswith('.weight'):
            lo, hi = (0.1, 0.3) if ('bn3' in name or 'downsample.1' in name) else (0.5, 1.0)
            t = lo + (hi - lo) * torch.rand(shape, generator=g)
        else:
            t = 0.1 * torch.randn(shape, generator=g)
            if name.startswith('ClassHead.') and name.endswith('.bias'):
                t[1::2] += class_bias / 2
                t[0::2] -= class_bias / 2
        sd[name] = t
    return sd


def nms(dets, thresh):
    """``torchvision.ops.nms`` on the CPU restated in numpy (the reference's ``py_cpu_nms``): boxes ordered by a stable
    descending sort of the scores, areas (x2-x1)*(y2-y1) and IoU in float32, a box is suppressed when its IoU with a kept box
    is > thresh (compared in float64, as torchvision compares against its double threshold).  Returns the kept indices."""
    dets = np.asarray(dets, dtype=np.float32)
    if dets.shape[0] == 0:
        return []
    x1, y1, x2, y2 = (dets[:, i] for i in range(4))
    areas = (x2 - x1) * (y2 - y1)
    order = np.argsort(-dets[:, 4], kind='stable')
    suppressed = np.zeros(dets.shape[0], dtype=bool)
    keep = []
    for _i, i in enumerate(order):
        if suppressed[i]:
            continue
        keep.append(int(i))
        rest = order[_i + 1:]
        rest = rest[~suppressed[rest]]
        if rest.size == 0:
            continue
        w = np.maximum(np.float32(0), np.minimum(x2[i], x2[rest]) - np.maximum(x1[i], x1[rest]))
        h = np.maximum(np.float32(0), np.minimum(y2[i], y2[rest]) - np.maximum(y1[i], y1[rest]))
        inter = w * h
        with np.errstate(invalid='ignore', divide='ignore'):       # 0/0 of zero-area boxes is NaN, never > thresh
            ovr = inter / ((areas[i] + areas[rest]) - inter)
        suppressed[rest[ovr.astype(np.float64) > thresh]] = True
    return keep


def finish_detections(cand, conf_threshold, nms_threshold):
    """The host steps of ``detect_faces`` after the threshold (retinaface.py:226-239) on candidate rows
    [x1,y1,x2,y2,score,landmarks(10)] in prior order: ``argsort()[::-1]``, NMS, ``[n, 15]`` float32."""
    boxes, scores, landmarks = cand[:, :4], cand[:, 4], cand[:, 5:]
    order = scores.argsort()[::-1]
    boxes, landmarks, scores = boxes[order], landmarks[order], scores[order]
    bounding_boxes = np.hstack((boxes, scores[:, np.newaxis])).astype(np.float32, copy=False)
    keep = nms(bounding_boxes, nms_threshold)
    bounding_boxes, landmarks = bounding_boxes[keep, :], landmarks[keep]
    return np.concatenate((bounding_boxes, landmarks), axis=1)


def bn_net_init(name, entry, g):
    """Default state of the detectors' entries: conv weights N(0, 1/fan_in), BatchNorm (1, 0) with running stats (0, 1),
    conv biases 0."""
    shape, dtype = entry
    leaf = name.rsplit('.', 1)[-1]
    if dtype == torch.int64:
        return torch.tensor(0, dtype=torch.long)
    if leaf in ('running_mean', 'running_var'):
        return torch.zeros(shape) if leaf == 'running_mean' else torch.ones(shape)
    if len(shape) == 4:
        fan_in = shape[1] * shape[2] * shape[3]
        return nn.Parameter(torch.randn(shape, generator=g) / fan_in ** 0.5)
    return nn.Parameter(torch.ones(shape) if leaf == 'weight' else torch.zeros(shape))


def cuda_u8_image(image, device, owner, kinds='a numpy array or a CUDA tensor'):
    """One uint8 HWC BGR image of ``detect_faces`` (a numpy array, copied to ``device``, or a CUDA tensor) as a CUDA tensor."""
    if isinstance(image, np.ndarray):
        if image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] != 3:
            raise NotImplementedError(f'detect_faces takes uint8 HWC BGR images with 3 channels, got {image.dtype} {image.shape}')
        if device.type != 'cuda':
            raise RuntimeError(f'{owner}: the module is not on a CUDA device; there is no CPU fallback')
        return torch.from_numpy(np.ascontiguousarray(image)).to(device)
    if torch.is_tensor(image):
        if image.dtype != torch.uint8 or image.dim() != 3 or image.shape[2] != 3:
            raise NotImplementedError(f'detect_faces takes uint8 HWC BGR images with 3 channels, got {image.dtype} {tuple(image.shape)}')
        if not image.is_cuda:
            raise RuntimeError(f'{owner}: a torch image must be a CUDA tensor; there is no CPU fallback')
        return image
    raise NotImplementedError(f'detect_faces takes {kinds}, got {type(image).__name__}')


class RetinaFace(NativeNet):
    """Parameter holder with the reference's ``state_dict``, ``forward`` and ``detect_faces`` on the wgmma conv engine."""

    def __init__(self, network_name='resnet50', half=False, phase='test'):
        if network_name != 'resnet50':
            raise NotImplementedError(f'codeformer_b200 builds RetinaFace with network_name="resnet50" (got {network_name!r}; '
                                      'mobile0.25 needs depthwise convs)')
        if half:
            raise NotImplementedError('codeformer_b200.RetinaFace runs in float32 (half=True is not built)')
        super().__init__('retinaface', (), retinaface_spec(), bn_net_init)
        self.phase = phase
        self.half_inference = False
        self.model_name = f'retinaface_{network_name}'
        self.resize = 1.
        self.eval()

    def _run(self, x, u8):
        lib = _lib.load()
        dev = x.device
        B, H, W = (x.shape[0], x.shape[1], x.shape[2]) if u8 else (x.shape[0], x.shape[2], x.shape[3])
        P = int(lib.cfb_retinaface_priors(H, W))
        with self._lock, torch.cuda.device(dev):
            self._prepare(dev)
            loc = torch.empty((B, P, 4), dtype=torch.float32, device=dev)
            conf = torch.empty((B, P, 2), dtype=torch.float32, device=dev)
            landms = torch.empty((B, P, 10), dtype=torch.float32, device=dev)
            ws = self._workspace(B, H, W, dev)
            fn = lib.cfb_retinaface_forward_u8 if u8 else lib.cfb_retinaface_forward
            _lib.check(fn(self._net, _lib.ptr(x), _lib.ptr(loc), _lib.ptr(conf), _lib.ptr(landms), B, H, W, _lib.ptr(ws),
                          ws.numel(), _lib.stream(dev)), 'cfb_retinaface_forward')
        return loc, conf, landms

    def forward(self, inputs):
        """inputs [B,3,H,W] fp32 CUDA (mean-subtracted BGR) -> (loc [B,P,4], softmax(conf) [B,P,2], landms [B,P,10])
        (retinaface.py:122-145, phase 'test')."""
        if not (torch.is_tensor(inputs) and inputs.is_cuda):
            raise RuntimeError('RetinaFace.forward: codeformer_b200 runs on a CUDA device only; there is no CPU fallback')
        if inputs.dtype != torch.float32 or inputs.dim() != 4 or inputs.shape[1] != 3:
            raise RuntimeError(f'RetinaFace.forward: expected float32 [B,3,H,W], got {inputs.dtype} {tuple(inputs.shape)}')
        if self.phase != 'test':
            raise NotImplementedError("codeformer_b200.RetinaFace returns the phase='test' outputs (softmaxed conf) only")
        return self._run(inputs.contiguous(), False)

    def forward_u8(self, images):
        """uint8 HWC BGR images [B,H,W,3] (CUDA) -> the ``forward`` outputs of ``images - (104, 117, 123)``."""
        if not (torch.is_tensor(images) and images.is_cuda and images.dtype == torch.uint8 and images.dim() == 4 and images.shape[3] == 3):
            raise RuntimeError('RetinaFace.forward_u8: expected a CUDA uint8 [B,H,W,3] tensor')
        return self._run(images.contiguous(), True)

    def candidates(self, loc, conf, landms, h, w, conf_threshold=0.8):
        """Rows [x1,y1,x2,y2,score,landmarks(10)] in pixels of the priors with score > conf_threshold, in prior order: one
        tensor per image (the decode, the threshold and the compaction of retinaface.py:214-225 on the device)."""
        lib = _lib.load()
        B, P = loc.shape[0], loc.shape[1]
        if P != int(lib.cfb_retinaface_priors(h, w)):
            raise RuntimeError(f'candidates: {P} priors do not belong to a {h}x{w} image')
        dev = loc.device
        with torch.cuda.device(dev):
            rows = torch.empty((B, P, 15), dtype=torch.float32, device=dev)
            counts = torch.empty((B,), dtype=torch.int32, device=dev)
            _lib.check(lib.cfb_retinaface_candidates(_lib.ptr(loc.contiguous()), _lib.ptr(conf.contiguous()), _lib.ptr(landms.contiguous()),
                                                     B, h, w, float(conf_threshold), _lib.ptr(rows), _lib.ptr(counts),
                                                     _lib.stream(dev)), 'cfb_retinaface_candidates')
            n = counts.cpu().tolist()
        return [rows[b, :n[b]] for b in range(B)]

    def detect_faces(self, image, conf_threshold=0.8, nms_threshold=0.4, use_origin_size=True):
        """``RetinaFace.detect_faces`` (retinaface.py:194-239): uint8 HWC BGR image (numpy or CUDA tensor) -> float32 [n, 15]
        (box, score, 5 landmarks), highest score first after NMS."""
        if not use_origin_size:
            raise NotImplementedError('codeformer_b200.RetinaFace.detect_faces runs at the original size (use_origin_size=True)')
        img = cuda_u8_image(image, next(self.parameters()).device, 'RetinaFace.detect_faces')
        self.resize = 1
        h, w = int(img.shape[0]), int(img.shape[1])
        loc, conf, landms = self.forward_u8(img.unsqueeze(0))
        cand = self.candidates(loc, conf, landms, h, w, conf_threshold)[0].cpu().numpy()
        return finish_detections(cand, conf_threshold, nms_threshold)


def init_detection_model(model_name='retinaface_resnet50', half=False, device='cuda', model_path=None):
    """``facelib.detection.init_detection_model`` (facelib/detection/__init__.py:13-71) without the download: pass the
    checkpoint path (``detection_Resnet50_Final.pth`` / ``yolov5l-face.pth``) or load the state dict yourself.
    RetinaFace: ``module.`` prefixes are stripped.  YOLOv5l: a ``YoloDetector`` whose ``.detector`` loads strictly, as is."""
    if model_name == 'YOLOv5l':
        from .yolov5face import YoloDetector
        model = YoloDetector(config_name='facelib/detection/yolov5face/models/yolov5l.yaml', device=device)
        if model_path is not None:
            model.detector.load_state_dict(torch.load(model_path, map_location='cpu'), strict=True)
        model.detector = model.detector.eval().to(device)
        return model
    if model_name != 'retinaface_resnet50':
        raise NotImplementedError(f'{model_name} is not built (codeformer_b200 builds retinaface_resnet50 and YOLOv5l)')
    model = RetinaFace(network_name='resnet50', half=half)
    if model_path is not None:
        load_net = torch.load(model_path, map_location='cpu')
        load_net = OrderedDict((k[7:] if k.startswith('module.') else k, v) for k, v in load_net.items())
        model.load_state_dict(load_net, strict=True)
    return model.eval().to(device)
