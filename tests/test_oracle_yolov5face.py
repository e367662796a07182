"""not gpu: the YOLOv5l-face oracle against the UNMODIFIED reference classes (skips without the reference tree), and the
state-dict contract of codeformer_b200.YOLOv5lFace."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from codeformer_b200 import yolov5face as Y
from oracle import ref_shim
from oracle import yolov5face_oracle as YO

torch.set_grad_enabled(False)


def _reference():
    """The reference's YoloDetector class and the absolute path of models/yolov5l.yaml."""
    if not ref_shim.available():
        pytest.skip('reference tree not available')
    for m in ('cv2', 'torchvision', 'yaml'):
        pytest.importorskip(m)
    R = ref_shim.REF_ROOT
    names = ('facelib', 'facelib.detection', 'facelib.utils')
    saved = {k: sys.modules.get(k) for k in names}
    sys.dont_write_bytecode = True
    if R not in sys.path:
        sys.path.insert(0, R)
    for name in names:
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(R, *name.split('.'))]
        sys.modules[name] = m
    try:
        from facelib.detection.yolov5face.face_detector import YoloDetector
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return YoloDetector, os.path.join(R, 'facelib', 'detection', 'yolov5face', 'models', 'yolov5l.yaml')


def _detector(sd=None, **kw):
    YoloDetector, cfg = _reference()
    det = YoloDetector(config_name=cfg, device='cpu', **kw)
    if sd is not None:
        det.detector.load_state_dict(sd, strict=True)
    det.detector.eval()
    return det


def _image(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def test_state_dict_contract():
    sd = Y.YOLOv5lFace().state_dict()
    spec = Y.yolov5l_spec()
    assert len(sd) == 662 and list(sd.keys()) == list(spec.keys())
    assert all(tuple(sd[k].shape) == tuple(spec[k][0]) and sd[k].dtype == spec[k][1] for k in spec)
    Y.YOLOv5lFace().load_state_dict(Y.random_yolov5l_state_dict(3), strict=True)
    assert Y.YOLOv5lFace().stride.tolist() == [8., 16., 32.]


def test_state_dict_equals_reference():
    det = _detector()
    ref = det.detector.state_dict()
    ours = Y.YOLOv5lFace().state_dict()
    assert list(ref.keys()) == list(ours.keys())
    assert all(ref[k].shape == ours[k].shape and ref[k].dtype == ours[k].dtype for k in ref)
    assert torch.equal(ref['model.23.anchor_grid'], ours['model.23.anchor_grid'])
    assert torch.equal(ref['model.23.anchors'], ours['model.23.anchors'])
    assert det.detector.stride.tolist() == Y.YOLOv5lFace().stride.tolist()
    Y.YOLOv5lFace().load_state_dict(ref, strict=True)
    det.detector.load_state_dict(ours, strict=True)


@pytest.mark.parametrize('h,w', [(160, 224), (352, 480)])
def test_oracle_forward_is_bit_identical_to_the_reference(h, w):
    sd = Y.random_yolov5l_state_dict(1)
    det = _detector(sd)
    x = torch.rand(1, 3, h, w, generator=torch.Generator().manual_seed(h))
    pred, raws = det.detector(x)
    opred, oraws = YO.forward(sd, x)
    assert pred.shape == (1, Y.predictions(h, w), 16)
    assert torch.equal(pred, opred)
    assert len(raws) == 3 and all(torch.equal(a, b) for a, b in zip(raws, oraws))


@pytest.mark.parametrize('h,w,target', [(640, 853, None), (256, 384, None), (600, 801, 480)])
def test_oracle_preprocess_is_bit_identical(h, w, target):
    """letterbox upscale (640x853 -> 672x864), an exact multiple of 32, and a target_size downscale before the letterbox."""
    import cv2
    det = _detector(target_size=target)
    imgs = [_image(h, w, 1), _image(h, w, 2)]
    ref = det._preprocess([cv2.cvtColor(im, cv2.COLOR_BGR2RGB) for im in imgs])
    ours = YO.preprocess(imgs, target)
    assert ref.dtype == ours.dtype == torch.float32 and torch.equal(ref, ours)
    first, second, canvas, _ = Y.letterbox_geometry(h, w, target)
    assert tuple(ours.shape[2:]) == canvas
    if (h, w) == (640, 853):
        assert canvas == (672, 864)


def test_oracle_detect_faces_equals_the_reference():
    sd = Y.random_yolov5l_state_dict(1)
    det = _detector(sd)
    img = _image(333, 427, 0)
    ref = det.detect_faces(img)
    ours = YO.detect_faces(sd, img)
    assert isinstance(ref, np.ndarray) and ref.dtype == np.int64 and ref.shape[0] > 0
    assert ours.dtype == np.int64 and np.array_equal(ref, ours)
    assert det.detect_faces(img, conf_thres=0.999) is None and YO.detect_faces(sd, img, conf_thres=0.999) is None
