"""not gpu: the RetinaFace-ResNet50 oracle against the UNMODIFIED reference class (skips without the reference tree), the numpy
NMS against torchvision's, the state-dict contract, and the FPN's nearest-neighbour index."""
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import codeformer_b200 as cb
from codeformer_b200 import detection as D
from oracle import ref_shim
from oracle import retinaface_oracle as RO

torch.set_grad_enabled(False)


def _reference_retinaface():
    """The reference's RetinaFace class with ``get_device()`` resolving to the CPU."""
    if not ref_shim.available():
        pytest.skip('reference tree not available')
    pytest.importorskip('cv2')
    pytest.importorskip('torchvision')
    R = ref_shim.REF_ROOT
    saved = {k: sys.modules.get(k) for k in ('basicsr', 'basicsr.utils', 'basicsr.utils.misc', 'facelib', 'facelib.detection',
                                             'facelib.utils')}
    sys.dont_write_bytecode = True
    if R not in sys.path:
        sys.path.insert(0, R)
    for name, path in (('basicsr', 'basicsr'), ('basicsr.utils', 'basicsr/utils'), ('facelib', 'facelib'),
                       ('facelib.detection', 'facelib/detection'), ('facelib.utils', 'facelib/utils')):
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(R, path)]
        sys.modules[name] = m
    misc = types.ModuleType('basicsr.utils.misc')
    misc.get_device = lambda: torch.device('cpu')
    sys.modules['basicsr.utils.misc'] = misc
    try:
        from facelib.detection.retinaface.retinaface import RetinaFace
        from facelib.detection.retinaface.retinaface_utils import py_cpu_nms
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return RetinaFace, py_cpu_nms


def _image(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def test_state_dict_contract():
    sd = cb.RetinaFace().state_dict()
    spec = D.retinaface_spec()
    assert len(sd) == 456 and list(sd.keys()) == list(spec.keys())
    assert all(tuple(sd[k].shape) == tuple(spec[k][0]) and sd[k].dtype == spec[k][1] for k in spec)
    cb.RetinaFace().load_state_dict(D.random_retinaface_state_dict(3), strict=True)


def test_state_dict_equals_reference():
    RetinaFace, _ = _reference_retinaface()
    ref = RetinaFace('resnet50').state_dict()
    ours = cb.RetinaFace().state_dict()
    assert list(ref.keys()) == list(ours.keys())
    assert all(ref[k].shape == ours[k].shape and ref[k].dtype == ours[k].dtype for k in ref)


@pytest.mark.parametrize('h,w', [(333, 427), (37, 50)])
def test_oracle_is_bit_identical_to_the_reference(h, w):
    RetinaFace, _ = _reference_retinaface()
    sd = D.random_retinaface_state_dict(1)
    net = RetinaFace('resnet50')
    net.load_state_dict(sd, strict=True)
    img = _image(h, w, 0)
    x = RO.input_from_u8(img)
    for a, b in zip(net(x), RO.forward(sd, x)):
        assert torch.equal(a, b)
    ref = net.detect_faces(img, 0.8, 0.4)
    ours = RO.detect_faces(sd, img, 0.8, 0.4)
    assert ref.dtype == ours.dtype == np.float32 and ref.shape == ours.shape
    assert np.array_equal(ref, ours)
    if (h, w) == (333, 427):
        assert 50 <= RO.candidates(sd, img).shape[0] <= 500 and ref.shape[0] > 0


def test_priors_equal_the_reference():
    RetinaFace, _ = _reference_retinaface()
    from facelib.detection.retinaface.retinaface_utils import PriorBox
    net = RetinaFace('resnet50')
    for h, w in [(333, 427), (37, 50), (640, 853)]:
        assert torch.equal(PriorBox(net.cfg, image_size=(h, w)).forward(), RO.priors(h, w))


def _torchvision_nms(dets, thr):
    tv = pytest.importorskip('torchvision')
    return [int(i) for i in tv.ops.nms(torch.Tensor(dets[:, :4]), torch.Tensor(dets[:, 4]), thr)]


@pytest.mark.parametrize('seed', range(6))
def test_numpy_nms_equals_torchvision(seed):
    rng = np.random.default_rng(seed)
    n = 200
    xy = rng.uniform(0, 100, (n, 2)).astype(np.float32)
    wh = rng.uniform(0, 40, (n, 2)).astype(np.float32)
    wh[rng.random(n) < 0.05] = 0                                # zero-area boxes
    boxes = np.concatenate([xy, xy + wh], 1)
    scores = np.round(rng.uniform(0.5, 1, n), 2).astype(np.float32)   # many tied scores
    dup = rng.integers(0, n, 20)
    boxes[dup[:10]] = boxes[dup[10:]]                           # duplicate boxes
    dets = np.concatenate([boxes, scores[:, None]], 1).astype(np.float32)
    for thr in (0.0, 0.3, 0.4, 0.7):
        assert D.nms(dets, thr) == _torchvision_nms(dets, thr)


def _nearest_index(out_size, in_size):
    x = torch.arange(in_size, dtype=torch.float32).view(1, 1, in_size, 1)
    return F.interpolate(x, size=[out_size, 1], mode='nearest').view(-1).long()


def test_fpn_nearest_index_is_the_halved_position():
    """For every fine/coarse pair the ceil chain produces (fine = 2*coarse or 2*coarse-1, fine up to 4096), torch's nearest
    map is y // 2; detection.cu computes torch's formula, which this pins."""
    for coarse in range(1, 2049):
        for fine in (2 * coarse - 1, 2 * coarse):
            if fine < 1 or fine > 4096:
                continue
            idx = _nearest_index(fine, coarse)
            assert torch.equal(idx, torch.arange(fine) // 2), (fine, coarse)
