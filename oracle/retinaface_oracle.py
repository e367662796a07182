"""RetinaFace-ResNet50 restated op for op on the CPU in fp32 (torch), from a state dict.

Reference: /root/reference/facelib/detection/retinaface/retinaface.py (forward :122-145, detect_faces :194-239),
retinaface_net.py (FPN, SSH, heads), retinaface_utils.py (PriorBox, decode, decode_landm, py_cpu_nms) and torchvision's
resnet50 (conv1 .. layer4).  tests/test_oracle_detection.py checks it bit for bit against the unmodified reference class.
"""
from itertools import product
from math import ceil

import numpy as np
import torch
import torch.nn.functional as F

from codeformer_b200.detection import RESNET50_BLOCKS, finish_detections

MEAN_BGR = (104., 117., 123.)
MIN_SIZES = [[16, 32], [64, 128], [256, 512]]
STEPS = [8, 16, 32]
VARIANCE = [0.1, 0.2]


def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + '.running_mean'], sd[p + '.running_var'], sd[p + '.weight'], sd[p + '.bias'], False, 0.1, 1e-5)


def _conv_bn(x, sd, p, stride=1, pad=1, act=True):
    y = _bn(F.conv2d(x, sd[p + '.0.weight'], None, stride, pad), sd, p + '.1')
    return F.leaky_relu(y, 0.) if act else y


def body(sd, x):
    """torchvision resnet50 conv1 .. layer4; returns the outputs of layer2, layer3, layer4."""
    x = F.relu(_bn(F.conv2d(x, sd['body.conv1.weight'], None, 2, 3), sd, 'body.bn1'))
    x = F.max_pool2d(x, 3, 2, 1)
    outs = []
    for li, nb in enumerate(RESNET50_BLOCKS):
        for b in range(nb):
            p = f'body.layer{li + 1}.{b}.'
            s = 2 if (b == 0 and li > 0) else 1
            y = F.relu(_bn(F.conv2d(x, sd[p + 'conv1.weight']), sd, p + 'bn1'))
            y = F.relu(_bn(F.conv2d(y, sd[p + 'conv2.weight'], None, s, 1), sd, p + 'bn2'))
            y = _bn(F.conv2d(y, sd[p + 'conv3.weight']), sd, p + 'bn3')
            idt = _bn(F.conv2d(x, sd[p + 'downsample.0.weight'], None, s), sd, p + 'downsample.1') if b == 0 else x
            x = F.relu(y + idt)
        if li >= 1:
            outs.append(x)
    return outs


def fpn(sd, feats):
    o1, o2, o3 = (_conv_bn(f, sd, f'fpn.output{k + 1}', pad=0) for k, f in enumerate(feats))
    o2 = o2 + F.interpolate(o3, size=[o2.size(2), o2.size(3)], mode='nearest')
    o2 = _conv_bn(o2, sd, 'fpn.merge2')
    o1 = o1 + F.interpolate(o2, size=[o1.size(2), o1.size(3)], mode='nearest')
    o1 = _conv_bn(o1, sd, 'fpn.merge1')
    return [o1, o2, o3]


def ssh(sd, x, p):
    c3 = _conv_bn(x, sd, p + '.conv3X3', act=False)
    c5_1 = _conv_bn(x, sd, p + '.conv5X5_1')
    c5 = _conv_bn(c5_1, sd, p + '.conv5X5_2', act=False)
    c7_2 = _conv_bn(c5_1, sd, p + '.conv7X7_2')
    c7 = _conv_bn(c7_2, sd, p + '.conv7x7_3', act=False)
    return F.relu(torch.cat([c3, c5, c7], dim=1))


def forward(sd, x):
    """x [B,3,H,W] fp32 (mean-subtracted) -> (loc [B,P,4], softmax(conf) [B,P,2], landms [B,P,10])."""
    feats = [ssh(sd, f, f'ssh{k + 1}') for k, f in enumerate(fpn(sd, body(sd, x)))]

    def head(name, k):
        outs = []
        for i, f in enumerate(feats):
            o = F.conv2d(f, sd[f'{name}.{i}.conv1x1.weight'], sd[f'{name}.{i}.conv1x1.bias'])
            outs.append(o.permute(0, 2, 3, 1).contiguous().view(o.shape[0], -1, k))
        return torch.cat(outs, dim=1)

    return head('BboxHead', 4), F.softmax(head('ClassHead', 2), dim=-1), head('LandmarkHead', 10)


def priors(h, w):
    """PriorBox(cfg_re50, image_size=(h, w)).forward(): float64 arithmetic, then float32."""
    anchors = []
    for k, step in enumerate(STEPS):
        for i, j in product(range(ceil(h / step)), range(ceil(w / step))):
            for m in MIN_SIZES[k]:
                anchors += [(j + 0.5) * step / w, (i + 0.5) * step / h, m / w, m / h]
    return torch.Tensor(anchors).view(-1, 4)


def decode(loc, pri):
    boxes = torch.cat((pri[:, :2] + loc[:, :2] * VARIANCE[0] * pri[:, 2:], pri[:, 2:] * torch.exp(loc[:, 2:] * VARIANCE[1])), 1)
    boxes[:, :2] -= boxes[:, 2:] / 2
    boxes[:, 2:] += boxes[:, :2]
    return boxes


def decode_landm(pre, pri):
    return torch.cat([pri[:, :2] + pre[:, 2 * j:2 * j + 2] * VARIANCE[0] * pri[:, 2:] for j in range(5)], dim=1)


def input_from_u8(img):
    """uint8 HWC BGR -> the mean-subtracted [1,3,H,W] fp32 tensor detect_faces feeds the network."""
    x = torch.from_numpy(img.astype(np.float32).transpose(2, 0, 1)).unsqueeze(0)
    return x - torch.tensor(MEAN_BGR).view(1, 3, 1, 1)


def candidates(sd, img, conf_threshold=0.8, outputs=None):
    """Rows [box(4), score, landmarks(10)] of the priors with score > conf_threshold, in prior order."""
    h, w = img.shape[:2]
    loc, conf, landms = outputs if outputs is not None else forward(sd, input_from_u8(img))
    pri = priors(h, w)
    scale = torch.tensor([w, h, w, h], dtype=torch.float32)
    scale1 = torch.tensor([w, h] * 5, dtype=torch.float32)
    boxes = (decode(loc.squeeze(0), pri) * scale / 1).numpy()
    scores = conf.squeeze(0).numpy()[:, 1]
    lms = (decode_landm(landms.squeeze(0), pri) * scale1 / 1).numpy()
    inds = np.where(scores > conf_threshold)[0]
    return np.concatenate((boxes[inds], scores[inds, None], lms[inds]), axis=1).astype(np.float32)


def detect_faces(sd, img, conf_threshold=0.8, nms_threshold=0.4):
    return finish_detections(candidates(sd, img, conf_threshold), conf_threshold, nms_threshold)
