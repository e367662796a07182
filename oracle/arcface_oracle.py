"""torch fp32 restatement (CPU) of ResNetArcFace('IRBlock', layers, use_se=False) and of gray_resize_for_identity.

Functional, from a state dict: /root/reference/basicsr/archs/arcface_arch.py:56-100 (IRBlock.forward), 229-245
(ResNetArcFace.forward), and the three lines of basicsr/models/codeformer_model.py:131-135 (importing that module pulls in
the training dependencies).  tests/test_oracle_arcface.py pins it bit for bit against the unmodified reference class.
"""
import torch
import torch.nn.functional as F


def gray_resize_for_identity(out, size=128):
    out_gray = (0.2989 * out[:, 0, :, :] + 0.5870 * out[:, 1, :, :] + 0.1140 * out[:, 2, :, :])
    out_gray = out_gray.unsqueeze(1)
    return F.interpolate(out_gray, (size, size), mode='bilinear', align_corners=False)


def faces_to_input(faces_bgr_u8):
    """uint8 HWC BGR faces [N,512,512,3] (numpy or torch) -> the normalised RGB tensor [N,3,512,512] of the caller
    (img2tensor(face / 255., bgr2rgb=True, float32=True) + normalize(0.5, 0.5))."""
    t = torch.as_tensor(faces_bgr_u8)
    x = (t.double() / 255.).float().flip(-1).permute(0, 3, 1, 2).contiguous()
    return (x - 0.5) / 0.5


def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + '.running_mean'], sd[p + '.running_var'], sd[p + '.weight'], sd[p + '.bias'], False, 0.0, 1e-5)


def arcface_forward(sd, x, layers=(2, 2, 2, 2)):
    """x fp32 [B,1,128,128] -> embeddings [B,512] (eval mode: BatchNorm on running statistics, dropout off)."""
    x = F.conv2d(x, sd['conv1.weight'], padding=1)
    x = F.prelu(_bn(x, sd, 'bn1'), sd['prelu.weight'])
    x = F.max_pool2d(x, 2, 2)
    for li, nb in enumerate(layers):
        for b in range(nb):
            p = f'layer{li + 1}.{b}'
            stride = 2 if (b == 0 and li > 0) else 1
            residual = x
            out = F.conv2d(_bn(x, sd, p + '.bn0'), sd[p + '.conv1.weight'], padding=1)
            out = F.prelu(_bn(out, sd, p + '.bn1'), sd[p + '.prelu.weight'])
            out = _bn(F.conv2d(out, sd[p + '.conv2.weight'], stride=stride, padding=1), sd, p + '.bn2')
            if p + '.downsample.0.weight' in sd:
                residual = _bn(F.conv2d(x, sd[p + '.downsample.0.weight'], stride=stride), sd, p + '.downsample.1')
            out += residual
            x = F.prelu(out, sd[p + '.prelu.weight'])
    x = _bn(x, sd, 'bn4')
    x = x.view(x.size(0), -1)
    x = F.linear(x, sd['fc5.weight'], sd['fc5.bias'])
    return F.batch_norm(x, sd['bn5.running_mean'], sd['bn5.running_var'], sd['bn5.weight'], sd['bn5.bias'], False, 0.0, 1e-5)
