"""CPU checks of tests/parsenet_fp16_emul.py, the float64 model of ParseNet in its fp16 precision that the GPU tests compare
against: without rounding it is the reference network (the CPU oracle), its conv is fp16_emul's conv on any device, and
with rounding it stays inside the fp16 error one expects of it."""
import pytest
import torch
import torch.nn.functional as F

from codeformer_b200 import parsing as P
from oracle import parsenet_oracle as PO
from tests import fp16_emul as E
from tests import parsenet_fp16_emul as PE

torch.set_grad_enabled(False)


def _rel(a, b):
    return float((a.double() - b.double()).abs().max()) / float(b.double().abs().max())


@pytest.mark.parametrize('size,batch', [(64, 2), (128, 1)])
def test_without_rounding_equals_the_oracle(size, batch):
    sd = P.random_parsenet_state_dict(P.parsenet_spec(size, size), 7)
    plan = P.parsenet_plan(size, size)[0]
    x = torch.rand(batch, 3, size, size, generator=torch.Generator().manual_seed(3)) * 2 - 1
    ref_m, ref_i = PO.parsenet_forward(sd, x, plan)
    got_m, got_i = PE.parsenet_forward(sd, x, plan, rounding=False, return_img=True)
    print(f'{size}: logits rel {_rel(got_m, ref_m):.2e}, img rel {_rel(got_i, ref_i):.2e}')
    assert got_m.shape == ref_m.shape and _rel(got_m, ref_m) < 1e-5 and _rel(got_i, ref_i) < 1e-5
    # with rounding the result moves, by about what fp16 operands cost over this depth
    r = _rel(PE.parsenet_forward(sd, x, plan), ref_m)
    print(f'{size}: fp16 emulation rel {r:.2e}')
    assert 1e-6 < r < 5e-2


@pytest.mark.parametrize('form', [dict(pad_mode=1), dict(pad_mode=1, sub=True), dict(pad_mode=2, up=True),
                                  dict(pad_mode=0, up=True)])
def test_conv_is_fp16_emul_conv(form):
    """The device-agnostic conv equals fp16_emul.conv3x3 bit for bit on the host (same roundings, same float64 ops)."""
    x = torch.randn(2, 64, 10, 14, generator=torch.Generator().manual_seed(1)) * 2
    w = torch.randn(32, 64, 3, 3, generator=torch.Generator().manual_seed(2)) / 24
    assert torch.equal(PE.conv3x3(x, w, **form), E.conv3x3(x, w, **form))
    ex = PE.conv3x3(x, w, rounding=False, **form)
    xi = F.interpolate(x.double(), scale_factor=2, mode='nearest') if form.get('up') else x.double()
    mode = 'constant' if form['pad_mode'] == 0 else 'reflect'
    ref = F.conv2d(F.pad(xi, (1, 1, 1, 1), mode=mode), w.double())
    assert torch.allclose(ex, ref[..., ::2, ::2] if form.get('sub') else ref, rtol=0, atol=1e-12)


def test_bn_fold_is_fp32_and_equals_batchnorm():
    sd = P.random_parsenet_state_dict(P.parsenet_spec(64, 64), 2)
    w, b = PE.fold_bn(sd, 'body.0.conv1')
    assert w.dtype == torch.float32 and b.dtype == torch.float32
    x = torch.randn(1, w.shape[1], 6, 6, generator=torch.Generator().manual_seed(4))
    q = 'body.0.conv1.norm.norm.'
    ref = F.batch_norm(F.conv2d(x, sd['body.0.conv1.conv2d.weight']), sd[q + 'running_mean'], sd[q + 'running_var'],
                       sd[q + 'weight'], sd[q + 'bias'], training=False, eps=1e-5)
    assert torch.allclose(F.conv2d(x, w, b), ref, rtol=1e-5, atol=1e-5)
