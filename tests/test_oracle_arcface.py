"""not gpu: the ResNetArcFace oracle against the UNMODIFIED reference class (skips without the reference tree), the golden
embeddings, the state-dict contract and the constructor's errors."""
import os

import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import arcface as A
from oracle import arcface_oracle as AO
from oracle import gen_golden_arcface as G
from oracle import ref_shim

torch.set_grad_enabled(False)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'arcface.npz')


def _reference_class():
    if not ref_shim.available():
        pytest.skip('reference tree not available')
    ref_shim.load()                       # seeds the basicsr namespaces; arcface_arch imports as is
    from basicsr.archs.arcface_arch import ResNetArcFace
    return ResNetArcFace


@pytest.mark.parametrize('layers', [(2, 2, 2, 2), (1, 2, 3, 1)])
def test_oracle_matches_reference_bit_for_bit(layers):
    Ref = _reference_class()
    ref = Ref('IRBlock', list(layers), use_se=False).eval()
    sd = A.random_arcface_state_dict(layers, seed=3)
    ref.load_state_dict(sd, strict=True)
    assert list(ref.state_dict().keys()) == list(A.arcface_spec(layers).keys())
    assert all(tuple(v.shape) == A.arcface_spec(layers)[k][0] for k, v in ref.state_dict().items())
    x = G.inputs()[:3]
    assert torch.equal(AO.arcface_forward(sd, x, layers), ref(x))


def test_state_dict_contract():
    net = cb.ResNetArcFace('IRBlock', [2, 2, 2, 2], use_se=False)
    sd = net.state_dict()
    assert len(sd) == 181
    assert list(sd.keys()) == list(A.arcface_spec().keys())
    assert sd['layer2.0.downsample.0.weight'].shape == (128, 64, 1, 1) and 'layer1.0.downsample.0.weight' not in sd
    assert sd['fc5.weight'].shape == (512, 32768) and sd['bn5.num_batches_tracked'].dtype == torch.int64
    net.load_state_dict(A.random_arcface_state_dict(), strict=True)
    assert cb.ARCH_REGISTRY.get('ResNetArcFace') is cb.ResNetArcFace


def test_reference_default_init_keys_load_strictly():
    Ref = _reference_class()
    ref_sd = Ref('IRBlock', [2, 2, 2, 2], use_se=False).state_dict()
    net = cb.ResNetArcFace(layers=[2, 2, 2, 2], use_se=False)
    net.load_state_dict(ref_sd, strict=True)
    assert all(torch.equal(net.state_dict()[k], v) for k, v in ref_sd.items())


def test_golden_reproduces():
    g = np.load(GOLDEN)
    emb = AO.arcface_forward(A.random_arcface_state_dict(seed=1), G.inputs())
    assert float((emb - torch.from_numpy(g['emb'])).abs().max()) < 1e-5


def test_gray_resize_restatement_is_the_reference_arithmetic():
    """The 4x bilinear resize of gray_resize_for_identity averages rows / columns 4y+1 and 4y+2 with weights 0.5."""
    faces = np.load(os.path.join(os.path.dirname(GOLDEN), 'faces.npz'))['faces'][:1]
    x = AO.faces_to_input(faces)
    gray = 0.2989 * x[:, 0] + 0.5870 * x[:, 1] + 0.1140 * x[:, 2]
    want = 0.5 * (0.5 * gray[:, 1::4, 1::4] + 0.5 * gray[:, 1::4, 2::4]) + 0.5 * (0.5 * gray[:, 2::4, 1::4] + 0.5 * gray[:, 2::4, 2::4])
    assert torch.equal(AO.gray_resize_for_identity(x)[:, 0], want)


def test_constructor_errors():
    with pytest.raises(NotImplementedError):
        cb.ResNetArcFace('IRBlock', [2, 2, 2, 2])                 # use_se=True, the reference's default
    with pytest.raises(NotImplementedError):
        cb.ResNetArcFace('BasicBlock', [2, 2, 2, 2], use_se=False)
    with pytest.raises(ValueError):
        cb.ResNetArcFace('IRBlock', [2, 2, 0, 2], use_se=False)
    net = cb.ResNetArcFace('IRBlock', [2, 2, 2, 2], use_se=False)
    with pytest.raises(RuntimeError):
        net.train()
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 1, 128, 128))                         # CPU input: no fallback
