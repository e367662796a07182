"""not gpu: the BiSeNet oracle against the UNMODIFIED reference class (skips without the reference tree), the state-dict
contract, and the seeded weights the GPU tests run (several classes and both mask values on a fixture face)."""
import os
import sys
import types

import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import bisenet as BS
from oracle import bisenet_oracle as BO
from oracle import ref_shim
from tests.util import golden

torch.set_grad_enabled(False)
MASK_COLORMAP = [0, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 0, 255, 0, 0, 0]


def _reference_bisenet():
    """The reference's BiSeNet class, imported without the package __init__ (which downloads weights)."""
    if not ref_shim.available():
        pytest.skip('reference tree not available')
    R = ref_shim.REF_ROOT
    saved = {k: sys.modules.get(k) for k in ('facelib', 'facelib.parsing')}
    sys.dont_write_bytecode = True
    for name, path in (('facelib', 'facelib'), ('facelib.parsing', 'facelib/parsing')):
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(R, path)]
        sys.modules[name] = m
    try:
        from facelib.parsing.bisenet import BiSeNet
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return BiSeNet


def face_input(n=2, hw=(512, 512)):
    """The normalised input (RGB, (x/255 - 0.5)/0.5) of the first n fixture faces, cropped to hw."""
    f = golden('faces.npz')['faces'][:n, :hw[0], :hw[1]]
    x = torch.from_numpy(np.ascontiguousarray(f.astype(np.float32) / 255.)).permute(0, 3, 1, 2).contiguous()
    return (x - 0.5) / 0.5


def test_state_dict_contract():
    net = cb.BiSeNet(num_class=19)
    sd = net.state_dict()
    spec = BS.bisenet_spec(19)
    assert len(sd) == 191 and list(sd.keys()) == list(spec.keys())
    assert all(tuple(sd[k].shape) == tuple(spec[k][0]) and sd[k].dtype == spec[k][1] for k in spec)
    assert sum(p.numel() for p in net.parameters()) == 13_300_416
    net.load_state_dict(BO.random_bisenet_state_dict(3), strict=True)


def test_state_dict_equals_reference():
    BiSeNet = _reference_bisenet()
    ref = BiSeNet(num_class=19).state_dict()
    ours = cb.BiSeNet(num_class=19).state_dict()
    assert list(ref.keys()) == list(ours.keys())
    assert all(ref[k].shape == ours[k].shape and ref[k].dtype == ours[k].dtype for k in ref)


@pytest.mark.parametrize('hw', [(512, 512), (96, 160)])
def test_oracle_is_bit_identical_to_the_reference(hw):
    BiSeNet = _reference_bisenet()
    sd = BO.random_bisenet_state_dict(1)
    net = BiSeNet(num_class=19).eval()
    net.load_state_dict(sd, strict=True)
    x = face_input(2, hw)
    ref = net(x)
    ours = BO.forward(sd, x)
    assert len(ref) == len(ours) == 3
    for a, b in zip(ref, ours):
        assert a.shape == (2, 19) + hw and torch.equal(a, b)


def test_seeded_weights_give_several_classes():
    sd = BO.random_bisenet_state_dict(1)
    out = BO.forward(sd, face_input(1))[0]
    cls = out.argmax(1)[0]
    share = torch.bincount(cls.flatten(), minlength=19).float() / cls.numel()
    mask = torch.tensor(MASK_COLORMAP)[cls]
    print('class shares %:', [round(float(s) * 100, 1) for s in share])
    assert int((share >= 0.01).sum()) >= 3
    assert bool((mask == 0).any()) and bool((mask == 255).any())
