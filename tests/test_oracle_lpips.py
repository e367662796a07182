"""not gpu: the LPIPS-VGG restatement (oracle/lpips_oracle.py) against torchvision's VGG-16 and the UNMODIFIED reference
LPIPSLoss (basicsr/losses/losses.py; skips without the reference tree), the state-dict layout, the uint8 convention tables
of the C host code, and the module's CPU-side behaviour (loading, constructor errors)."""
import ctypes
import functools
import os
import sys
import types

import numpy as np
import pytest
import torch
import torchvision

from codeformer_b200 import _lib
from codeformer_b200 import lpips as LP
from oracle import lpips_oracle as LO
from oracle import ref_shim


def test_backbone_equals_torchvision_slices():
    sd = LO.random_lpips_state_dict(3)
    lp = LO.LPIPS()
    lp.load_state_dict(sd, strict=True)
    features = torchvision.models.vgg16(weights=None).features
    features.load_state_dict({k.split('.', 2)[2]: v for k, v in sd.items() if k.startswith('net.')}, strict=True)
    x = torch.randn(2, 3, 48, 40, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        outs = lp.net(x)
        ref, h = [], x
        for i, layer in enumerate(features):
            h = layer(h)
            if i in (3, 8, 15, 22, 29):
                ref.append(h)
    assert [tuple(o.shape[1:2]) for o in outs] == [(c,) for c in LO.CHANNELS]
    for a, b in zip(outs, ref):
        assert torch.equal(a, b)


def test_spec_matches_oracle_state_dict():
    spec = LP.lpips_spec()
    sd = LO.LPIPS().state_dict()
    assert list(spec) == list(sd)
    for k, (shape, dtype) in spec.items():
        assert tuple(sd[k].shape) == shape and sd[k].dtype == dtype, k
    assert len(spec) == 2 + 26 + 10
    # the package module has the same state dict, lins sharing lin0..4
    net = LP.LPIPS()
    nsd = net.state_dict()
    assert list(nsd) == list(spec)
    assert nsd['lins.3.model.1.weight'].data_ptr() == nsd['lin3.model.1.weight'].data_ptr()


def test_loading():
    sd = LO.random_lpips_state_dict(2)
    net = LP.LPIPS()
    net.load_state_dict(sd, strict=True)
    assert torch.equal(net.state_dict()['net.slice4.19.weight'], sd['net.slice4.19.weight'])
    # the lpips weight file holds the lin keys only; lpips loads it with strict=False
    lin_only = {k: torch.full_like(v, 0.5) for k, v in sd.items() if k.startswith('lin') and not k.startswith('lins')}
    missing, unexpected = net.load_state_dict(lin_only, strict=False)
    assert not unexpected and all(k.startswith(('net.', 'scaling_layer.', 'lins.')) for k in missing)
    assert torch.equal(net.state_dict()['lins.4.model.1.weight'], torch.full((1, 512, 1, 1), 0.5))
    # torchvision's vgg16 layout (features.N.*, classifier.*) onto net.slice*
    tv = {f'features.{idx}.{leaf}': torch.randn(cout, cin, 3, 3) if leaf == 'weight' else torch.randn(cout)
          for idx, cin, cout in LP.VGG16_CONVS for leaf in ('weight', 'bias')}
    tv['classifier.0.weight'] = torch.zeros(1)
    net.load_vgg16_features(tv)
    assert torch.equal(net.state_dict()['net.slice3.14.bias'], tv['features.14.bias'])
    assert torch.equal(net.state_dict()['net.slice1.0.weight'], tv['features.0.weight'])


def test_model_path(tmp_path):
    sd = LO.random_lpips_state_dict(4)
    p = tmp_path / 'vgg.pth'
    torch.save({k: v for k, v in sd.items() if k.startswith('lin') and not k.startswith('lins')}, p)
    net = LP.LPIPS(model_path=str(p))
    assert torch.equal(net.state_dict()['lin1.model.1.weight'], sd['lin1.model.1.weight'])


@pytest.mark.parametrize('kw', [{'net': 'alex'}, {'net': 'squeeze'}, {'version': '0.0'}, {'lpips': False}, {'spatial': True}])
def test_unsupported_forms_raise(kw):
    with pytest.raises(NotImplementedError):
        LP.LPIPS(**kw)


def test_cpu_input_raises():
    net = LP.LPIPS()
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        net(torch.zeros(1, 3, 32, 32), torch.zeros(1, 3, 32, 32))


@pytest.mark.parametrize('convention', ['lpips', 'codeformer'])
def test_u8_tables(convention):
    """The host tables (cfb_lpips_u8_table) equal the convention's chain on all 256 byte values, bit for bit."""
    table = np.zeros((3, 256), np.float32)
    shift = np.array(LO.SHIFT, np.float32)
    scale = np.array(LO.SCALE, np.float32)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)       # noqa: E731
    assert _lib.load().cfb_lpips_u8_table(LP.CONVENTIONS[convention], vp(shift), vp(scale), vp(table)) == 0
    ref = LO.u8_table(convention).numpy()
    assert np.array_equal(table.view(np.uint32), ref.view(np.uint32))
    assert _lib.load().cfb_lpips_u8_table(7, vp(shift), vp(scale), vp(table)) != 0


def test_u8_chains():
    """The conventions restate their sources: 'lpips' is im2tensor of the RGB image, 'codeformer' the training tensor
    through LPIPSLoss(use_input_norm=True, range_norm=True)."""
    rng = np.random.default_rng(0)
    bgr = rng.integers(0, 256, (5, 7, 3)).astype(np.uint8)
    x = LO.input_tensor(bgr, 'lpips')
    assert torch.equal(x, (torch.from_numpy(bgr[:, :, ::-1].astype(np.float64).copy()).permute(2, 0, 1)[None] / 127.5 - 1).float())
    y = LO.input_tensor(bgr, 'codeformer')
    assert float(y.min()) >= -1 and float(y.max()) <= 1 and y.dtype == torch.float32


@functools.lru_cache(maxsize=None)
def _reference_lpips_loss():
    """The reference's LPIPSLoss, imported unmodified with a stub ``lpips`` module whose ``LPIPS`` is the restatement;
    sys.modules is restored afterwards."""
    saved = dict(sys.modules)
    try:
        ref_shim.load()
        stub = types.ModuleType('lpips')
        stub.LPIPS = LO.LPIPS
        sys.modules['lpips'] = stub
        pkg = types.ModuleType('basicsr.losses')
        pkg.__path__ = [os.path.join(ref_shim.REF_ROOT, 'basicsr', 'losses')]
        sys.modules['basicsr.losses'] = pkg
        from basicsr.losses.losses import LPIPSLoss
        return LPIPSLoss
    finally:
        for k in [k for k in sys.modules if k not in saved]:
            del sys.modules[k]
        sys.modules.update(saved)


@pytest.mark.parametrize('range_norm', [False, True])
@pytest.mark.parametrize('use_input_norm', [False, True])
def test_reference_lpips_loss_equals_oracle(range_norm, use_input_norm):
    if not ref_shim.available():
        pytest.skip('reference tree not available')
    RefLoss = _reference_lpips_loss()
    sd = LO.random_lpips_state_dict(6)
    torch.manual_seed(0)
    ref = RefLoss(loss_weight=0.7, use_input_norm=use_input_norm, range_norm=range_norm)
    ref.perceptual.load_state_dict(sd, strict=True)
    ours = LO.LPIPSLoss(loss_weight=0.7, use_input_norm=use_input_norm, range_norm=range_norm)
    ours.perceptual.load_state_dict(sd, strict=True)
    assert list(ref.state_dict()) == list(ours.state_dict())
    g = torch.Generator().manual_seed(7)
    pred = torch.rand(2, 3, 32, 40, generator=g) * 2 - 1
    target = (pred + 0.3 * torch.randn(2, 3, 32, 40, generator=g)).clamp(-1, 1)
    with torch.no_grad():
        a, b = ref(pred, target), ours(pred, target)
    assert torch.equal(a, b) and float(a) > 0
