"""CPU checks of the FID oracle (oracle/fid_oracle.py) and of the package's host-side FID pieces: the restated network against
the patched torchvision model bit for bit, the wrapper's state-dict layout, the torchvision-name mapping and BasicSR's
calculate_fid."""
import numpy as np
import pytest
import torch

from oracle import fid_oracle as fo
from codeformer_b200 import fid


@pytest.fixture(scope='module')
def sd():
    return fo.random_fid_state_dict(1)


@pytest.mark.parametrize('size,resize', [((299, 299), False), ((512, 512), True), ((64, 96), True)])
def test_oracle_forward_equals_reference_model(sd, size, resize):
    torch.manual_seed(0)
    x = torch.rand(2, 3, *size)
    with torch.no_grad():
        ref = fo.reference_model(sd, resize_input=resize)(x)[0]
        got = fo.forward(sd, x, resize_input=resize)
    assert ref.shape == (2, 2048, 1, 1)
    assert torch.equal(ref, got)
    # activations of order 1 after all 94 ReLU convs
    assert 0.05 < ref.abs().mean().item() < 20


def test_counts():
    convs = fid.inception_convs()
    assert len(convs) == 94
    assert len(fo.torchvision_model().state_dict()) == 566      # with fc.* and the BatchNorm counters


def test_state_dict_layout(sd):
    assert list(fid.fid_inception_spec().keys()) == list(fo.reference_model().state_dict().keys())
    for k, (shape, dtype) in fid.fid_inception_spec().items():
        assert tuple(sd[k].shape) == tuple(shape) and sd[k].dtype == dtype, k


def test_load_torchvision_names(sd):
    net = fid.InceptionV3()
    net.load_fid_inception_weights(fo.torchvision_names(sd))
    ref = fo.reference_model(sd).state_dict()
    got = net.state_dict()
    assert set(got) == set(ref)
    for k in ref:
        assert torch.equal(got[k].cpu(), ref[k]), k


def test_constructor_errors():
    with pytest.raises(NotImplementedError):
        fid.InceptionV3(output_blocks=(0,))
    with pytest.raises(NotImplementedError):
        fid.InceptionV3(output_blocks=(2, 3))
    with pytest.raises(NotImplementedError):
        fid.InceptionV3(use_fid_inception=False)
    with pytest.raises(NotImplementedError):
        fid.InceptionV3(requires_grad=True)


def test_calculate_fid_diagonal():
    rng = np.random.default_rng(0)
    d = 64
    mu1, mu2 = rng.normal(size=d), rng.normal(size=d)
    a, b = rng.uniform(0.1, 2, d), rng.uniform(0.1, 2, d)
    closed = np.sum((mu1 - mu2) ** 2) + np.sum(a) + np.sum(b) - 2 * np.sum(np.sqrt(a * b))
    got = fid.calculate_fid(mu1, np.diag(a), mu2, np.diag(b))
    assert abs(got - closed) <= 1e-10 * max(1.0, abs(closed))


def test_calculate_fid_eps_retry(monkeypatch, capsys):
    calls = []
    real = fid._sqrtm

    def flaky(m):
        calls.append(m.copy())
        if len(calls) == 1:
            return np.full_like(m, np.nan)
        return real(m)
    monkeypatch.setattr(fid, '_sqrtm', flaky)
    s = np.diag([1.0, 2.0, 3.0])
    got = fid.calculate_fid(np.zeros(3), s, np.zeros(3), s, eps=1e-6)
    assert len(calls) == 2
    assert np.allclose(calls[1], (s + 1e-6 * np.eye(3)) @ (s + 1e-6 * np.eye(3)))
    assert abs(got - (2 * 6 - 2 * np.sum(np.diag(s) + 1e-6))) < 1e-9
    assert 'singular' in capsys.readouterr().out


def test_calculate_fid_imaginary_raises(monkeypatch):
    monkeypatch.setattr(fid, '_sqrtm', lambda m: np.eye(m.shape[0]) * (1 + 0.1j))
    with pytest.raises(ValueError, match='Imaginary component'):
        fid.calculate_fid(np.zeros(2), np.eye(2), np.zeros(2), np.eye(2))
    # a small imaginary part is dropped
    monkeypatch.setattr(fid, '_sqrtm', lambda m: np.eye(m.shape[0]) * (1 + 1e-5j))
    assert abs(fid.calculate_fid(np.zeros(2), np.eye(2), np.zeros(2), np.eye(2))) < 1e-12
