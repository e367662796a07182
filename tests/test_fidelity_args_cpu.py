"""The fidelity-weight argument of the CodeFormer forwards (``codeformer_b200.arch.fidelity_weights``), without a GPU: what is a
scalar (today's path, a float), what is one weight per face (a float32 tensor), and what is refused."""
import numpy as np
import pytest
import torch

from codeformer_b200.arch import fidelity_weights


@pytest.mark.parametrize('w', [0.5, 0, 1, -0.25, float('nan'), np.float32(0.7), np.float64(0.3), np.array(0.5),
                               torch.tensor(0.25), torch.tensor(1.0, dtype=torch.float64), '0.5'])
def test_scalars_stay_floats(w):
    r = fidelity_weights(w, 3)
    assert type(r) is float
    assert np.isnan(r) if isinstance(w, float) and np.isnan(w) else r == float(w)


@pytest.mark.parametrize('w', [[0.5, 0.0, -1.0], (0.5, 0, 1), np.array([0.5, 0.0, 1.0]), np.array([0.5, 0.0, 1.0], np.float32),
                               np.array([0.5, 0.0, 1.0], np.float16), torch.tensor([0.5, 0.0, 1.0]),
                               torch.tensor([0.5, 0.0, 1.0], dtype=torch.float64), torch.tensor([0.5, 0.0, 1.0, 9.0])[:3],
                               torch.tensor([0.5, 9.0, 0.0, 9.0, 1.0])[::2], torch.tensor([0.5, 0.0, 1.0], requires_grad=True)])
def test_vectors_become_float32(w):
    r = fidelity_weights(w, 3)
    assert torch.is_tensor(r) and r.dtype == torch.float32 and r.shape == (3,) and r.is_contiguous() and not r.requires_grad
    expect = torch.tensor([float(v) for v in (w.detach() if torch.is_tensor(w) else w)], dtype=torch.float32)
    assert torch.equal(r, expect)


def test_values_round_as_the_scalar_path():
    """A per-face value reaches the kernel as the float32 nearest to it, as a scalar w does through ctypes.c_float."""
    import ctypes
    vals = [0.1, 1 / 3, 0.7, 2 ** -30, 0.30000000000000004]
    r = fidelity_weights(vals, len(vals))
    assert [float(v) for v in r] == [ctypes.c_float(v).value for v in vals]


def test_nan_and_negative_pass_through():
    r = fidelity_weights([float('nan'), -2.0, 0.0], 3)
    assert np.isnan(float(r[0])) and float(r[1]) == -2.0 and float(r[2]) == 0.0


def test_empty_batch():
    r = fidelity_weights([], 0)
    assert torch.is_tensor(r) and r.shape == (0,)


@pytest.mark.parametrize('w,n', [([0.5, 0.5], 3), (np.zeros(4), 3), (torch.zeros(2), 3), (torch.zeros(3, 1), 3),
                                 (np.zeros((1, 3)), 3), ([0.5], 2)])
def test_wrong_length_or_shape(w, n):
    with pytest.raises(RuntimeError, match='one fidelity weight per face'):
        fidelity_weights(w, n)


@pytest.mark.parametrize('w', [np.array([1, 0, 1]), np.array([True, False, True]), torch.tensor([1, 0, 1]),
                               torch.tensor([True, False, True]), np.array(['a', 'b', 'c']), ['a', 'b', 'c'],
                               torch.tensor([1, 0, 1], dtype=torch.uint8)])
def test_non_float_dtypes(w):
    with pytest.raises(ValueError):
        fidelity_weights(w, 3)
