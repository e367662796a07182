"""CPU model of the Transformer-stage LayerNorm (tests/layernorm_emul.py): the kernel's fp32 order of operations meets the
float64 bar of tests/test_gpu_transformer_stage.py on that test's rows, and the bar rejects by at least 4x each arithmetic
fault it is there to catch -- a one-pass variance, eps 1e-6, a mean that misses one float4.  Mutants cannot be built on the
GPU, so this file is the evidence that the GPU bar has teeth.

It also settles whether the fp32 row mean needs a fix at large r = |mean| / std: no.  Its rounding error, r * 2^-24 relative
to the row's standard deviation, is the same size as the rounding of x - mean, which every fp32 LayerNorm (torch's
included) carries; the restatement stays within 1.3x of torch at r up to 1e4."""
import numpy as np
import pytest

from tests import layernorm_emul as L

T = 3 * 256


@pytest.fixture(scope='module')
def rows():
    x, classes = L.row_classes(T, 1)
    gamma, beta = L.affine(2)
    y64, y32 = L.reference(x, gamma, beta)
    return x, classes, gamma, beta, y64, y32


def _ratios(rows, mutant):
    """{class: restated error / bar}"""
    x, classes, gamma, beta, y64, y32 = rows
    y = L.layer_norm_f32(x, gamma, beta, mutant)
    return {n: ek / (L.LN_K * et + L.LN_FLOOR) for n, (ek, et) in L.class_errors(y, y64, y32, gamma, classes).items()}


def test_row_classes():
    """the classes are what they say: r of the DC rows, std of the near-constant rows, exact constants"""
    x, classes = L.row_classes(T, 1)
    xd = x.astype(np.float64)
    m, s = xd.mean(1), xd.std(1)
    for r in L.R_VALUES:
        rr = np.abs(m[classes[f'dc r={r:g}']]) / s[classes[f'dc r={r:g}']]
        assert rr.min() > 0.7 * r and rr.max() < 1.3 * r
    assert s[classes['near-constant']].max() < 1.5e-4 < np.sqrt(L.EPS)
    assert (x[classes['constant 2']] == 2).all() and (x[classes['constant 0.1']] == np.float32(0.1)).all()
    big = np.abs(xd[classes['massive channel']]).max(1) / np.median(np.abs(xd[classes['massive channel']]), 1)
    assert big.min() > 300
    for rows_ in classes.values():                  # every class has rows of each of the 3 images
        assert len(set(rows_ // 256)) == 3


def test_restatement_meets_the_bar(rows):
    r = _ratios(rows, None)
    print({k: f'{v:.3g}' for k, v in r.items()})
    assert max(r.values()) <= 1.0, r


def test_fp32_row_mean_is_not_the_weak_point(rows):
    """at r = 1e4 the restated kernel is no worse than float32 torch: the mean's rounding is not worth a fix"""
    x, classes, gamma, beta, y64, y32 = rows
    y = L.layer_norm_f32(x, gamma, beta)
    ek, et = L.class_errors(y, y64, y32, gamma, classes)['dc r=10000']
    assert ek <= 1.3 * et and et > 1e-4                # ... where the rounding of x - mean is already ~r 2^-24


@pytest.mark.parametrize('mutant,where', [('one_pass', 'dc r=1000'), ('eps', 'near-constant'),
                                          ('drop_float4', 'benign')])
def test_bar_rejects_the_mutant(rows, mutant, where):
    r = _ratios(rows, mutant)
    print(mutant, {k: f'{v:.3g}' for k, v in r.items()})
    assert r[where] >= 4.0, r
