"""CPU: the bar of tests/test_gpu_split_error_model.py has teeth.  On that file's CASES (at a smaller spatial size) and operands,
split_bar accepts the float64 emulation of the split-fp16 arithmetic, with exact and with truncating accumulation, and rejects
every mutant that loses lo products (tests/split_emul.py MUTANTS) by at least 4x.  Mutants cannot be built on the GPU, so this
is what shows that a kernel losing part of its lo arithmetic would fail there."""
import math

import pytest
import torch

from tests import split_emul as S
from tests.test_gpu_split_error_model import CASES, TAU, case_inputs, kinds, operand

MARGIN = 4.0


def _separable(c, kind, m):
    """The H100 accumulates sign-aligned sums with an error of ~1.2e-5 B (DESIGN.md section 4), the size of one lost k-block
    of lo at Cin >= 256 under those operands, and the Upsample parity sums re-round the aligned weights (their lo is no longer
    pushed): the aligned bar cannot separate those two mutants; the random-operand run of the same case does."""
    return kind == 'random' or not (m == 'kblock' or (m == 'w_lo' and c.g.up))


def _small(c):
    return dict(N=min(c.N, 2), H=c.H if c.H <= 24 else 16, W=c.W if c.W <= 24 else 16)


def _mutants(c):
    return [m for m in S.MUTANTS if (m != 'cat' or c.cin1) and (m != 'upper64' or c.Cout % 128 == 0)]


ALL = [(c, k) for c in CASES for k in kinds(c)]


@pytest.mark.parametrize('c,kind', ALL, ids=[f'{c.name}-{k}' for c, k in ALL])
def test_bar_accepts_the_split_and_rejects_every_mutant(c, kind):
    torch.set_num_threads(min(8, torch.get_num_threads()))
    x, w, b, sc, sh, *_ = case_inputs(c, kind, **_small(c))
    xo = operand(c, x, sc, sh)
    ref, B, floor = S.bounds(xo, w, c.g)
    tau = TAU[kind]
    exact = S.split_bar(S.model(xo, w, c.g, cin1=c.cin1), ref, B, floor, tau)
    trunc = S.split_bar(S.model(xo, w, c.g, cin1=c.cin1, trunc=True), ref, B, floor, tau)
    margins = {m: S.split_bar(S.model(xo, w, c.g, mutant=m, cin1=c.cin1), ref, B, floor, tau).worst for m in _mutants(c)}
    print(f'{c.name:22s} {kind:8s} exact {exact.worst:.3f} trunc {trunc.worst:.3f} mutant margins ' +
          ' '.join(f'{m} {v:.1f}' for m, v in margins.items()))
    assert exact.ok and trunc.ok, (exact, trunc)
    weak = {m: v for m, v in margins.items() if not v >= MARGIN and _separable(c, kind, m)}
    assert not weak, f'mutants the bar does not reject by {MARGIN}x: {weak}'


def test_split_bar_reports_the_worst_output_and_fails_nan():
    ref = torch.zeros(2, 3, 4, 8, dtype=torch.float64)
    B = torch.ones_like(ref)
    out = ref.clone()
    out[1, 2, 3, 5] = 3e-6
    bar = S.split_bar(out, ref, B, torch.zeros_like(ref), 1e-6, tile=128)
    assert not bar.ok and bar.where == (1, 2, 3, 5) and bar.tile == 128 and math.isclose(bar.worst, 3.0)
    assert S.split_bar(out, ref, B, torch.zeros_like(ref), 4e-6).ok
    out[0, 0, 0, 0] = float('nan')
    bad = S.split_bar(out, ref, B, torch.zeros_like(ref), 1.0)
    assert not bad.ok and bad.where == (0, 0, 0, 0)

