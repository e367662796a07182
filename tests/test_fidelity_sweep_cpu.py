"""Fidelity sweeps without a GPU: the chunk plan of ``restore_images_sweep``, the validation of the sweep's weights and the
workspace sizing of the sweep entry point."""
import ctypes

import numpy as np
import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import _lib
from codeformer_b200.arch import sweep_chunks, sweep_weights


@pytest.mark.parametrize('n', [0, 1, 7, 32, 33, 100])
@pytest.mark.parametrize('k', [1, 2, 3, 4, 5, 8, 40])
@pytest.mark.parametrize('max_batch', [1, 4, 32])
def test_chunk_plan(n, k, max_batch):
    chunks = sweep_chunks(n, k, max_batch)
    assert [lo for lo, _ in chunks] == list(range(0, n, max(1, max_batch // k)))
    assert (chunks[-1][1] if chunks else 0) == n
    assert all(lo < hi for lo, hi in chunks)
    assert all(hi == lo2 for (_, hi), (lo2, _) in zip(chunks, chunks[1:]))
    per = max(1, max_batch // k)
    assert all(hi - lo <= per for lo, hi in chunks)
    if k <= max_batch:
        assert all((hi - lo) * k <= max_batch for lo, hi in chunks)     # the decoder batch stays within max_batch
    else:
        assert all(hi - lo == 1 for lo, hi in chunks)


def test_weights_normalised():
    for ws in ([0.5, 1.0], (0, 1), [True], np.array([0.5, 1.0]), np.array([0.5], np.float64), torch.tensor([0.5, 1.0]),
               torch.tensor([0.5, 1.0], dtype=torch.float64), [float('nan'), -1.0, 1.7]):
        t = sweep_weights(ws)
        assert t.dtype == torch.float32 and t.dim() == 1 and t.is_contiguous() and not t.is_cuda
        assert np.array_equal(t.numpy(), np.asarray(ws, np.float32), equal_nan=True)


@pytest.mark.parametrize('bad', [[], (), np.zeros(0, np.float32), torch.zeros(0), 0.5, np.float32(0.5), np.array(0.5),
                                 torch.tensor(0.5), [[0.5, 1.0]], np.zeros((2, 2), np.float32), torch.zeros(2, 1),
                                 np.array([1, 2]), torch.tensor([1, 2]), ['a', 'b'], 'ab', None, [0.5, [1.0]]])
def test_weights_rejected(bad):
    with pytest.raises(ValueError):
        sweep_weights(bad)


def test_sweep_input_checks_before_any_device_work():
    net = cb.CodeFormer()
    with pytest.raises(RuntimeError, match='CUDA uint8'):
        net.forward_u8_sweep(torch.zeros((1, 512, 512, 3), dtype=torch.uint8), [0.5])


def test_sweep_workspace_plan():
    lib = _lib.load()
    net = cb.CodeFormer()
    h = ctypes.c_void_p(lib.cfb_net_create(ctypes.byref(net._cfb_config())))
    assert h
    try:
        one = lib.cfb_workspace_bytes(h, 1)
        s1, s4, s2x2 = lib.cfb_sweep_workspace_bytes(h, 1, 1), lib.cfb_sweep_workspace_bytes(h, 1, 4), \
            lib.cfb_sweep_workspace_bytes(h, 2, 2)
        assert 0 < s1 <= one                     # K = 1: the per-face-w plan, no expansion
        assert s1 < s4 and s1 < s2x2
        assert s4 >= lib.cfb_workspace_bytes(h, 4) - (1 << 20) - one     # a decoder at batch 4, an encoder at batch 1
        assert lib.cfb_sweep_workspace_bytes(h, 0, 3) >= 0
        assert lib.cfb_sweep_workspace_bytes(h, 1, 0) < 0 and b'k >= 1' in lib.cfb_last_error()
        assert lib.cfb_sweep_workspace_bytes(h, -1, 2) < 0
    finally:
        lib.cfb_net_destroy(h)
    vq = cb.VQAutoEncoder(512, 64, [1, 2, 2, 4, 4, 8], 'nearest', 2, [16], 1024)
    hv = ctypes.c_void_p(lib.cfb_net_create(ctypes.byref(vq._cfb_config())))
    try:
        assert lib.cfb_sweep_workspace_bytes(hv, 1, 2) < 0
    finally:
        lib.cfb_net_destroy(hv)
