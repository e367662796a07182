"""Host-only planning of the networks on the conv engine (RRDBNet, ParseNet, RetinaFace, YOLOv5-face): the workspace a forward
asks for (a dry run of the arena allocation sequence over the planned channel counts) and the default parameters of a freshly
built module.  Both are pinned to the values of the builds before the shared network core."""
import ctypes
import hashlib

import pytest
import torch

import codeformer_b200 as cb
from codeformer_b200 import _lib


@pytest.mark.parametrize('api,create,sizes', [
    ('retinaface', (), [((1, 64, 64), 921600), ((2, 480, 640), 137629696), ((1, 37, 50), 471040)]),
    ('yolov5face', (), [((1, 64, 64), 921600), ((2, 640, 640), 183504896), ((1, 96, 160), 3444736)]),
    ('parsenet', (512, 512, 32, 64, 19, 10, 32, 256), [((1, 512, 512), 268439552), ((4, 512, 512), 1073745920)]),
    ('rrdb', (3, 3, 2, 64, 23, 32), [((1, 400, 400), 481288192)]),
])
def test_dry_run_workspace_bytes(api, create, sizes):
    lib = _lib.load()
    h = ctypes.c_void_p(getattr(lib, f'cfb_{api}_create')(*create))
    assert h.value, lib.cfb_last_error()
    try:
        for (b, hh, ww), want in sizes:
            assert getattr(lib, f'cfb_{api}_workspace_bytes')(h, b, hh, ww) == want, (api, b, hh, ww)
    finally:
        getattr(lib, f'cfb_{api}_destroy')(h)


def _digest(sd):
    m = hashlib.sha256()
    for k, v in sd.items():
        m.update(k.encode())
        m.update(str(v.dtype).encode())
        m.update(v.contiguous().numpy().tobytes())
    return m.hexdigest()[:16]


@pytest.mark.parametrize('make,digest,entries,split', [
    (lambda: cb.RRDBNet(3, 3, scale=2), '1c9e2dd6d2336e99', 702, None),
    (lambda: cb.ParseNet(512, 512, parsing_ch=19), '2b196b39182e4fc6', 238, (130, 108)),
    (lambda: cb.RetinaFace(), 'b413dd00ddc78a89', 456, (237, 219)),
    (lambda: cb.YOLOv5lFace(), 'cbdc7dfcd91b7b75', 662, (333, 329)),
])
def test_default_state_dict(make, digest, entries, split):
    net = make()
    sd = net.state_dict()
    assert len(sd) == entries
    if split is not None:
        assert (len(list(net.parameters())), len(list(net.buffers()))) == split
    assert _digest(sd) == digest
    assert all(isinstance(p, torch.nn.Parameter) for p in net.parameters())
