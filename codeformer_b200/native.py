"""What the modules whose forward is one libcfb200 network handle (``cfb_<api>_create`` / ``_set_param`` / ``_prepare`` /
``_workspace_bytes`` / ``_destroy``) share: RRDBNet, ParseNet, RetinaFace and YOLOv5lFace.  The module owns the parameters
under the reference's state-dict names; the handle holds device copies prepared from them, rebuilt whenever a parameter
was loaded, moved or modified."""
import ctypes
import threading

import torch
import torch.nn as nn

from . import _lib


def upload_params(lib, api, handle, params, device):
    """Register every (name, tensor) of ``params`` with the handle (``cfb_<api>_set_param``).  Returns the fp32 contiguous
    tensors the handle points into: the caller keeps them alive until the next upload."""
    set_param = getattr(lib, f'cfb_{api}_set_param')
    keep = []
    for k, v in params:
        if v.device != device:
            raise RuntimeError(f'parameter {k} is on {v.device} but the input is on {device}; call net.to(device)')
        t = v.detach()
        if t.dtype != torch.float32 or not t.is_contiguous():
            t = t.float().contiguous()
        keep.append(t)
        _lib.check(set_param(handle, k.encode(), _lib.ptr(t), t.numel()), f'cfb_{api}_set_param')
    return keep


class NativeNet(nn.Module):
    """Parameter holder of a network that runs on a libcfb200 handle.  ``spec`` maps the state-dict names, in registration
    order, to what ``init(name, entry, generator)`` turns into the default tensor: an ``nn.Parameter``, or a tensor that is
    registered as a buffer.  The generator is seeded with 0 and drawn from in spec order.  ``api`` is the infix of the C
    functions, ``create_args`` the arguments of ``cfb_<api>_create``."""

    def __init__(self, api, create_args, spec, init):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        for name, entry in spec.items():
            mod, parts = self, name.split('.')
            for p in parts[:-1]:
                if not hasattr(mod, p):
                    mod.add_module(p, nn.Module())
                mod = getattr(mod, p)
            t = init(name, entry, g)
            if isinstance(t, nn.Parameter):
                mod.register_parameter(parts[-1], t)
            else:
                mod.register_buffer(parts[-1], t)
        object.__setattr__(self, '_api', api)
        object.__setattr__(self, '_create_args', tuple(create_args))
        object.__setattr__(self, '_lock', threading.Lock())
        object.__setattr__(self, '_net', None)
        object.__setattr__(self, '_sig', None)
        object.__setattr__(self, '_keep', None)
        object.__setattr__(self, '_ws', None)

    def train(self, mode=True):
        if mode:
            raise RuntimeError(f'codeformer_b200.{type(self).__name__} is inference-only (BatchNorm runs on its running '
                               'statistics); call .eval()')
        return super().train(False)

    def _handle(self):
        """The native handle, created on first use (host-only: the workspace queries need no device)."""
        if self._net is None:
            h = getattr(_lib.load(), f'cfb_{self._api}_create')(*self._create_args)
            if not h:
                _lib.check(1, f'cfb_{self._api}_create')
            object.__setattr__(self, '_net', ctypes.c_void_p(h))
        return self._net

    def _prepare(self, device):
        """(Re)build the native weight copies when parameters were loaded, moved or modified."""
        lib = _lib.load()
        params = [(k, v) for k, v in self.state_dict(keep_vars=True).items() if v.dtype != torch.int64]
        sig = tuple((k, v.data_ptr(), v._version, str(v.device)) for k, v in params)
        if self._net is not None and sig == self._sig:
            return
        keep = upload_params(lib, self._api, self._handle(), params, device)
        _lib.check(getattr(lib, f'cfb_{self._api}_prepare')(self._net, ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)),
                   f'cfb_{self._api}_prepare')
        object.__setattr__(self, '_sig', sig)
        object.__setattr__(self, '_keep', keep)

    def _workspace(self, batch, h, w, device):
        """The module's workspace for a batch x h x w forward on ``device``: grows, never shrinks."""
        need = getattr(_lib.load(), f'cfb_{self._api}_workspace_bytes')(self._handle(), batch, h, w)
        if need < 0:
            _lib.check(1, f'cfb_{self._api}_workspace_bytes')
        if self._ws is None or self._ws.numel() < need or self._ws.device != device:
            object.__setattr__(self, '_ws', None)
            object.__setattr__(self, '_ws', torch.empty(int(need), dtype=torch.uint8, device=device))
        return self._ws

    def __del__(self):
        try:
            if getattr(self, '_net', None) is not None:
                getattr(_lib.load(), f'cfb_{self._api}_destroy')(self._net)
        except Exception:
            pass
