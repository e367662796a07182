"""What the modules whose forward is one libcfb200 network handle (``cfb_<api>_create`` / ``_set_param`` / ``_prepare`` /
``_destroy``) share: CodeFormer / VQAutoEncoder, RRDBNet, ParseNet, RetinaFace and YOLOv5lFace.  The module owns the
parameters under the reference's state-dict names; the handle holds device copies prepared from them, rebuilt whenever a
parameter was loaded, moved or modified."""
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


class NativeHandle(nn.Module):
    """The libcfb200 handle of a module: created on first use, (re)prepared from the module's parameters and destroyed with
    the module.  ``api`` is the infix of the C functions; a subclass gives ``_create_args()``, the arguments of
    ``cfb_<api>_create``.  Calls that use the handle hold ``_lock``."""

    def __init__(self, api):
        super().__init__()
        object.__setattr__(self, '_api', api)
        object.__setattr__(self, '_lock', threading.Lock())
        object.__setattr__(self, '_net', None)
        object.__setattr__(self, '_sig', None)
        object.__setattr__(self, '_keep', None)

    def _handle(self):
        """The native handle, created on first use (host-only: the workspace queries need no device)."""
        if self._net is None:
            h = getattr(_lib.load(), f'cfb_{self._api}_create')(*self._create_args())
            if not h:
                _lib.check(1, f'cfb_{self._api}_create')
            object.__setattr__(self, '_net', ctypes.c_void_p(h))
        return self._net

    def _params(self):
        """(name, tensor) of what the handle is given: the whole state dict."""
        return list(self.state_dict(keep_vars=True).items())

    def _prepare(self, device):
        """(Re)build the native weight copies when parameters were loaded, moved or modified.  Returns whether it did."""
        lib = _lib.load()
        params = self._params()
        sig = tuple((k, v.data_ptr(), v._version, str(v.device)) for k, v in params)
        if self._net is not None and sig == self._sig:
            return False
        keep = upload_params(lib, self._api, self._handle(), params, device)
        _lib.check(getattr(lib, f'cfb_{self._api}_prepare')(self._net, _lib.stream(device)), f'cfb_{self._api}_prepare')
        object.__setattr__(self, '_sig', sig)
        object.__setattr__(self, '_keep', keep)
        return True

    def __del__(self):
        try:
            if getattr(self, '_net', None) is not None:
                getattr(_lib.load(), f'cfb_{self._api}_destroy')(self._net)
        except Exception:
            pass


class Precision:
    """The conv precision switch, mixed in before ``NativeHandle``.  ``'fp32'`` (default): split-fp16 x3 operands, fp32
    parity.  ``'fp16'``: fp16 operands with one tensor-core product per k-step, fp32 accumulation and fp32 activations.  The
    class docstring of each network says which of its convs follow it.  Every ``_prepare`` hands it to
    ``cfb_<api>_set_precision``, so it is kept across ``load_state_dict``, ``.to()`` and re-preparation, and switching never
    re-prepares the weights."""

    PRECISIONS = {'fp32': 0, 'fp16': 1}
    _precision = 'fp32'

    @property
    def precision(self):
        """``'fp32'`` or ``'fp16'`` (see ``set_precision``)."""
        return self._precision

    def set_precision(self, precision):
        """Select the conv precision, ``'fp32'`` or ``'fp16'``.  Returns the module."""
        if precision not in self.PRECISIONS:
            raise ValueError(f"{type(self).__name__}.set_precision: expected one of {sorted(self.PRECISIONS)}, got {precision!r}")
        object.__setattr__(self, '_precision', precision)
        return self

    def _prepare(self, device):
        prepared = super()._prepare(device)
        _lib.check(getattr(_lib.load(), f'cfb_{self._api}_set_precision')(self._net, self.PRECISIONS[self._precision]),
                   f'cfb_{self._api}_set_precision')
        return prepared


class NativeNet(NativeHandle):
    """Parameter holder of a network that runs on a libcfb200 handle.  ``spec`` maps the state-dict names, in registration
    order, to what ``init(name, entry, generator)`` turns into the default tensor: an ``nn.Parameter``, or a tensor that is
    registered as a buffer.  The generator is seeded with 0 and drawn from in spec order.  ``create_args`` are the arguments
    of ``cfb_<api>_create``."""

    def __init__(self, api, create_args, spec, init):
        super().__init__(api)
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
        object.__setattr__(self, '_args', tuple(create_args))
        object.__setattr__(self, '_ws', None)

    def train(self, mode=True):
        if mode:
            raise RuntimeError(f'codeformer_b200.{type(self).__name__} is inference-only (BatchNorm runs on its running '
                               'statistics); call .eval()')
        return super().train(False)

    def _create_args(self):
        return self._args

    def _params(self):
        return [(k, v) for k, v in self.state_dict(keep_vars=True).items() if v.dtype != torch.int64]   # not BatchNorm's counter

    def _workspace(self, batch, h, w, device):
        """The module's workspace for a batch x h x w forward on ``device``: grows, never shrinks."""
        need = getattr(_lib.load(), f'cfb_{self._api}_workspace_bytes')(self._handle(), batch, h, w)
        if need < 0:
            _lib.check(1, f'cfb_{self._api}_workspace_bytes')
        if self._ws is None or self._ws.numel() < need or self._ws.device != device:
            object.__setattr__(self, '_ws', None)
            object.__setattr__(self, '_ws', torch.empty(int(need), dtype=torch.uint8, device=device))
        return self._ws
