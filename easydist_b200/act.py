"""Sharded-op kernel dispatch for the SwiGLU gate of the Llama MLP: `mul(silu(a), b)` and its
backward `mul(dy, silu(a))`, `mul(dy, b)`, `silu_backward(., a)` run on edb_swiglu_fwd / _bwd of
libedb.so (edb_rms.cu), which recompute silu(a) instead of keeping it from forward to backward;
elsewhere the same ATen chains run and are counted."""
import torch
from torch._subclasses.fake_tensor import FakeTensor

from . import _lib
from ._lib import check
from .norm import _DT, _stream

_stats = {"edb_swiglu_fwd": 0, "edb_swiglu_bwd": 0, "aten_swiglu": 0}
aten = torch.ops.aten


def stats():
    return dict(_stats)


def reset_stats():
    for k in _stats:
        _stats[k] = 0


def _supported(*ts):
    x = ts[0]
    if isinstance(x, FakeTensor) or not x.is_cuda or x.dtype not in _DT or x.numel() == 0:
        return False
    return all(t.dtype == x.dtype and t.device == x.device and tuple(t.shape) == tuple(x.shape)
               for t in ts[1:])


def swiglu_fwd(gate, up):
    """T(T(silu(gate)) * up)."""
    if not _supported(gate, up):
        if not isinstance(gate, FakeTensor):
            _stats["aten_swiglu"] += 1
        return aten.mul.Tensor(aten.silu.default(gate), up)
    gate, up = gate.contiguous(), up.contiguous()
    out = torch.empty_like(gate)
    check(_lib.load().edb_swiglu_fwd(out.data_ptr(), gate.data_ptr(), up.data_ptr(), gate.numel(),
                                     _DT[gate.dtype], _stream(gate)))
    _stats["edb_swiglu_fwd"] += 1
    return out


def swiglu_bwd(dy, gate, up):
    """(dgate, dup) = (silu_backward(T(dy * up), gate), T(dy * T(silu(gate))))."""
    if not _supported(dy, gate, up):
        if not isinstance(dy, FakeTensor):
            _stats["aten_swiglu"] += 1
        dup = aten.mul.Tensor(dy, aten.silu.default(gate))
        return aten.silu_backward.default(aten.mul.Tensor(dy, up), gate), dup
    dy, gate, up = dy.contiguous(), gate.contiguous(), up.contiguous()
    dgate, dup = torch.empty_like(gate), torch.empty_like(up)
    check(_lib.load().edb_swiglu_bwd(dgate.data_ptr(), dup.data_ptr(), dy.data_ptr(), gate.data_ptr(),
                                     up.data_ptr(), gate.numel(), _DT[gate.dtype], _stream(gate)))
    _stats["edb_swiglu_bwd"] += 1
    return dgate, dup
