"""Sharded-op kernel dispatch for the rotary position embedding (RoPE) of the Llama attention: the
half-split chain `cat(x1*c - x2*s, x2*c + x1*s)`, the rotate_half chain `x*cat(c,c) +
cat(-x2,x1)*cat(s,s)` and their autograd backwards run on edb_rope of libedb.so (edb_rope.cu), which
reads the strided input once and writes the output once; elsewhere the half-split ATen chain runs op
for op and is counted.  All four chains compute the same bits (see rope())."""
import ctypes
import sys

import torch
from torch._subclasses.fake_tensor import FakeTensor

from . import _lib
from ._lib import check
from .norm import _DT, _stream

_stats = {"edb_rope_fwd": 0, "edb_rope_bwd": 0, "aten_rope": 0}
aten = torch.ops.aten
MAX_HEAD_DIM = 512


def stats():
    return dict(_stats)


def reset_stats():
    for k in _stats:
        _stats[k] = 0


def _chain(x, cos, sin, inverse):
    """The half-split ATen chain (workloads._rope) or, inverse, its autograd backward with x = dy."""
    h = x.shape[-1] // 2
    x1, x2 = aten.slice.Tensor(x, 3, 0, h), aten.slice.Tensor(x, 3, h, sys.maxsize)
    if not inverse:
        return aten.cat.default([aten.sub.Tensor(aten.mul.Tensor(x1, cos), aten.mul.Tensor(x2, sin)),
                                 aten.add.Tensor(aten.mul.Tensor(x2, cos), aten.mul.Tensor(x1, sin))], -1)
    d1 = aten.add.Tensor(aten.mul.Tensor(x2, sin), aten.mul.Tensor(x1, cos))
    d2 = aten.add.Tensor(aten.mul.Tensor(x2, cos), aten.mul.Tensor(aten.neg.default(x1), sin))
    shape = list(x.shape)
    return aten.add.Tensor(aten.slice_backward.default(d2, shape, 3, h, sys.maxsize, 1),
                           aten.slice_backward.default(d1, shape, 3, 0, h, 1))


def formula(x, cos, sin, inverse=False):
    """The kernel's arithmetic restated with ATen ops: fp32 products and sums, rounded to x.dtype
    where the kernel rounds (for tests and documentation; dispatch uses _chain)."""
    h = x.shape[-1] // 2
    x1, x2, c, s = x[..., :h].float(), x[..., h:].float(), cos.float(), sin.float()
    if inverse:
        s = -s
    r = lambda t: t.to(x.dtype).float()
    y1, y2 = r(x1 * c) - r(x2 * s), r(x2 * c) + r(x1 * s)
    if inverse:
        y1, y2 = y1 + 0.0, y2 + 0.0
    return torch.cat((y1, y2), -1).to(x.dtype)


def _supported(x, cos, sin):
    if isinstance(x, FakeTensor) or not x.is_cuda or x.dtype not in _DT or x.dim() != 4 or x.numel() == 0:
        return False
    hd = int(x.shape[-1])
    if hd % 2 or hd > MAX_HEAD_DIM or x.stride(-1) != 1:
        return False
    tab = (int(x.shape[2]), hd // 2)
    return all(t.dtype == x.dtype and t.device == x.device and tuple(t.shape) == tab
               and t.stride(-1) == 1 for t in (cos, sin))


def rope(x, cos, sin, inverse=False, stride=None, transposed=False):
    """RoPE of x [B, H, T, hd] with [T, hd/2] tables; inverse=True gives the backward (x = dy).

    With x1, x2 the halves of the last dimension and T() the rounding to x.dtype (fp32 arithmetic):
    y1 = T(T(x1*c) - T(x2*s')), y2 = T(T(x2*c) + T(x1*s')), s' = -s when inverse — bit-identical to
    every chain lowering.fuse_rope replaces.  The result has x's shape and the given strides
    (default: contiguous); transposed=True returns it as the contiguous [B, T, H, hd] tensor that
    `y.transpose(1, 2).contiguous()` would give."""
    B, H, T, hd = x.shape
    if transposed:
        out = x.new_empty((B, T, H, hd))
        y = out.transpose(1, 2)
    else:
        out = y = x.new_empty_strided(x.shape, stride) if stride is not None else x.new_empty(x.shape)
    if not _supported(x, cos, sin) or y.stride(-1) != 1:
        if not isinstance(x, FakeTensor):
            _stats["aten_rope"] += 1
        y.copy_(_chain(x, cos, sin, inverse))
        return out
    if cos.stride(0) != sin.stride(0) or cos.stride(0) < hd // 2:
        cos, sin = cos.contiguous(), sin.contiguous()
    xs = (ctypes.c_int64 * 3)(*x.stride()[:3])
    ys = (ctypes.c_int64 * 3)(*y.stride()[:3])
    check(_lib.load().edb_rope(y.data_ptr(), x.data_ptr(), cos.data_ptr(), sin.data_ptr(), B, H, T,
                               hd // 2, xs, ys, cos.stride(0), int(bool(inverse)), _DT[x.dtype],
                               _stream(x)))
    _stats["edb_rope_bwd" if inverse else "edb_rope_fwd"] += 1
    return out
