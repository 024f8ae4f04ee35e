"""Sharded-op kernel dispatch for gradient-norm clipping, `torch.nn.utils.clip_grad_norm_(params,
max_norm)` with norm_type 2, on edb_clip.cu of libedb.so.

Traced, the clip is one `linalg_vector_norm(g, 2.0)` per gradient, `stack`, the total norm and the
coefficient `clamp(max_norm / (total + 1e-6), max=1)`, then one in-place `mul_(g, coef)` per gradient.
`lowering.fuse_grad_clip` replaces the T norms and the stack with one `grad_norms` node, and the T
`mul_` nodes with the `grad_scale=` of the fused SGD (optim.sgd_momentum_) or one `scale_` node;
`lowering.transform_fsdp` computes the norms of sharded gradients from `grad_sumsq` of the shards.
On FakeTensors, CPU tensors or lists the kernels do not take (mixed dtypes or devices, other dtypes,
views that are not dense) the replaced ATen ops run op for op and the call is counted."""
from ctypes import byref, c_size_t

import torch
from torch._subclasses.fake_tensor import FakeTensor
from torch.fx.node import has_side_effect

from . import _lib
from ._lib import check, i64_array
from .norm import _DT, _stream
from .optim import _ptr_array

aten = torch.ops.aten
RAW, NORM = 0, 1  # EDB_SUMSQ_RAW / EDB_SUMSQ_NORM
_stats = {"edb_sumsq": 0, "aten_sumsq": 0, "edb_scale": 0, "aten_scale": 0}
_workspaces = {}


def stats():
    return dict(_stats)


def reset_stats():
    for k in _stats:
        _stats[k] = 0


def _dense(t):
    """t covers exactly numel consecutive elements from data_ptr() (a permutation of a contiguous
    tensor, e.g. the t() of a weight gradient)."""
    expect = 1
    for stride, size in sorted((st, s) for s, st in zip(t.shape, t.stride()) if s != 1):
        if stride != expect:
            return False
        expect *= size
    return True


def _native(ts):
    """One CUDA device, one kernel dtype, every tensor a dense span of its storage."""
    if not ts or isinstance(ts[0], FakeTensor):
        return False
    t0 = ts[0]
    return t0.is_cuda and t0.dtype in _DT and all(
        t.device == t0.device and t.dtype == t0.dtype and _dense(t) for t in ts)


def _count(key, ts):
    if ts and not isinstance(ts[0], FakeTensor):
        _stats[key] += 1


def _sumsq(grads, mode):
    numels = i64_array([g.numel() for g in grads])
    dt = _DT[grads[0].dtype]
    lib = _lib.load()
    key = (tuple(g.numel() for g in grads), dt, grads[0].device)
    ws = _workspaces.get(key)
    if ws is None:
        nbytes = c_size_t()
        check(lib.edb_grad_sumsq_workspace(len(grads), numels, dt, byref(nbytes)))
        ws = _workspaces[key] = torch.empty(max(16, nbytes.value), dtype=torch.uint8,
                                            device=grads[0].device)
    out = torch.empty(len(grads), dtype=torch.float32 if mode == RAW else grads[0].dtype,
                      device=grads[0].device)
    # a dense view (e.g. the t() of a weight gradient) is read as its storage: the sum of squares
    # does not depend on the order of the elements, and data_ptr() is the lowest address of the span
    check(lib.edb_grad_sumsq(len(grads), _ptr_array(grads), numels, out.data_ptr(), ws.data_ptr(),
                             mode, dt, _stream(grads[0])))
    _stats["edb_sumsq"] += 1
    return out


def grad_norms(grads):
    """[T] tensor of the gradients' dtype: `stack([linalg_vector_norm(g, 2.0) for g in grads])`.
    The kernel gives T(sqrtf(s)) with s the fp32 sum of squares in a fixed order."""
    grads = list(grads)
    if not grads:
        raise ValueError("grad_norms: empty gradient list")
    if _native(grads):
        return _sumsq(grads, NORM)
    _count("aten_sumsq", grads)
    return aten.stack.default([aten.linalg_vector_norm.default(g, 2.0) for g in grads])


def grad_sumsq(grads):
    """[T] fp32: the sum of squares of every gradient, accumulated in fp32 (the kernel's fixed
    order; elsewhere `sum(g.float() * g.float())`)."""
    grads = list(grads)
    if not grads:
        raise ValueError("grad_sumsq: empty gradient list")
    if _native(grads):
        return _sumsq(grads, RAW)
    _count("aten_sumsq", grads)
    sq = []
    for g in grads:
        f = aten._to_copy.default(g, dtype=torch.float32)
        sq.append(aten.sum.default(aten.mul.Tensor(f, f)))
    return aten.stack.default(sq)


@has_side_effect
def scale_(grads, coef):
    """In place: g = g * coef for every gradient, bit-identical to the per-tensor `mul_(g, coef)` of
    clip_grad_norm_ (coef: a one-element tensor of the gradients' dtype, on their device)."""
    grads = list(grads)
    if _native(grads) and coef.dtype == grads[0].dtype and coef.device == grads[0].device \
            and coef.numel() == 1:
        check(_lib.load().edb_multi_scale_(len(grads), _ptr_array(grads),
                                           i64_array([g.numel() for g in grads]), coef.data_ptr(),
                                           _DT[coef.dtype], _stream(coef)))
        _stats["edb_scale"] += 1
        return None
    _count("aten_scale", grads)
    for g in grads:
        aten.mul_.Tensor(g, coef)
    return None
