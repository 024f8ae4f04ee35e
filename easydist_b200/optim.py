"""Sharded-op kernel dispatch for the optimizer region: the re-inplaced foreach triple of
torch.optim.SGD(momentum) runs as one multi-tensor kernel (edb_optim.cu).

`lowering.fuse_optimizer_updates` rewrites
    _foreach_mul_(bufs, mu); _foreach_add_(bufs, grads[, alpha]); _foreach_add_(params, bufs, alpha=-lr)
into `sgd_momentum_(params, grads, bufs, mu, grad_alpha, neg_lr)`.  The reference keeps the optimizer
inside the compiled graph (easydist/torch/compile_dp.py:201-260), so this is part of the step."""
import ctypes

import torch
from torch._subclasses.fake_tensor import FakeTensor
from torch.fx.node import has_side_effect

from . import _lib
from ._lib import check, i64_array

aten = torch.ops.aten
_stats = {"edb_sgd": 0, "aten_sgd": 0}
_DT = {torch.bfloat16: _lib.DTYPE_CODES["bfloat16"], torch.float32: _lib.DTYPE_CODES["float32"]}


def stats():
    return dict(_stats)


def reset_stats():
    for k in _stats:
        _stats[k] = 0


def _ptr_array(tensors):
    return (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


def _tensor_ok(p, g, m, dt):
    if isinstance(p, FakeTensor) or not p.is_cuda:
        return False
    if not (p.dtype == g.dtype == m.dtype == dt and p.shape == g.shape == m.shape):
        return False
    if not (p.is_contiguous() and g.is_contiguous() and m.is_contiguous()):
        return False
    return not ((p.data_ptr() | g.data_ptr() | m.data_ptr()) & 15)


def _scale_ok(c, p):
    return c.dtype == p.dtype and c.device == p.device and c.numel() == 1


def _aten(params, grads, bufs, mu, grad_alpha, neg_lr, grad_scale=None):
    if grad_scale is not None:  # clip_grad_norm_'s mul_(g, coef), without writing g
        grads = [aten.mul.Tensor(g, grad_scale) for g in grads]
    aten._foreach_mul_.Scalar(bufs, mu)
    aten._foreach_add_.List(bufs, grads, alpha=grad_alpha)
    aten._foreach_add_.List(params, bufs, alpha=neg_lr)


@has_side_effect
def sgd_momentum_(params, grads, bufs, mu, grad_alpha, neg_lr, grad_scale=None):
    """In place: bufs = mu*bufs + grad_alpha*grads; params += neg_lr*bufs (per tensor).  Tensors the
    kernel's contract does not cover (other dtypes, views that are not 16-byte aligned, e.g. slices
    of a gradient bucket) take the three ATen ops; both groups are counted.

    grad_scale (a one-element tensor of the parameters' dtype): the update uses T(g*grad_scale), the
    rounding of gradient clipping's `mul_(g, grad_scale)`; the gradients themselves are not written."""
    if not params or len(params) != len(grads) or len(params) != len(bufs):
        raise ValueError("sgd_momentum_: params, grads and bufs must be lists of equal length")
    if isinstance(params[0], FakeTensor):
        return _aten(params, grads, bufs, mu, grad_alpha, neg_lr, grad_scale)
    native = {}
    rest = []
    for i, (p, g, m) in enumerate(zip(params, grads, bufs)):
        if p.dtype in _DT and _tensor_ok(p, g, m, p.dtype) and \
                (grad_scale is None or _scale_ok(grad_scale, p)):
            native.setdefault(p.dtype, []).append(i)
        else:
            rest.append(i)
    if rest:
        _stats["aten_sgd"] += 1
        _aten([params[i] for i in rest], [grads[i] for i in rest], [bufs[i] for i in rest], mu,
              grad_alpha, neg_lr, grad_scale)
    for dt, idx in native.items():
        lib = _lib.load()
        ps, gs, ms = [params[i] for i in idx], [grads[i] for i in idx], [bufs[i] for i in idx]
        stream = torch.cuda.current_stream(ps[0].device).cuda_stream
        if grad_scale is None:
            check(lib.edb_sgd_momentum(len(ps), _ptr_array(ps), _ptr_array(gs), _ptr_array(ms),
                                       i64_array([p.numel() for p in ps]), float(mu),
                                       float(grad_alpha), float(neg_lr), _DT[dt], stream))
        else:
            check(lib.edb_sgd_momentum_scaled(len(ps), _ptr_array(ps), _ptr_array(gs), _ptr_array(ms),
                                              i64_array([p.numel() for p in ps]), float(mu),
                                              float(grad_alpha), float(neg_lr), grad_scale.data_ptr(),
                                              _DT[dt], stream))
        _stats["edb_sgd"] += 1
    return None
