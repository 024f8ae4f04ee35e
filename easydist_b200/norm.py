"""Sharded-op kernel dispatch for LayerNorm: `aten.native_layer_norm` and
`aten.native_layer_norm_backward` nodes of the compiled graph run on the HBM-streaming kernels of
libedb.so (edb_norm.cu); shapes they do not cover go to ATen and are counted."""
from ctypes import byref, c_size_t

import torch
from torch._subclasses.fake_tensor import FakeTensor

from . import _lib
from ._lib import check

_stats = {"edb_ln_fwd": 0, "edb_ln_bwd": 0, "aten_ln": 0, "edb_colsum": 0, "aten_sum": 0,
          "edb_rms_fwd": 0, "edb_rms_bwd": 0, "aten_rms": 0}
_DT = {torch.bfloat16: _lib.DTYPE_CODES["bfloat16"], torch.float32: _lib.DTYPE_CODES["float32"]}
_workspaces = {}
aten = torch.ops.aten


def stats():
    return dict(_stats)


def reset_stats():
    for k in _stats:
        _stats[k] = 0


def _supported(x, normalized_shape, weight):
    if isinstance(x, FakeTensor) or not x.is_cuda or x.dtype not in _DT:
        return False
    if len(normalized_shape) != 1 or weight is None or weight.dtype != x.dtype:
        return False
    H = int(normalized_shape[0])
    per, hmax = (256, 2048) if x.dtype == torch.bfloat16 else (128, 1024)
    return H % per == 0 and H <= hmax and (H // per) in (1, 2, 3, 4, 6, 8) and x.numel() > 0


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _dense(t):
    """`t` when it is contiguous and 16-byte aligned, the layout every LayerNorm and RMSNorm kernel
    reads (H consecutive elements per row, 16-byte vectors); otherwise a dense copy in a fresh
    allocation.  `.contiguous()` alone keeps a contiguous view at a misaligned storage offset."""
    if t.is_contiguous() and t.data_ptr() % 16 == 0:
        return t
    return t.clone(memory_format=torch.contiguous_format)


def native_layer_norm(input, normalized_shape, weight, bias, eps):
    if not _supported(input, normalized_shape, weight) or (bias is not None and bias.dtype != input.dtype):
        if not isinstance(input, FakeTensor):
            _stats["aten_ln"] += 1
        return aten.native_layer_norm.default(input, normalized_shape, weight, bias, eps)
    x, weight = _dense(input), _dense(weight)
    bias = _dense(bias) if bias is not None else None
    H = int(normalized_shape[0])
    rows = x.numel() // H
    y = torch.empty_like(x)
    stat_shape = list(x.shape[:-1]) + [1]
    mean = torch.empty(stat_shape, dtype=torch.float32, device=x.device)
    rstd = torch.empty(stat_shape, dtype=torch.float32, device=x.device)
    lib = _lib.load()
    check(lib.edb_layer_norm_fwd(y.data_ptr(), mean.data_ptr(), rstd.data_ptr(), x.data_ptr(),
                                 weight.data_ptr(), bias.data_ptr() if bias is not None else None,
                                 rows, H, float(eps), _DT[x.dtype], _stream(x)))
    _stats["edb_ln_fwd"] += 1
    return y, mean, rstd


def _workspace(H, device):
    key = (H, device)
    ws = _workspaces.get(key)
    if ws is None:
        nbytes = c_size_t()
        check(_lib.load().edb_layer_norm_bwd_workspace(H, byref(nbytes)))
        ws = torch.empty(max(16, nbytes.value), dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


def native_layer_norm_backward(grad_out, input, normalized_shape, mean, rstd, weight, bias,
                               output_mask, *, _add=None):
    """`_add`: a tensor of input's shape added to dx inside the kernel (the gradient accumulation
    `aten.add.Tensor(dx, residual_grad)` that follows in the traced backward pass)."""
    ok = (_supported(input, normalized_shape, weight) and grad_out.dtype == input.dtype
          and mean.dtype == torch.float32 and rstd.dtype == torch.float32 and output_mask[0])
    if ok and _add is not None:
        ok = _add.dtype == input.dtype and _add.shape == input.shape
    if not ok:
        if not isinstance(input, FakeTensor):
            _stats["aten_ln"] += 1
        res = aten.native_layer_norm_backward.default(grad_out, input, normalized_shape, mean, rstd,
                                                      weight, bias, output_mask)
        if _add is not None:
            res = (aten.add.Tensor(res[0], _add),) + tuple(res[1:])
        return res
    x, dy, weight = _dense(input), _dense(grad_out), _dense(weight)
    H = int(normalized_shape[0])
    rows = x.numel() // H
    dx = torch.empty_like(x)
    dw = torch.empty_like(weight) if output_mask[1] else None
    db = torch.empty_like(weight) if output_mask[2] else None
    ws = _workspace(H, x.device)
    lib = _lib.load()
    add = _dense(_add) if _add is not None else None
    check(lib.edb_layer_norm_bwd_add(dx.data_ptr(), dw.data_ptr() if dw is not None else None,
                                     db.data_ptr() if db is not None else None, dy.data_ptr(),
                                     x.data_ptr(), mean.contiguous().data_ptr(),
                                     rstd.contiguous().data_ptr(), weight.data_ptr(),
                                     add.data_ptr() if add is not None else None, ws.data_ptr(), rows,
                                     H, _DT[x.dtype], _stream(x)))
    _stats["edb_ln_bwd"] += 1
    return dx, dw, db


_cs_workspaces = {}


def sum_dim_intlist(x, dim, keepdim=False, *, dtype=None):
    """aten.sum.dim_IntList; the column-sum case (2-D, dim == [0]) — every bias gradient of the
    train step — runs on edb_colsum, everything else on ATen."""
    ok = (not isinstance(x, FakeTensor) and x.is_cuda and x.dim() == 2 and list(dim) == [0]
          and dtype is None and x.dtype in _DT and x.stride(1) == 1 and x.numel() > 0)
    if ok:
        epv = 8 if x.dtype == torch.bfloat16 else 4
        ok = x.shape[1] % epv == 0 and x.stride(0) % epv == 0 and x.data_ptr() % 16 == 0 \
            and x.shape[0] >= 64
    if not ok:
        if not isinstance(x, FakeTensor):
            _stats["aten_sum"] += 1
        return aten.sum.dim_IntList(x, dim, keepdim, dtype=dtype)
    rows, cols = x.shape
    key = (cols, x.device)
    ws = _cs_workspaces.get(key)
    lib = _lib.load()
    if ws is None:
        nbytes = c_size_t()
        check(lib.edb_colsum_workspace(cols, byref(nbytes)))
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=x.device)
        _cs_workspaces[key] = ws
    out = torch.empty((1, cols) if keepdim else (cols,), dtype=x.dtype, device=x.device)
    check(lib.edb_colsum(out.data_ptr(), x.data_ptr(), ws.data_ptr(), rows, cols, x.stride(0),
                         _DT[x.dtype], _stream(x)))
    _stats["edb_colsum"] += 1
    return out


# RMSNorm rounding contracts (include/edb.h): the hand-written Llama form
# `(x.float() * rsqrt(mean(x^2) + eps)).to(T) * w` rounds the normed value to T before the weight
# multiply; aten._fused_rms_norm rounds once at the end
RMS_CAST_THEN_SCALE, RMS_FUSED = 0, 1
RMS_MAX_H = 16384
_rms_workspaces = {}


def _rms_supported(x, w, H):
    if isinstance(x, FakeTensor) or not x.is_cuda or x.dtype not in _DT or x.numel() == 0:
        return False
    if w is None or w.dtype != x.dtype or tuple(w.shape) != (H,) or x.shape[-1] != H:
        return False
    epv = 8 if x.dtype == torch.bfloat16 else 4
    return H % epv == 0 and H <= RMS_MAX_H


def _rms_fwd_chain(x, w, eps):
    """The ATen ops `RMSNorm.forward` of workloads.py traces to, op for op."""
    low = x.dtype != torch.float32
    x32 = aten._to_copy.default(x, dtype=torch.float32) if low else x
    v = aten.mean.dim(aten.pow.Tensor_Scalar(x32, 2), [-1], True)
    rstd = aten.rsqrt.default(aten.add.Tensor(v, eps))
    n = aten.mul.Tensor(x32, rstd)
    if low:
        n = aten._to_copy.default(n, dtype=x.dtype)
    return aten.mul.Tensor(n, w), rstd


def _rms_bwd_chain(dy, x, rstd, w, output_mask, add):
    """The backward of `_rms_fwd_chain` as autograd traces it, op for op: dw from the rounded
    normed value, dx in two separately rounded pieces added onto the running gradient `add`."""
    low = x.dtype != torch.float32
    x32 = aten._to_copy.default(x, dtype=torch.float32) if low else x
    dw = None
    if output_mask[1]:
        n = aten.mul.Tensor(x32, rstd)
        if low:
            n = aten._to_copy.default(n, dtype=x.dtype)
        dw = aten.sum.dim_IntList(aten.mul.Tensor(dy, n), list(range(dy.dim() - 1)), True)
        dw = aten.view.default(dw, list(w.shape))
    g = aten.mul.Tensor(dy, w)
    g32 = aten._to_copy.default(g, dtype=torch.float32) if low else g
    p1 = aten.mul.Tensor(g32, rstd)
    s = aten.sum.dim_IntList(aten.mul.Tensor(g32, x32), [dy.dim() - 1], True)
    m = aten.mul.Tensor(aten.mul.Scalar(s, -0.5), aten.pow.Tensor_Scalar(rstd, 3))
    d = aten.div.Scalar(aten.expand.default(m, list(x.shape)), x.shape[-1])
    p2 = aten.mul.Tensor(d, aten.mul.Scalar(aten.pow.Tensor_Scalar(x32, 1.0), 2.0))
    if low:
        p1 = aten._to_copy.default(p1, dtype=x.dtype)
        p2 = aten._to_copy.default(p2, dtype=x.dtype)
    dx = aten.add.Tensor(p1, p2) if add is None else aten.add.Tensor(aten.add.Tensor(add, p1), p2)
    return dx, dw


def rms_norm_fwd(x, w, eps, mode):
    """RMSNorm over the last dimension -> (y, rstd [..., 1] fp32) on edb_rms_norm_fwd.  Elsewhere
    (FakeTensor, CPU, unsupported shape) the ATen ops the kernel replaces: the decomposed Llama chain
    for RMS_CAST_THEN_SCALE, aten._fused_rms_norm for RMS_FUSED (counted as `aten_rms`)."""
    H = int(x.shape[-1])
    if not _rms_supported(x, w, H):
        if not isinstance(x, FakeTensor):
            _stats["aten_rms"] += 1
        if mode == RMS_FUSED:
            return aten._fused_rms_norm.default(x, [H], w, eps)
        return _rms_fwd_chain(x, w, eps)
    x, w = _dense(x), _dense(w)
    rows = x.numel() // H
    y = torch.empty_like(x)
    rstd = torch.empty(list(x.shape[:-1]) + [1], dtype=torch.float32, device=x.device)
    check(_lib.load().edb_rms_norm_fwd(y.data_ptr(), rstd.data_ptr(), x.data_ptr(), w.data_ptr(), rows,
                                       H, float(eps), mode, _DT[x.dtype], _stream(x)))
    _stats["edb_rms_fwd"] += 1
    return y, rstd


def rms_norm_bwd(dy, x, rstd, w, mode, output_mask, *, _add=None):
    """Backward of `rms_norm_fwd` -> (dx, dw) on edb_rms_norm_bwd; dw is None unless output_mask[1].
    `_add`: the running gradient of x, added to dx inside the kernel (the trailing `aten.add.Tensor`s
    of the traced backward)."""
    H = int(x.shape[-1])
    ok = (_rms_supported(x, w, H) and dy.dtype == x.dtype and tuple(dy.shape) == tuple(x.shape)
          and rstd.dtype == torch.float32 and rstd.numel() * H == x.numel() and output_mask[0])
    if ok and _add is not None:
        ok = _add.dtype == x.dtype and tuple(_add.shape) == tuple(x.shape)
    if not ok:
        if not isinstance(x, FakeTensor):
            _stats["aten_rms"] += 1
        if mode == RMS_FUSED:
            dx, dw = aten._fused_rms_norm_backward.default(dy, x, [H], rstd, w, list(output_mask))
            if _add is not None:
                dx = aten.add.Tensor(dx, _add)
            return dx, dw
        return _rms_bwd_chain(dy, x, rstd, w, output_mask, _add)
    x, dy, w = _dense(x), _dense(dy), _dense(w)
    rows = x.numel() // H
    dx = torch.empty_like(x)
    dw = torch.empty_like(w) if output_mask[1] else None
    lib = _lib.load()
    key = (H, x.device)
    ws = _rms_workspaces.get(key)
    if ws is None:
        nbytes = c_size_t()
        check(lib.edb_rms_norm_bwd_workspace(H, byref(nbytes)))
        ws = _rms_workspaces[key] = torch.empty(max(16, nbytes.value), dtype=torch.uint8,
                                                device=x.device)
    add = _dense(_add) if _add is not None else None
    check(lib.edb_rms_norm_bwd(dx.data_ptr(), dw.data_ptr() if dw is not None else None,
                               dy.data_ptr(), x.data_ptr(), rstd.contiguous().data_ptr(), w.data_ptr(),
                               add.data_ptr() if add is not None else None, ws.data_ptr(), rows, H,
                               mode, _DT[x.dtype], _stream(x)))
    _stats["edb_rms_bwd"] += 1
    return dx, dw


def fused_rms_norm(input, normalized_shape, weight, eps):
    """Node target for `aten._fused_rms_norm` (what F.rms_norm / nn.RMSNorm dispatch to on CUDA)."""
    if len(normalized_shape) != 1 or weight is None:
        if not isinstance(input, FakeTensor):
            _stats["aten_rms"] += 1
        return aten._fused_rms_norm.default(input, normalized_shape, weight, eps)
    if eps is None and input.dtype in _DT:  # ATen's default: the epsilon of the fp32 accumulation
        eps = torch.finfo(torch.float32).eps
    return rms_norm_fwd(input, weight, eps, RMS_FUSED)


def fused_rms_norm_backward(grad_out, input, normalized_shape, rstd, weight, output_mask, *,
                            _add=None):
    """Node target for `aten._fused_rms_norm_backward`; `_add` as in `rms_norm_bwd`."""
    if len(normalized_shape) != 1 or weight is None:
        if not isinstance(input, FakeTensor):
            _stats["aten_rms"] += 1
        dx, dw = aten._fused_rms_norm_backward.default(grad_out, input, normalized_shape, rstd,
                                                       weight, output_mask)
        return (dx if _add is None else aten.add.Tensor(dx, _add)), dw
    return rms_norm_bwd(grad_out, input, rstd, weight, RMS_FUSED, output_mask, _add=_add)
