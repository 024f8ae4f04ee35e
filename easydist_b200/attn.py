"""Sharded-op kernel dispatch for scaled-dot-product attention: the fused-attention forward and
backward nodes of a traced step (`aten._scaled_dot_product_cudnn_attention`, which SDPA traces to on
the H100, `aten._scaled_dot_product_flash_attention[_for_cpu]`, and their backwards) of a step
compiled under deterministic algorithms run on edb_attn_fwd / edb_attn_bwd of libedb.so
(edb_attn.cu), whose backward gives the same bits on every run, when q, k and v are CUDA bf16
tensors of one shape with head dim 64 or 128, a contiguous last dim, 16-byte aligned pointers and
positive strides, and the scale is positive.  Elsewhere (fake and CPU tensors, other dtypes and
head dims, other layouts, broadcast views)
the ATen op the node called runs op for op and is counted (on CUDA with misaligned inputs copied
to aligned ones, which ATen's flash kernels need).

The native logsumexp is the natural-log row logsumexp [B, H, T] of scale·q·kᵀ, the quantity ATen's
ops return; only the native backward is guaranteed to read it back the same way."""
import ctypes
import math

import torch
from torch._subclasses.fake_tensor import FakeTensor

from . import _lib
from ._lib import check
from .norm import _stream

_stats = {"edb_attn_fwd": 0, "edb_attn_bwd": 0, "aten_attn_fwd": 0, "aten_attn_bwd": 0}
aten = torch.ops.aten
HEAD_DIMS = (64, 128)
# the ATen pairs the rewrite replaces, by the name of the `aten_op` argument that selects them
FWD_OPS = {"flash": aten._scaled_dot_product_flash_attention.default,
           "cpu": aten._scaled_dot_product_flash_attention_for_cpu.default,
           "cudnn": aten._scaled_dot_product_cudnn_attention.default}
BWD_OPS = {"flash": aten._scaled_dot_product_flash_attention_backward.default,
           "cpu": aten._scaled_dot_product_flash_attention_for_cpu_backward.default,
           "cudnn": aten._scaled_dot_product_cudnn_attention_backward.default}


def stats():
    return dict(_stats)


def reset_stats():
    for k in _stats:
        _stats[k] = 0


def _supported(scale, *ts):
    """The kernels take ts: CUDA bf16 of q's shape, hd 64 or 128, last dim contiguous, 16-byte
    aligned data and positive 16-byte (B, H, T) strides (no broadcast views); and a positive finite
    scale (the online softmax shifts by the row maximum of the raw scores)."""
    if scale is not None and not (0 < float(scale) < math.inf):
        return False
    q = ts[0]
    if isinstance(q, FakeTensor) or not q.is_cuda or q.dim() != 4 or int(q.shape[-1]) not in HEAD_DIMS:
        return False
    return all(not isinstance(t, FakeTensor) and t.dtype == torch.bfloat16 and t.device == q.device
               and t.shape == q.shape and t.stride(-1) == 1 and t.data_ptr() % 16 == 0
               and all(s > 0 and s % 8 == 0 for s in t.stride()[:3]) for t in ts)


def _aligned(*ts):
    """ts with every tensor whose data is not 16-byte aligned replaced by an aligned copy: ATen's
    CUDA flash kernels fault on misaligned pointers instead of refusing them."""
    return [t if t.data_ptr() % 16 == 0 else t.clone(memory_format=torch.contiguous_format) for t in ts]


def _scale(q, scale):
    return float(scale) if scale is not None else q.shape[-1] ** -0.5


def _strides(*ts):
    return (ctypes.c_int64 * (3 * len(ts)))(*[s for t in ts for s in t.stride()[:3]])


def _op(aten_op, q):
    return aten_op or ("cpu" if q.device.type == "cpu" else "flash")


def attention_fwd(q, k, v, is_causal=False, scale=None, out_stride=None, lse_stride=None, aten_op=None):
    """(out, lse) of softmax(scale·q·kᵀ [causal]) v for q, k, v [B, H, T, hd]; scale None means
    1/sqrt(hd).  out is written with `out_stride` (default: the [B, T, H, hd] buffer that
    `out.transpose(1, 2).contiguous()` reads for free), lse [B, H, T] fp32 with `lse_stride`
    (default contiguous; four strides give cuDNN's [B, H, T, 1]).  Off the kernel: the ATen op
    `aten_op` names (default: the flash op of q's device), its (out, lse)."""
    if not _supported(scale, q, k, v):
        if not isinstance(q, FakeTensor):
            _stats["aten_attn_fwd"] += 1
        op = _op(aten_op, q)
        if op == "cpu":
            return FWD_OPS[op](q, k, v, 0.0, is_causal, scale=scale)
        if op == "cudnn":
            r = FWD_OPS[op](*_aligned(q, k, v), None, True, 0.0, is_causal, False, scale=scale)
        else:
            r = FWD_OPS[op](*_aligned(q, k, v), 0.0, is_causal, False, scale=scale)
        return r[0], r[1]
    B, H, T, hd = q.shape
    if out_stride is None:
        out = q.new_empty((B, T, H, hd)).transpose(1, 2)
    else:
        out = q.new_empty_strided(q.shape, out_stride)
    lse = (q.new_empty((B, H, T), dtype=torch.float32) if lse_stride is None
           else q.new_empty_strided((B, H, T, 1)[:len(lse_stride)], lse_stride, dtype=torch.float32))
    if not _supported(scale, out) or lse.data_ptr() % 4:
        # a layout the kernel cannot write: compute into its own and copy over
        o2, l2 = attention_fwd(q, k, v, is_causal, scale)
        out.copy_(o2)
        lse.view(B, H, T).copy_(l2)
        return out, lse
    st = (ctypes.c_int64 * 15)(*_strides(q, k, v, out), *lse.stride()[:3])
    check(_lib.load().edb_attn_fwd(out.data_ptr(), lse.data_ptr(), q.data_ptr(), k.data_ptr(),
                                   v.data_ptr(), B, H, T, hd, st, _scale(q, scale), int(bool(is_causal)),
                                   _stream(q)))
    _stats["edb_attn_fwd"] += 1
    return out, lse


def attention_bwd(dout, q, k, v, out, lse, is_causal=False, scale=None, strides=None, aten_op=None):
    """(dq, dk, dv) of attention_fwd(q, k, v, is_causal, scale) = (out, lse) for the output
    gradient dout; `strides`, when given, the strides of dq, dk and dv (default contiguous).
    Deterministic on the kernel.  Off the kernel: the ATen backward `aten_op` names (default: the
    flash backward of q's device)."""
    if not _supported(scale, dout, q, k, v, out):
        if not isinstance(q, FakeTensor):
            _stats["aten_attn_bwd"] += 1
        op = _op(aten_op, q)
        if op == "cpu":
            return BWD_OPS[op](dout, q, k, v, out, lse, 0.0, is_causal, scale=scale)
        T = q.shape[2]
        seed = torch.empty((2,), dtype=torch.uint64, device=q.device)
        offset = torch.empty((), dtype=torch.uint64, device=q.device)
        args = _aligned(dout, q, k, v, out, lse)
        if op == "cudnn":
            return BWD_OPS[op](*args, seed, offset, None, None, None, T, T, 0.0, is_causal, scale=scale)
        return BWD_OPS[op](*args, None, None, T, T, 0.0, is_causal, seed, offset, scale=scale)
    B, H, T, hd = q.shape
    grads = [q.new_empty_strided(q.shape, s) if s is not None else q.new_empty(q.shape)
             for s in (strides or (None, None, None))]
    if not _supported(scale, *grads):
        got = attention_bwd(dout, q, k, v, out, lse, is_causal, scale)
        for g, x in zip(grads, got):
            g.copy_(x)
        return tuple(grads)
    if lse.dtype != torch.float32 or lse.data_ptr() % 4 or tuple(lse.shape[:3]) != (B, H, T) \
            or lse.numel() != B * H * T:
        raise ValueError(f"attention_bwd: lse {tuple(lse.shape)} {lse.dtype}, want ({B}, {H}, {T}) fp32")
    lib = _lib.load()
    nbytes = ctypes.c_size_t()
    check(lib.edb_attn_bwd_workspace(B, H, T, ctypes.byref(nbytes)))
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=q.device)
    dq, dk, dv = grads
    st = (ctypes.c_int64 * 27)(*_strides(dout, q, k, v, out, dq, dk, dv), *lse.stride()[:3])
    check(lib.edb_attn_bwd(dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), dout.data_ptr(), q.data_ptr(),
                           k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(), ws.data_ptr(), B,
                           H, T, hd, st, _scale(q, scale), int(bool(is_causal)), _stream(q)))
    _stats["edb_attn_bwd"] += 1
    return dq, dk, dv
