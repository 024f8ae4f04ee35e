"""Sharded-op kernel dispatch for token and position embeddings on edb_embed.cu of libedb.so.

Traced, an embedding is `aten.embedding(W, idx)` forward (GPT-2 adds `aten.embedding(P, pos)` with an
`aten.add`) and `aten.embedding_dense_backward(dy, idx, V, padding_idx, False)` backward; a tied
LM-head weight then gets `aten.add(mm_lm_wgrad, embedding_dense_backward(...))`.  `embedding_fwd`
replaces the forward (one gather pass, bit-identical), `embedding_bwd` the dense backward (a
deterministic sort-based sum instead of a zero fill, a radix sort and segment kernels), and
`embedding_bwd_acc_` the tied add: the embedding gradient is added in place into the LM-head
gradient, touching only the rows the tokens index.  On FakeTensors, CPU tensors, other dtypes,
tables that are not contiguous or `acc` whose rows are not contiguous, the replaced ATen ops run op
for op and the call is counted as `aten_embed`.  scale_grad_by_freq and sparse gradients are never
routed here (lowering.fuse_embedding leaves them alone)."""
from ctypes import byref, c_size_t

import torch
from torch._subclasses.fake_tensor import FakeTensor
from torch.fx.node import has_side_effect

from . import _lib
from ._lib import check
from .norm import _DT, _dense, _stream

aten = torch.ops.aten
_IDX = {torch.int32: _lib.DTYPE_CODES["int32"], torch.int64: _lib.DTYPE_CODES["int64"]}
_stats = {"edb_embed_fwd": 0, "edb_embed_bwd": 0, "edb_embed_bwd_acc": 0, "aten_embed": 0}
_workspaces = {}


def stats():
    return dict(_stats)


def reset_stats():
    for k in _stats:
        _stats[k] = 0


def _count_aten(t):
    if not isinstance(t, FakeTensor):
        _stats["aten_embed"] += 1


def _table_ok(w, dtype, device):
    return (w.dim() == 2 and w.dtype == dtype and w.device == device and w.is_contiguous()
            and w.shape[1] > 0)


def _idx_ok(idx, device):
    return idx.dtype in _IDX and idx.device == device


def embedding_fwd(W, idx, P=None, pos=None):
    """`aten.embedding(W, idx)` [+ `aten.embedding(P, pos)`, pos [T] broadcast over idx's leading
    dimensions]: y[..., t, :] = T(float(W[idx[..., t]]) + float(P[pos[t]])), bit-identical to the
    ATen ops.  Ids outside the table read zeros on the kernel (ATen's device assert fires instead)."""
    ok = not isinstance(W, FakeTensor) and W.is_cuda and W.dtype in _DT \
        and _table_ok(W, W.dtype, W.device) and _idx_ok(idx, W.device)
    if ok and P is not None:
        ok = _table_ok(P, W.dtype, W.device) and P.shape[1] == W.shape[1] and pos.dim() == 1 \
            and _idx_ok(pos, W.device) and pos.dtype == idx.dtype and idx.dim() >= 1 \
            and idx.shape[-1] == pos.shape[0] and pos.numel() > 0
    if not ok:
        _count_aten(W)
        y = aten.embedding.default(W, idx)
        return y if P is None else aten.add.Tensor(y, aten.embedding.default(P, pos))
    C = int(W.shape[1])
    y = W.new_empty(tuple(idx.shape) + (C,))
    ix = _dense(idx)
    ps = _dense(pos) if P is not None else None
    check(_lib.load().edb_embedding_fwd(
        y.data_ptr(), W.data_ptr(), ix.data_ptr(), P.data_ptr() if P is not None else None,
        ps.data_ptr() if ps is not None else None, idx.numel(), C, W.shape[0],
        P.shape[0] if P is not None else 0, pos.numel() if P is not None else 0, _IDX[idx.dtype],
        _DT[W.dtype], _stream(W)))
    _stats["edb_embed_fwd"] += 1
    return y


def _workspace(rows, V, device):
    key = (rows, V, device)
    ws = _workspaces.get(key)
    if ws is None:
        nbytes = c_size_t()
        check(_lib.load().edb_embedding_bwd_workspace(rows, V, byref(nbytes)))
        ws = _workspaces[key] = torch.empty(max(16, nbytes.value), dtype=torch.uint8, device=device)
    return ws


def _bwd_ok(dy, idx):
    return not isinstance(dy, FakeTensor) and dy.is_cuda and dy.dtype in _DT and dy.dim() >= 1 \
        and dy.shape[-1] > 0 and _idx_ok(idx, dy.device) \
        and tuple(dy.shape[:-1]) == tuple(idx.shape)


def _launch(out, ld_out, dy, idx, V, padding_idx, accumulate):
    C = int(dy.shape[-1])
    d, ix = _dense(dy), _dense(idx)
    rows = ix.numel()
    ws = _workspace(rows, V, dy.device)
    check(_lib.load().edb_embedding_bwd(out.data_ptr(), ld_out, d.data_ptr(), C, ix.data_ptr(),
                                        ws.data_ptr(), rows, C, V, int(padding_idx),
                                        int(accumulate), _IDX[idx.dtype], _DT[dy.dtype],
                                        _stream(dy)))


def embedding_bwd(dy, idx, V, padding_idx=-1):
    """`aten.embedding_dense_backward(dy, idx, V, padding_idx, False)`: the [V, C] gradient,
    g[v] = T(sum of dy over the positions with idx == v), summed in fp32 in increasing position
    (deterministic); zeros for padding_idx and for rows nothing indexed.  Ids outside [0, V) are
    skipped on the kernel."""
    if not _bwd_ok(dy, idx):
        _count_aten(dy)
        return aten.embedding_dense_backward.default(dy, idx, V, padding_idx, False)
    C = int(dy.shape[-1])
    out = dy.new_empty((int(V), C))
    _launch(out, C, dy, idx, int(V), padding_idx, False)
    _stats["edb_embed_bwd"] += 1
    return out


@has_side_effect
def embedding_bwd_acc_(acc, dy, idx, padding_idx=-1):
    """In place, and returns acc: `acc + aten.embedding_dense_backward(dy, idx, V, padding_idx,
    False)` with V = acc.shape[0].  acc[v] = T(float(acc[v]) + float(g[v])) for the indexed rows
    other than padding_idx (g as in embedding_bwd, rounded to T first); the kernel neither reads
    nor writes any other row of acc."""
    ok = _bwd_ok(dy, idx) and acc.dim() == 2 and acc.dtype == dy.dtype and acc.device == dy.device \
        and acc.shape[1] == dy.shape[-1] and acc.stride(1) == 1 and acc.stride(0) >= acc.shape[1]
    if not ok:
        _count_aten(dy)
        return aten.add_.Tensor(acc, aten.embedding_dense_backward.default(
            dy, idx, acc.shape[0], padding_idx, False))
    _launch(acc, acc.stride(0), dy, idx, int(acc.shape[0]), padding_idx, True)
    _stats["edb_embed_bwd_acc"] += 1
    return acc
