"""Host side of the compute dispatch (norm.py, loss.py, optim.py) with the C-ABI mocked out: which
shapes / dtypes / layouts reach which entry point with which arguments, and what goes to ATen
(counted) instead — no GPU, no compute."""
import ctypes

import pytest
import torch

from easydist_b200 import _lib, loss, norm, optim


class _FakeLib:
    def __init__(self):
        self.calls = []
        self.peeks = {}   # entry point -> [(argument index, element count, dtype)] to copy at call time
        self.seen = []    # (entry point, argument index, the memory that pointer addressed)

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            for i, n, dt in self.peeks.get(name, ()):
                nbytes = n * torch.finfo(dt).bits // 8
                raw = (ctypes.c_char * nbytes).from_address(args[i])
                self.seen.append((name, i, torch.frombuffer(bytearray(raw), dtype=dt)))
            if name.endswith("_workspace"):
                args[-1]._obj.value = 1024          # byref(c_size_t)
            return 0
        return fn


@pytest.fixture
def lib(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(_lib, "load", lambda *a, **k: fake)
    for mod in (norm, loss):
        monkeypatch.setattr(mod, "_stream", lambda t: None)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: type("S", (), {"cuda_stream": 0})())
    for m in (norm, loss, optim):
        m.reset_stats()
    return fake


def test_layer_norm_shapes_the_kernel_takes(lib):
    x = torch.zeros(6, 7, 1024, dtype=torch.bfloat16)
    w = torch.ones(1024, dtype=torch.bfloat16)
    y, mean, rstd = norm.native_layer_norm(x, [1024], w, w, 1e-5)
    (name, a), = lib.calls
    assert name == "edb_layer_norm_fwd" and a[6:8] == (42, 1024)       # rows, H
    assert a[9] == _lib.DTYPE_CODES["bfloat16"] and abs(a[8] - 1e-5) < 1e-12
    assert y.shape == x.shape and mean.shape == (6, 7, 1) and mean.dtype == torch.float32
    # H = 100 is outside the kernel's contract: ATen, counted
    norm.native_layer_norm(torch.zeros(4, 100), [100], torch.ones(100), None, 1e-5)
    assert norm.stats()["edb_ln_fwd"] == 1 and norm.stats()["aten_ln"] == 1


def test_column_sum_dispatch_conditions(lib):
    x = torch.zeros(4096, 1024, dtype=torch.bfloat16)
    out = norm.sum_dim_intlist(x, [0], True)
    name, a = lib.calls[-1]
    assert name == "edb_colsum" and a[3:6] == (4096, 1024, 1024) and out.shape == (1, 1024)
    lib.calls.clear()
    for bad in (torch.zeros(8, 1024, dtype=torch.bfloat16),          # too few rows
                torch.zeros(4096, 1030, dtype=torch.bfloat16),       # cols % 8
                torch.zeros(2, 64, 64)):                             # not 2-D
        norm.sum_dim_intlist(bad, [0], True)
    assert not lib.calls and norm.stats()["aten_sum"] == 3
    assert norm.sum_dim_intlist(torch.ones(4, 4), [1], False).tolist() == [4.0] * 4


def test_cross_entropy_passes_strides_and_builds_a_tma_legal_gradient(lib):
    rows, vocab = 8, 50257
    logits = torch.zeros(rows, 50264, dtype=torch.bfloat16)[:, :vocab]     # padded GEMM output
    target = torch.zeros(rows, dtype=torch.int64)
    l, tw, lse = loss.cross_entropy_fwd(logits, target, -100, 1)
    name, a = lib.calls[-1]
    assert name == "edb_cross_entropy_fwd"
    assert a[5] == 50264 and a[7:12] == (rows, vocab, -100, 1, _lib.DTYPE_CODES["bfloat16"])
    assert l.shape == () and tw.shape == () and lse.shape == (rows,) and lse.dtype == torch.float32
    dx = loss.cross_entropy_bwd(torch.ones(()), logits, target, lse, tw, -100, 1)
    name, a = lib.calls[-1]
    assert name == "edb_cross_entropy_bwd" and a[1] == 50264 and a[3] == 50264
    assert dx.shape == (rows, vocab) and dx.stride() == (50264, 1) and dx.dtype == torch.bfloat16
    # 3-D logits or int32 targets are not this kernel's case
    lib.calls.clear()
    loss.cross_entropy_fwd(torch.zeros(4, 10, dtype=torch.float64), torch.zeros(4, dtype=torch.int64), -100, 1)
    assert not lib.calls and loss.stats()["aten_ce"] == 1


def test_sgd_splits_the_lists_between_the_kernel_and_aten(lib):
    def trio(n, dtype=torch.float32):
        return torch.zeros(n, dtype=dtype), torch.ones(n, dtype=dtype), torch.zeros(n, dtype=dtype)

    a, b = trio(64), trio(32, torch.bfloat16)
    base = torch.zeros(40)
    c = (base[1:33], torch.ones(32), torch.zeros(32))                    # not 16-byte aligned
    params, grads, bufs = zip(a, b, c)
    optim.sgd_momentum_(list(params), list(grads), list(bufs), 0.9, 1, -0.1)
    kinds = sorted((name, args[0], args[8]) for name, args in lib.calls)
    assert kinds == sorted([("edb_sgd_momentum", 1, _lib.DTYPE_CODES["bfloat16"]),
                            ("edb_sgd_momentum", 1, _lib.DTYPE_CODES["float32"])])
    assert optim.stats() == {"edb_sgd": 2, "aten_sgd": 1}
    assert torch.allclose(c[0], torch.full((32,), -0.1))                 # the ATen group really ran
    with pytest.raises(ValueError):
        optim.sgd_momentum_([a[0]], [], [a[2]], 0.9, 1, -0.1)


# ---- layouts of the norm operands -------------------------------------------------------------

def _at_offset(t, k):
    """t's values in a contiguous view that starts k elements into a wider buffer (k = 1, 2, 3: not
    16-byte aligned for 2- and 4-byte types)."""
    buf = torch.full((t.numel() + k + 8,), float("nan"), dtype=t.dtype)
    v = buf[k:k + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def _strided(t):
    """t's values at every second element of a buffer twice as long (the padding is NaN)."""
    buf = torch.full((t.numel() * 2,), float("nan"), dtype=t.dtype)
    v = buf[::2]
    v.copy_(t.reshape(-1))
    return v.view(t.shape) if t.dim() == 1 else v.reshape(t.shape)


def _ptr_ok(name, a, idx):
    return all(a[i] is None or a[i] % 16 == 0 for i in idx), (name, [a[i] for i in idx])


_LN_FWD_PTRS, _LN_BWD_PTRS = (0, 1, 2, 3, 4, 5), (0, 1, 2, 3, 4, 7, 8, 9)
_RMS_FWD_PTRS, _RMS_BWD_PTRS = (0, 1, 2, 3), (0, 1, 2, 3, 5, 6, 7)


@pytest.mark.parametrize("which", ["weight", "bias"])
@pytest.mark.parametrize("layout", ["stride2", "offset1", "offset3"])
def test_layer_norm_weight_and_bias_reach_the_kernel_dense_and_aligned(lib, which, layout):
    """The kernel reads H consecutive elements at the weight / bias pointer: a strided or misaligned
    parameter must arrive as a dense, aligned copy holding the same values."""
    H = 256
    g = torch.Generator().manual_seed(1)
    x = torch.randn(4, H, generator=g).bfloat16()
    w, b = torch.randn(H, generator=g).bfloat16(), torch.randn(H, generator=g).bfloat16()
    make = _strided if layout == "stride2" else (lambda t: _at_offset(t, int(layout[-1])))
    wv, bv = (make(w), b) if which == "weight" else (w, make(b))
    pos = 4 if which == "weight" else 5
    lib.peeks = {"edb_layer_norm_fwd": [(pos, H, torch.bfloat16)],
                 "edb_layer_norm_bwd_add": [(7, H, torch.bfloat16)]}
    norm.native_layer_norm(x, [H], wv, bv, 1e-5)
    name, a = lib.calls[-1]
    assert name == "edb_layer_norm_fwd" and _ptr_ok(name, a, _LN_FWD_PTRS)[0]
    assert a[pos] != (wv if which == "weight" else bv).data_ptr()
    assert torch.equal(lib.seen[-1][2], w if which == "weight" else b)
    mean = torch.zeros(4, 1)
    norm.native_layer_norm_backward(x, x, [H], mean, mean, wv, bv, [True, True, True])
    name, a = lib.calls[-1]
    assert name == "edb_layer_norm_bwd_add" and _ptr_ok(name, a, _LN_BWD_PTRS)[0]
    assert torch.equal(lib.seen[-1][2], w)
    assert norm.stats()["aten_ln"] == 0


@pytest.mark.parametrize("k", [1, 2, 3])
def test_misaligned_norm_activations_reach_the_kernel_aligned(lib, k):
    """x, dy and the accumulated gradient `_add` at a storage offset that breaks 16-byte alignment:
    `.contiguous()` would hand them over unmoved, and the kernel rejects them."""
    g = torch.Generator().manual_seed(k)
    for dt, H in ((torch.bfloat16, 256), (torch.float32, 128)):
        x, dy, add = (torch.randn(3, H, generator=g).to(dt) for _ in range(3))
        w = torch.randn(H, generator=g).to(dt)
        xo, dyo, addo = (_at_offset(t, k) for t in (x, dy, add))
        stat = torch.zeros(3, 1)
        lib.calls.clear()
        lib.peeks = {"edb_layer_norm_fwd": [(3, 3 * H, dt)],
                     "edb_layer_norm_bwd_add": [(3, 3 * H, dt), (4, 3 * H, dt), (8, 3 * H, dt)],
                     "edb_rms_norm_fwd": [(2, 3 * H, dt)],
                     "edb_rms_norm_bwd": [(2, 3 * H, dt), (3, 3 * H, dt), (6, 3 * H, dt)]}
        lib.seen.clear()
        norm.native_layer_norm(xo, [H], w, w, 1e-5)
        norm.native_layer_norm_backward(dyo, xo, [H], stat, stat, w, w, [True, True, True], _add=addo)
        for mode in (norm.RMS_CAST_THEN_SCALE, norm.RMS_FUSED):
            norm.rms_norm_fwd(xo, w, 1e-5, mode)
            norm.rms_norm_bwd(dyo, xo, stat, w, mode, [True, True], _add=addo)
        names = [c[0] for c in lib.calls if not c[0].endswith("_workspace")]
        assert names == ["edb_layer_norm_fwd", "edb_layer_norm_bwd_add"] + \
            ["edb_rms_norm_fwd", "edb_rms_norm_bwd"] * 2
        ptrs = {"edb_layer_norm_fwd": _LN_FWD_PTRS, "edb_layer_norm_bwd_add": _LN_BWD_PTRS,
                "edb_rms_norm_fwd": _RMS_FWD_PTRS, "edb_rms_norm_bwd": _RMS_BWD_PTRS}
        for name, a in lib.calls:
            if name in ptrs:
                ok, got = _ptr_ok(name, a, ptrs[name])
                assert ok, (dt, got)
        want = {3: x, 4: x, 8: add, 2: x, 6: add}
        want_ln_bwd = {3: dy, 4: x, 8: add}
        want_rms_bwd = {2: dy, 3: x, 6: add}
        for name, i, got in lib.seen:
            ref = want_ln_bwd[i] if name == "edb_layer_norm_bwd_add" else \
                want_rms_bwd[i] if name == "edb_rms_norm_bwd" else want[i]
            assert torch.equal(got, ref.reshape(-1)), (dt, name, i)
    assert norm.stats()["aten_ln"] == 0 and norm.stats()["aten_rms"] == 0


def test_dense_aligned_norm_operands_reach_the_kernel_without_a_copy(lib):
    H = 512
    x, dy, add = (torch.randn(5, H).bfloat16() for _ in range(3))
    w, b = torch.randn(H).bfloat16(), torch.randn(H).bfloat16()
    stat = torch.zeros(5, 1)
    norm.native_layer_norm(x, [H], w, b, 1e-5)
    norm.native_layer_norm_backward(dy, x, [H], stat, stat, w, b, [True, True, True], _add=add)
    norm.rms_norm_fwd(x, w, 1e-5, norm.RMS_FUSED)
    norm.rms_norm_bwd(dy, x, stat, w, norm.RMS_FUSED, [True, True], _add=add)
    calls = {name: a for name, a in lib.calls}
    p = lambda t: t.data_ptr()
    assert calls["edb_layer_norm_fwd"][3:6] == (p(x), p(w), p(b))
    a = calls["edb_layer_norm_bwd_add"]
    assert (a[3], a[4], a[7], a[8]) == (p(dy), p(x), p(w), p(add))
    assert calls["edb_rms_norm_fwd"][2:4] == (p(x), p(w))
    a = calls["edb_rms_norm_bwd"]
    assert (a[2], a[3], a[5], a[6]) == (p(dy), p(x), p(w), p(add))
