"""Column sums, LayerNorm dw / db and cross-entropy (H100) against the float64 bounds of
tests/reduce_ref.py, which follow each kernel's summation order.  The largest err / bound of each group
is printed at the end of the module (pytest -s)."""
import math

import pytest
import torch

from tests import reduce_ref as R
from tests.test_gpu_kernel_sweep import LN_WIDTHS

pytestmark = pytest.mark.gpu
_WORST = {}
DT_IDS = ["bf16", "fp32"]
DTYPES = [torch.bfloat16, torch.float32]


@pytest.fixture(scope="module")
def rt():
    from easydist_b200 import runtime
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    r = runtime.init(rank=0, world=1, device=0, heap_bytes=2 << 30) \
        if not runtime.is_initialized() else runtime.get_runtime()
    yield r
    if _WORST:
        print("\nlargest err/bound per group: " +
              ", ".join(f"{k} {v:.3f}" for k, v in sorted(_WORST.items())))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _record(group, q, what):
    _WORST[group] = max(_WORST.get(group, 0.0), q)
    assert q <= 1.0, (group, what, q)


def _check(group, got, ref, bound, what):
    _record(group, R.worst(got, ref, bound), what)


def _sentinel(n, dtype):
    return (torch.arange(n, device="cuda") % 251 - 125).to(dtype)


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


# ---- column sums ---------------------------------------------------------------------------------

COLSUM_ROWS = [64, 65, 127, 8192 + 1, 32768]


def _colsum_cols(dtype):
    n = R.epv(dtype)
    return [n, 31 * n, 32 * n, 33 * n, 1032, 3072, 50264]


def _colsum_check(group, got, x, sms):
    rows, cols = x.shape
    s64, A = R.colsum_ref(x)
    bound = R.colsum_bound(s64, A, R.colsum_depth(rows, cols, x.dtype, sms), x.dtype)
    _check(group, got.reshape(-1), s64, bound, (rows, cols))


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_colsum_matches_fp64_bound(rt, dtype):
    """Every stripe shape (one vector column, 31 / 32 / 33 lanes' worth, a partial last stripe,
    the GPT-2 widths), the 64-row minimum, partial splits, the 128-split cap, data at scale 1 and
    1e-3, keepdim both ways.  32768 x 50264 is left out: its float64 reference alone is 13 GB."""
    from easydist_b200 import norm
    torch.manual_seed(20)
    sms, i, configs = _sms(), 0, set()
    for cols in _colsum_cols(dtype):
        for rows in COLSUM_ROWS:
            if rows * cols > 5e8:
                continue
            splits, rps = R.colsum_config(rows, cols, dtype, sms)
            configs.add((splits == 128, splits > 1 and rows % rps != 0))
            for scale in (1.0, 1e-3):
                x = (torch.randn(rows, cols, device="cuda") * scale).to(dtype)
                keepdim = i % 2 == 0
                i += 1
                norm.reset_stats()
                got = norm.sum_dim_intlist(x, [0], keepdim)
                assert norm.stats()["edb_colsum"] == 1, (rows, cols)
                assert got.shape == ((1, cols) if keepdim else (cols,)) and got.dtype == dtype
                _colsum_check("colsum_" + DT_IDS[DTYPES.index(dtype)], got, x, sms)
    assert (True, False) in configs and (False, True) in configs, configs  # cap, partial last split


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_colsum_strided_cached_guarded_and_graphed(rt, dtype):
    """ld > cols with poisoned padding columns; two row counts on one cached workspace (many splits,
    then one); `out` inside guard elements through the C-ABI; the same bits on a repeat and from a
    CUDA-graph replay, also after new values are written into the input."""
    from ctypes import byref, c_size_t

    from easydist_b200 import _lib, norm
    from easydist_b200._lib import check
    torch.manual_seed(21)
    sms, n, group = _sms(), R.epv(dtype), "colsum_misc_" + DT_IDS[DTYPES.index(dtype)]
    for cols in (32 * n, 1032):
        for pad in (n, 64):
            buf = torch.full((4096, cols + pad), 1e4, device="cuda", dtype=dtype)
            x = buf[:, :cols]
            x.copy_(torch.randn(4096, cols, device="cuda"))
            norm.reset_stats()
            got = norm.sum_dim_intlist(x, [0], True)
            assert norm.stats()["edb_colsum"] == 1 and x.stride(0) == cols + pad
            _colsum_check(group, got, x, sms)
    cols = 1024
    big = torch.randn(32768, cols, device="cuda").to(dtype)
    small = torch.randn(65, cols, device="cuda").to(dtype)
    assert R.colsum_config(32768, cols, dtype, sms)[0] > 1
    assert R.colsum_config(65, cols, dtype, sms)[0] == 1
    first = norm.sum_dim_intlist(big, [0], True)
    second = norm.sum_dim_intlist(small, [0], True)
    _colsum_check(group, first, big, sms)
    _colsum_check(group, second, small, sms)
    assert torch.equal(norm.sum_dim_intlist(big, [0], True), first)
    assert torch.equal(norm.sum_dim_intlist(small, [0], True), second)
    # guard elements around out
    lib = _lib.load()
    for cols, rows in ((1032, 777), (n, 8193)):
        x = torch.randn(rows, cols, device="cuda").to(dtype)
        nbytes = c_size_t()
        check(lib.edb_colsum_workspace(cols, byref(nbytes)))
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device="cuda")
        guard = 64
        sentinel = _sentinel(cols + 2 * guard, dtype)
        out = sentinel.clone()
        check(lib.edb_colsum(out.data_ptr() + guard * out.element_size(), x.data_ptr(), ws.data_ptr(),
                             rows, cols, x.stride(0), norm._DT[dtype],
                             torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        inner = torch.zeros_like(out, dtype=torch.bool)
        inner[guard:guard + cols] = True
        assert torch.equal(_bits(out)[~inner], _bits(sentinel)[~inner]), (rows, cols)
        _colsum_check(group, out[guard:guard + cols], x, sms)
    # CUDA graph
    x = torch.randn(8193, 1032, device="cuda").to(dtype)
    eager = norm.sum_dim_intlist(x, [0], True)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = norm.sum_dim_intlist(x, [0], True)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    x.copy_(torch.randn(x.shape, device="cuda"))
    g.replay()
    eager = norm.sum_dim_intlist(x, [0], True)
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    _colsum_check(group, out, x, sms)


# ---- LayerNorm dw / db ---------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_layer_norm_dw_db_match_fp64_bound(rt, dtype):
    """Every width, rows from one CTA to several passes of the persistent grid: a shrunk grid
    (4 * sms + 3 rows), exactly one pass (8 * sms), one row more, and 8192; dy at gradient scale."""
    from easydist_b200 import norm
    torch.manual_seed(22)
    sms, dt = _sms(), DT_IDS[DTYPES.index(dtype)]
    for H in LN_WIDTHS[dtype]:
        for rows in (1, 4 * sms + 3, 8 * sms, 8 * sms + 1, 8192):
            x = torch.randn(rows, H, device="cuda").to(dtype)
            w = (torch.randn(H, device="cuda") * 0.5 + 1).to(dtype)
            b = torch.randn(H, device="cuda").to(dtype)
            dy = (torch.randn(rows, H, device="cuda") * 1e-2).to(dtype)
            norm.reset_stats()
            _, mean, rstd = norm.native_layer_norm(x, [H], w, b, 1e-5)
            _, dw, db = norm.native_layer_norm_backward(dy, x, [H], mean, rstd, w, b, [True, True, True])
            assert norm.stats()["edb_ln_bwd"] == 1 and norm.stats()["aten_ln"] == 0
            dw64, db64, Sw, Sb, Dx = R.ln_dwdb_ref(dy, x, mean, rstd, 1e-5)
            depth = R.ln_depth(rows, sms)
            _check("ln_dw_" + dt, dw, dw64, R.ln_dw_bound(dw64, Sw, Dx, depth, dtype), (H, rows))
            _check("ln_db_" + dt, db, db64, R.ln_db_bound(db64, Sb, depth, dtype), (H, rows))


# ---- cross-entropy -------------------------------------------------------------------------------

CE_VOCABS = [1, 7, None, 2049, 50257, 50304]  # None: one vector (EPV)
CE_ROWS = [1, 3, 1024, 1025, 4097]
LAYOUTS = ["contig", "padded", "misaligned"]


def _logits(rows, vocab, dtype, layout, scale=1.0, shift=0.0):
    """contig: ld = vocab; padded: ld = vocab rounded up to 8, + 8; misaligned: that ld, base one
    element past a 16-byte boundary.  Padding is poisoned with 1e4."""
    vals = torch.randn(rows, vocab, device="cuda") * scale + shift
    if layout == "contig":
        return vals.to(dtype)
    ld = (vocab + 7) // 8 * 8 + 8
    if layout == "padded":
        x = torch.full((rows, ld), 1e4, device="cuda", dtype=dtype)[:, :vocab]
    else:
        flat = torch.full((rows * ld + 8,), 1e4, device="cuda", dtype=dtype)
        x = flat[1:1 + rows * ld].view(rows, ld)[:, :vocab]
    x.copy_(vals)
    return x


def _targets(rows, vocab, dtype, ignore_index=-100, every=7):
    """Random targets, plus 0, vocab - 1 (in the scalar tail when vocab % EPV != 0), every lane of
    one vector, and ignored rows."""
    n = R.epv(dtype)
    t = torch.randint(0, vocab, (rows,), device="cuda")
    if rows > 2:
        t[2::every] = ignore_index
    t[0] = 0
    if rows > 1:
        t[1] = vocab - 1
    if rows > 3 + n and vocab >= 2 * n:
        t[3:3 + n] = torch.arange(n, 2 * n, device="cuda")
    return t


def _ce_run(x, target, ign, red, go):
    from easydist_b200 import loss
    loss.reset_stats()
    l, tw, lse = loss.cross_entropy_fwd(x, target, ign, red)
    dx = loss.cross_entropy_bwd(torch.full((), go, device="cuda"), x, target, lse, tw, ign, red)
    st = loss.stats()
    assert st["edb_ce_fwd"] == 1 and st["edb_ce_bwd"] == 1 and st["aten_ce"] == 0, st
    return l, tw, lse, dx


def _ce_check(group, x, target, ign, red, go, l, tw, lse, dx):
    vec = R.ce_vec_fwd(x)
    ref = R.ce_ref(x, target, ign, red, go)
    what = (tuple(x.shape), x.stride(0), vec, red, go)
    assert float(tw) == ref["count"], what
    if ref["count"] == 0 and red == 1:
        assert math.isnan(float(l)), what  # 0 / 0, as ATen
    else:
        q = abs(float(l) - float(ref["loss"])) / R.ce_loss_bound(ref, x.dtype, vec, red)
        _record(group + "_loss", q, what)
    _check(group + "_lse", lse, ref["lse"], R.ce_lse_bound(ref, x.dtype, vec), what)
    assert dx.dtype == x.dtype and dx.shape == x.shape
    _check(group + "_dx", dx, ref["dx"], R.ce_dx_bound(ref, x.dtype, vec), what)
    assert bool((dx[~ref["keep"]] == 0).all()), what
    if dx.stride(0) != x.shape[1]:
        pad = dx.as_strided((x.shape[0], dx.stride(0) - x.shape[1]), (dx.stride(0), 1),
                            dx.storage_offset() + x.shape[1])
        assert bool((pad == 0).all()), what
    return vec


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_cross_entropy_matches_fp64_bound(rt, dtype):
    """Every vocabulary x row count, the layout cycling through contig / padded / misaligned (so both
    the 16-byte and the scalar path at small and large vocabularies), reduction and grad_out (0.5,
    -3) alternating, logit scale 1, 3 or 30."""
    torch.manual_seed(23)
    dt, n = DT_IDS[DTYPES.index(dtype)], R.epv(dtype)
    paths, i = set(), 0
    for vocab in CE_VOCABS:
        vocab = vocab or n
        for rows in CE_ROWS:
            layout = LAYOUTS[i % 3]
            red, go, scale = 1 + i % 2, (0.5, -3.0)[(i // 2) % 2], (1.0, 3.0, 30.0)[(i // 3) % 3]
            i += 1
            x = _logits(rows, vocab, dtype, layout, scale)
            t = _targets(rows, vocab, dtype)
            vec = _ce_check("ce_" + dt, x, t, -100, red, go, *_ce_run(x, t, -100, red, go))
            paths.add((vocab > 1000, vec))
    assert paths == {(False, False), (False, True), (True, False), (True, True)}, paths


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_cross_entropy_edges(rt, dtype):
    """ignore_index 0 (a valid class), all rows ignored (mean: NaN as ATen, sum: 0, no gradient),
    a +1000 logit shift, -inf in the padding columns 50257..50303 of a 50304 vocabulary."""
    torch.manual_seed(24)
    dt = DT_IDS[DTYPES.index(dtype)]
    for layout in ("contig", "misaligned"):
        x = _logits(1025, 2049, dtype, layout, 3.0)
        t = torch.randint(0, 4, (1025,), device="cuda")
        for red, go in ((1, 0.5), (2, -3.0)):
            _ce_check("ce_edge_" + dt, x, t, 0, red, go, *_ce_run(x, t, 0, red, go))
        t = torch.full((1025,), -100, device="cuda")
        for red in (1, 2):
            l, tw, lse, dx = _ce_run(x, t, -100, red, 0.5)
            assert float(tw) == 0 and bool((dx == 0).all())
            assert math.isnan(float(l)) if red == 1 else float(l) == 0.0
            _ce_check("ce_edge_" + dt, x, t, -100, red, 0.5, l, tw, lse, dx)
    for layout in ("padded", "misaligned"):
        for scale in (1.0, 30.0):
            x = _logits(1024, 2049, dtype, layout, scale, shift=1000.0)
            t = _targets(1024, 2049, dtype)
            _ce_check("ce_shift_" + dt, x, t, -100, 1, 0.5, *_ce_run(x, t, -100, 1, 0.5))
    for layout in ("contig", "misaligned"):
        x = _logits(1025, 50304, dtype, layout, 3.0)
        x[:, 50257:] = -math.inf
        t = _targets(1025, 50257, dtype)
        _ce_check("ce_neginf_" + dt, x, t, -100, 2, -3.0, *_ce_run(x, t, -100, 2, -3.0))


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_cross_entropy_bwd_writes_its_rows_and_zeroes_padding(rt, dtype):
    """dlogits through the C-ABI inside a sentinel buffer: every element outside the rows x ld_out
    block keeps its bits, the padding columns [vocab, ld_out) are zero.  A 16-byte forward with a
    16-byte backward (ld_out % 8 == 0, aligned), and with a scalar backward (ld_out odd, or dx one
    element past a 16-byte boundary)."""
    from easydist_b200 import _lib, loss
    from easydist_b200._lib import check
    torch.manual_seed(25)
    dt, lib = DT_IDS[DTYPES.index(dtype)], _lib.load()
    rows, vocab, ign = 1025, 2049, -100
    x = _logits(rows, vocab, dtype, "padded", 3.0)
    t = _targets(rows, vocab, dtype)
    assert R.ce_vec_fwd(x)
    for red, go in ((1, 0.5), (2, -3.0)):
        l, tw, lse = loss.cross_entropy_fwd(x, t, ign, red)
        g = torch.full((), go, device="cuda")
        for ld_out, shift in (((vocab + 7) // 8 * 8, 0), ((vocab + 7) // 8 * 8 + 1, 0),
                              ((vocab + 7) // 8 * 8, 1)):
            flat0 = _sentinel((rows + 2) * ld_out + 2, dtype)
            flat = flat0.clone()
            off = ld_out + shift
            dx_vec = ld_out % R.epv(dtype) == 0 and (flat.data_ptr() + off * flat.element_size()) % 16 == 0
            assert dx_vec == (ld_out % 2 == 0 and shift == 0)
            check(lib.edb_cross_entropy_bwd(flat.data_ptr() + off * flat.element_size(), ld_out,
                                            x.data_ptr(), x.stride(0), t.data_ptr(), lse.data_ptr(),
                                            g.data_ptr(), tw.data_ptr(), rows, vocab, ign, red,
                                            loss._DT[dtype], torch.cuda.current_stream().cuda_stream))
            torch.cuda.synchronize()
            inside = torch.zeros_like(flat, dtype=torch.bool)
            inside[off:off + rows * ld_out] = True
            assert torch.equal(_bits(flat)[~inside], _bits(flat0)[~inside]), (ld_out, shift)
            dx = flat[off:off + rows * ld_out].view(rows, ld_out)
            assert bool((dx[:, vocab:] == 0).all()), (ld_out, shift)
            _ce_check("ce_guard_" + dt, x, t, ign, red, go, l, tw, lse, dx[:, :vocab])


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_cross_entropy_cuda_graph_matches_eager(rt, dtype):
    """Forward and backward captured in one CUDA graph: the replay equals the eager call bit for
    bit, also after new logits are written into the static input."""
    from easydist_b200 import loss
    torch.manual_seed(26)
    x = _logits(1025, 50257, dtype, "padded", 3.0)
    t = _targets(1025, 50257, dtype)
    g = torch.full((), 0.5, device="cuda")

    def step():
        l, tw, lse = loss.cross_entropy_fwd(x, t, -100, 1)
        return l, lse, loss.cross_entropy_bwd(g, x, t, lse, tw, -100, 1)

    eager = step()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for refill in (False, True):
        if refill:
            x.copy_(torch.randn(x.shape, device="cuda") * 3)
        graph.replay()
        if refill:
            eager = step()
        torch.cuda.synchronize()
        for a, b in zip(out, eager):
            assert torch.equal(a, b), refill
