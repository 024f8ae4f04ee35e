"""The wgmma GEMM and the LayerNorm kernels across their dispatch space (H100), against float64
references of the same operation on the same bf16 / fp32 operands.

GEMM: every operand layout at the default, 128- and 256-wide tiles; tile-edge, unaligned and
persistent (several tiles per CTA) shapes; split-K eligibility, uneven slices and the reduce
kernel's column tail; the fused epilogues; writes outside the M x N box; CUDA-graph capture (same
launches and the same bits as the eager call).  The bound is tests/gemm_ref.py's; the largest
err / bound of each group is printed at the end of the module (pytest -s).
"""
import contextlib
import math

import pytest
import torch

from tests import gemm_ref

pytestmark = pytest.mark.gpu

LAYOUTS = [(True, True), (True, False), (False, True), (False, False)]  # (A K-major, B K-major)
LAYOUT_IDS = ["a_k-b_k", "a_k-b_n", "a_m-b_k", "a_m-b_n"]
_WORST = {}


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


def persistent_shape():
    """>= 3 waves of 128 x 256 tiles whatever the SM count, an M tail, and 7 k-blocks (K = 392: not a
    multiple of the 4- or 6-stage ring, so stage and phase carry over between a CTA's tiles)."""
    n_tiles = 10
    return 128 * math.ceil(3 * _sms() / n_tiles) + 72, 256 * n_tiles, 392


@contextlib.contextmanager
def option(rt, name, value):
    old = rt.get_option(name)
    if value is not None:
        rt.set_option(name, value)
    try:
        yield
    finally:
        rt.set_option(name, old)


def _layout(A, B, a_k, b_k):
    """Views of A [M,K] and B [K,N] with the requested storage order (values unchanged)."""
    a = A if a_k else A.t().contiguous().t()
    b = B.t().contiguous().t() if b_k else B
    return a, b


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).bfloat16()


def _check(group, c, r, bound, what):
    q = gemm_ref.ratio(c, r, bound)
    _WORST[group] = max(_WORST.get(group, 0.0), q)
    assert q <= 1.0, (what, q)


def _splits_expected(M, N, K, sms):
    """Host rule of edb_gemm.cu (no prefetch, no epilogue): split when the tiles fill at most half
    of the SMs and K has >= 16 k-blocks, into min(sms // tiles, k_blocks // 8, 8) slices."""
    bn = 128 if N <= 128 else 256
    tiles = math.ceil(M / 128) * math.ceil(N / bn)
    kb = math.ceil(K / 64)
    return 2 * tiles <= sms and kb >= 16 and min(sms // tiles, kb // 8, 8) > 1


# ---- the sweep -----------------------------------------------------------------------------------

EDGE_SHAPES = [(2, 8, 8), (63, 72, 40), (64, 120, 64), (65, 128, 72), (127, 136, 1000),
               (128, 256, 64), (129, 264, 72), (257, 520, 1000), (65, 8, 1000), (2, 520, 40),
               (257, 128, 8), (127, 264, 64), (128, 128, 1000)]
# formerly checked against an fp32 reference in test_gpu_single.py; the last four run split-K
GEMM_SHAPES = [(128, 128, 64), (128, 256, 128), (256, 512, 256), (384, 200, 136), (100, 72, 40),
               (4096, 1024, 1024), (1024, 4096, 1024), (512, 1024, 4096), (640, 3072, 1024),
               (1024, 1024, 4096), (304, 200, 2056), (128, 256, 2048), (1000, 72, 1544)]
UNALIGNED_SHAPES = [(97, 50, 43), (1000, 1003, 130), (33, 264, 1001)]


@pytest.mark.parametrize("bn", [None, 128, 256], ids=["bn_default", "bn128", "bn256"])
@pytest.mark.parametrize("a_k,b_k", LAYOUTS, ids=LAYOUT_IDS)
def test_gemm_matches_fp64_bound(rt, a_k, b_k, bn):
    """gemm.mm, gemm.addmm and gemm.mm_add at tile edges, unaligned extents (padded staging, never
    ATen) and a persistent grid, every layout, every tile width."""
    from easydist_b200 import gemm
    torch.manual_seed(0)
    with option(rt, "gemm_force_bn", bn):
        for (M, N, K) in EDGE_SHAPES + GEMM_SHAPES + UNALIGNED_SHAPES + [persistent_shape()]:
            A, B = _rand(M, K), _rand(K, N)
            a, b = _layout(A, B, a_k, b_k)
            gemm.reset_stats()
            c = gemm.mm(a, b)
            st = gemm.stats()
            assert st["edb_gemm"] == 1 and st["aten_mm"] == 0, (M, N, K, st)
            aligned = (a_k or M % 8 == 0) and (not a_k or K % 8 == 0) and \
                (b_k or N % 8 == 0) and (not b_k or K % 8 == 0)
            assert (st["padded_operands"] > 0) == (not aligned), (M, N, K, st)
            assert c.shape == (M, N)
            r, bound = gemm_ref.reference(A, B)
            _check("mm", c, r, bound, (M, N, K))
            if N % 8:
                continue  # the fused bias and residual need N % 8 == 0
            bias, res = _rand(N), _rand(M, N)
            gemm.reset_stats()
            c = gemm.addmm(bias, a, b)
            assert gemm.stats()["edb_gemm"] == 1 and gemm.stats()["aten_mm"] == 0
            r, bound = gemm_ref.reference(A, B, bias=bias)
            _check("addmm", c, r, bound, (M, N, K))
            gemm.reset_stats()
            c = gemm.mm_add(a, b, res)
            assert gemm.stats()["edb_gemm_epi"] == 1 and gemm.stats()["aten_mm"] == 0
            r, bound = gemm_ref.reference(A, B, add=res)
            _check("mm_add", c, r, bound, (M, N, K))


# ---- split-K -------------------------------------------------------------------------------------

SPLITK_CASES = [(1024, 1024, 960), (1024, 1024, 1024), (1024, 1024, 1032), (1024, 100, 1032),
                (1024, 102, 1032), (512, 512, 4096), (512, 102, 2048), (1000, 72, 1544)]


@pytest.mark.parametrize("a_k,b_k", LAYOUTS, ids=LAYOUT_IDS)
def test_gemm_split_k_edges(rt, a_k, b_k):
    """Eligibility boundary (15 vs 16 k-blocks), uneven last slice, ldc padding (N = 100) and the
    reduce kernel's scalar tail (N = 102), with and without bias: 2 launches (GEMM + reduce) where
    split, 1 where not; the result meets the bound and repeats bit for bit."""
    from easydist_b200 import gemm
    torch.manual_seed(1)
    sms = _sms()
    assert _splits_expected(1024, 1024, 1024, sms) and not _splits_expected(1024, 1024, 960, sms)
    for (M, N, K) in SPLITK_CASES:
        A, B = _rand(M, K), _rand(K, N)
        a, b = _layout(A, B, a_k, b_k)
        want = 2 if _splits_expected(M, N, K, sms) else 1
        for bias in ([None, _rand(N)] if N % 8 == 0 else [None]):
            gemm.reset_stats()
            n0 = rt.launch_count()
            c = gemm.mm(a, b) if bias is None else gemm.addmm(bias, a, b)
            copies = gemm.stats()["padded_operands"]  # box copies that stage an unaligned operand
            assert rt.launch_count() - n0 == want + copies, (M, N, K, bias is None)
            r, bound = gemm_ref.reference(A, B, bias=bias)
            _check("split_k", c, r, bound, (M, N, K, bias is None))
            c2 = gemm.mm(a, b) if bias is None else gemm.addmm(bias, a, b)
            assert torch.equal(c, c2), (M, N, K)


# ---- epilogues -----------------------------------------------------------------------------------

@pytest.mark.parametrize("bn", [128, 256], ids=["bn128", "bn256"])
@pytest.mark.parametrize("a_k,b_k", LAYOUTS, ids=LAYOUT_IDS)
def test_gemm_epilogues(rt, a_k, b_k, bn):
    """mm_add (with and without bias) and mm_gelu_bwd: M and N tails, a persistent grid, a long K
    (epilogues never split: one launch), aux as a strided view (ld_aux = N + 8)."""
    from easydist_b200 import gemm
    torch.manual_seed(2)
    with option(rt, "gemm_force_bn", bn):
        for (M, N, K) in [(129, 264, 200), persistent_shape(), (256, 512, 4096)]:
            A, B = _rand(M, K), _rand(K, N, scale=0.05)
            a, b = _layout(A, B, a_k, b_k)
            res = _rand(M, N + 8)[:, :N]
            pre = _rand(M, N + 8, scale=2.0)[:, :N]
            bias = _rand(N)
            for kind in ("add", "add_bias", "gelu_bwd"):
                gemm.reset_stats()
                n0 = rt.launch_count()
                if kind == "gelu_bwd":
                    c = gemm.mm_gelu_bwd(a, b, pre)
                    r, bound = gemm_ref.reference(A, B, gelu_pre=pre)
                else:
                    bi = bias if kind == "add_bias" else None
                    c = gemm.mm_add(a, b, res, bi)
                    r, bound = gemm_ref.reference(A, B, bias=bi, add=res)
                st = gemm.stats()
                assert st["edb_gemm_epi"] == 1 and st["aten_mm"] == 0, (kind, M, st)
                assert rt.launch_count() - n0 == 1 + st["padded_operands"], (kind, M)
                _check("epi_" + kind, c, r, bound, (M, N, K))


# ---- guard bands ---------------------------------------------------------------------------------

@pytest.mark.parametrize("case", ["plain", "bias", "split_k_n102", "add"])
def test_gemm_writes_exactly_its_box(rt, case):
    """C as the interior of a larger buffer (ldc = N rounded up to 8, + 16; one guard row above and
    below, filled with a sentinel pattern): every guard element keeps its bits."""
    from easydist_b200._lib import check
    torch.manual_seed(3)
    M, N, K = (1024, 102, 1032) if case == "split_k_n102" else (129, 264, 200)
    A, B = _rand(M, K), _rand(K, N)
    Bt = B.t().contiguous()  # B K-major: ldb = K, a multiple of 8
    ldc = (N + 7) // 8 * 8 + 16
    sentinel = (torch.arange((M + 2) * ldc, device="cuda") % 251 - 125).bfloat16().view(M + 2, ldc)
    buf = sentinel.clone()
    C = buf[1:M + 1]
    bias = _rand(N) if case == "bias" else None
    n0 = rt.launch_count()
    if case == "add":
        aux = _rand(M, N + 8)[:, :N]
        check(rt.lib.edb_gemm_epi_bf16(C.data_ptr(), A.data_ptr(), Bt.data_ptr(), None,
                                       aux.data_ptr(), aux.stride(0), 1, M, N, K, K, K, ldc, 1, 1,
                                       0, 0, None, None, None, None, None, rt.stream()))
        r, bound = gemm_ref.reference(A, B, add=aux)
    else:
        check(rt.lib.edb_gemm_bf16(C.data_ptr(), A.data_ptr(), Bt.data_ptr(),
                                   bias.data_ptr() if bias is not None else None, M, N, K, K, K, ldc,
                                   1, 1, 0, rt.stream()))
        r, bound = gemm_ref.reference(A, B, bias=bias)
    want = 2 if case == "split_k_n102" else 1
    assert rt.launch_count() - n0 == want
    torch.cuda.synchronize()
    guard = torch.ones_like(buf, dtype=torch.bool)
    guard[1:M + 1, :N] = False
    assert torch.equal(buf.view(torch.int16)[guard], sentinel.view(torch.int16)[guard]), case
    _check("guard_" + case, C[:, :N], r, bound, case)


# ---- CUDA graphs ---------------------------------------------------------------------------------

def _graph_cases():
    Mp, Np, Kp = persistent_shape()
    return {
        "persistent": ((Mp, Np, Kp), lambda g, a, b, x: g.mm(a, b)),
        "split_k": ((1024, 1024, 1032), lambda g, a, b, x: g.mm(a, b)),
        "split_k_bias": ((1024, 1024, 1024), lambda g, a, b, x: g.addmm(x[0], a, b)),
        "padded_n_split_k": ((512, 102, 2048), lambda g, a, b, x: g.mm(a, b)),
        "epi_add": ((1024, 1024, 1024), lambda g, a, b, x: g.mm_add(a, b, x[1], x[0])),
        "epi_gelu_bwd": ((1024, 1024, 1024), lambda g, a, b, x: g.mm_gelu_bwd(a, b, x[1])),
    }


@pytest.mark.parametrize("case", ["persistent", "split_k", "split_k_bias", "padded_n_split_k",
                                  "epi_add", "epi_gelu_bwd"])
def test_gemm_cuda_graph_matches_eager(rt, case):
    """Captured as torch.cuda.graph captures by default (its own capture stream) and on a brand-new
    stream: the capture issues the eager call's launches (split-K stays split) and every replay,
    also after new values are written into the static inputs, equals the eager call bit for bit."""
    from easydist_b200 import gemm
    torch.manual_seed(4)
    (M, N, K), fn = _graph_cases()[case]
    a = _rand(K, M).t()  # wgrad layout: A M-major
    b = _rand(N, K).t()  # B K-major: no staging copy, also for N = 102
    extra = (_rand(N), _rand(M, N))

    def refill():
        for t in (a, b) + extra:
            t.copy_(torch.randn(t.shape, device="cuda"))

    n0 = rt.launch_count()
    eager = fn(gemm, a, b, extra)
    launches = rt.launch_count() - n0
    assert launches == (2 if case.startswith(("split_k", "padded_n_split")) else 1)
    for where in ("default_capture_stream", "new_stream"):
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        n0 = rt.launch_count()
        if where == "new_stream":
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side), torch.cuda.graph(g, stream=side):
                out = fn(gemm, a, b, extra)
            torch.cuda.current_stream().wait_stream(side)
        else:
            with torch.cuda.graph(g):
                out = fn(gemm, a, b, extra)
        assert rt.launch_count() - n0 == launches, (where, rt.launch_count() - n0, launches)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager), where
        refill()
        g.replay()
        eager = fn(gemm, a, b, extra)
        torch.cuda.synchronize()
        assert torch.equal(out, eager), (where, "new inputs")
        del g


# ---- LayerNorm -----------------------------------------------------------------------------------

LN_WIDTHS = {torch.bfloat16: [256, 512, 768, 1024, 1536, 2048],
             torch.float32: [128, 256, 384, 512, 768, 1024]}


def _ln_ref(x, w, b, dy, eps=1e-5):
    x, w, dy = x.double(), w.double(), dy.double()
    mu = x.mean(-1, keepdim=True)
    rstd = ((x - mu) ** 2).mean(-1, keepdim=True).add(eps).rsqrt()
    xh = (x - mu) * rstd
    y = xh * w + (b.double() if b is not None else 0.0)
    g = dy * w
    dx = rstd * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
    return y, mu, rstd, dx, (dy * xh).sum(0), dy.sum(0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_layer_norm_every_width_matches_fp64(rt, dtype):
    """edb_layer_norm_fwd / bwd / bwd_add at every supported width (every vector-count template
    instance) vs float64, rows from 1 to more than one pass of the persistent backward grid, with
    bias=None and the output masks that drop dw or db.  Tolerances of
    test_gpu_single.test_layer_norm_kernels_match_aten."""
    from easydist_b200 import norm
    torch.manual_seed(5)
    if dtype == torch.float32:
        tol, red = dict(rtol=1e-5, atol=1e-5), (1e-4, 1e-4)
    else:
        tol, red = dict(rtol=2 ** -7, atol=2e-2), (2 ** -6, 0.05)
    many = 2 * _sms() * 4 + 1  # one row more than a pass of the backward grid (2 CTAs/SM x 4 warps)
    for H in LN_WIDTHS[dtype]:
        for rows in (1, 3, many, 8192):
            x = torch.randn(rows, H, device="cuda").to(dtype)
            w = (torch.randn(H, device="cuda") * 0.5 + 1).to(dtype)
            b = torch.randn(H, device="cuda").to(dtype)
            dy = torch.randn(rows, H, device="cuda").to(dtype)
            add = torch.randn(rows, H, device="cuda").to(dtype)
            red_tol = dict(rtol=red[0], atol=red[1] * rows ** 0.5)
            for bias in (b, None) if rows == many else (b,):
                norm.reset_stats()
                y, mean, rstd = norm.native_layer_norm(x, [H], w, bias, 1e-5)
                ry, rmu, rrs, rdx, rdw, rdb = _ln_ref(x, w, bias, dy)
                assert torch.allclose(mean.double(), rmu, rtol=1e-5, atol=1e-6), (H, rows)
                assert torch.allclose(rstd.double(), rrs, rtol=1e-5, atol=1e-6), (H, rows)
                assert torch.allclose(y.double(), ry, **tol), (H, rows, bias is None)
                masks = [[True, True, True]]
                if rows == many:
                    masks += [[True, False, False], [True, True, False], [True, False, True]]
                for mask in masks:
                    dx, dw, db = norm.native_layer_norm_backward(dy, x, [H], mean, rstd, w, bias, mask)
                    assert torch.allclose(dx.double(), rdx, **tol), (H, rows, mask)
                    assert (dw is None) == (not mask[1]) and (db is None) == (not mask[2])
                    if mask[1]:
                        assert torch.allclose(dw.double(), rdw, **red_tol), (H, rows, mask)
                    if mask[2]:
                        assert torch.allclose(db.double(), rdb, **red_tol), (H, rows, mask)
                assert norm.stats()["aten_ln"] == 0 and norm.stats()["edb_ln_fwd"] == 1, norm.stats()
            # fused accumulation: the same two roundings as the kernel followed by aten.add
            dx0, dw0, db0 = norm.native_layer_norm_backward(dy, x, [H], mean, rstd, w, b,
                                                            [True, True, True])
            dx1, dw1, db1 = norm.native_layer_norm_backward(dy, x, [H], mean, rstd, w, b,
                                                            [True, True, True], _add=add)
            assert torch.equal(dx1, dx0 + add) and torch.equal(dw1, dw0) and torch.equal(db1, db0)
            assert torch.allclose(dx1.double(), rdx + add.double(), rtol=tol["rtol"],
                                  atol=tol["atol"] + 2.0 ** -8 * float(rdx.abs().max())), (H, rows)
