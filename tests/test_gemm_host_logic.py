"""Host side of easydist_b200.gemm with the C-ABI mocked out: operand-layout classification
(K-major / MN-major for both operands), leading dimensions, padded staging for strides that break
TMA's 16-byte rule (vocab 50257), padded outputs — no GPU, no compute."""
import pytest
import torch

from easydist_b200 import _lib, gemm


class _FakeLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return 0
        return fn


@pytest.fixture
def lib(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(_lib, "load", lambda *a, **k: fake)
    monkeypatch.setattr(gemm, "_stream", lambda t: None)
    gemm.reset_stats()
    return fake


def _gemm_args(call):
    name, a = call
    assert name == "edb_gemm_bf16"
    keys = ["C", "A", "B", "bias", "M", "N", "K", "lda", "ldb", "ldc", "a_k", "b_k", "acc", "stream"]
    return dict(zip(keys, a))


@pytest.mark.parametrize("a_k,b_k", [(True, True), (True, False), (False, True), (False, False)])
def test_operand_layouts_map_to_kmajor_flags_without_copies(lib, a_k, b_k):
    M, N, K = 64, 48, 32
    A = torch.zeros(M, K, dtype=torch.bfloat16)
    B = torch.zeros(K, N, dtype=torch.bfloat16)
    a = A if a_k else A.t().contiguous().t()          # [M,K] with stride (1, M)
    b = B.t().contiguous().t() if b_k else B          # [K,N] with stride (1, K) = stored [N,K]
    out = gemm._launch(a, b, None)
    (call,) = lib.calls                               # no staging copy
    g = _gemm_args(call)
    assert (g["M"], g["N"], g["K"]) == (M, N, K)
    assert (g["a_k"], g["b_k"]) == (int(a_k), int(b_k))
    assert g["lda"] == (K if a_k else M) and g["ldb"] == (K if b_k else N) and g["ldc"] == N
    assert g["A"] == a.data_ptr() and g["B"] == b.data_ptr() and g["bias"] is None
    assert out.shape == (M, N) and out.is_contiguous()
    assert gemm.recorded_calls()[-1][:5] == (M, N, K, a_k, b_k)


def test_unaligned_leading_dims_are_staged_and_unaligned_n_gets_a_padded_output(lib):
    V, H, T = 50257, 64, 16
    x = torch.zeros(T, H, dtype=torch.bfloat16)
    W = torch.zeros(V, H, dtype=torch.bfloat16)
    logits = gemm._launch(x, W.t(), None)             # N = 50257: padded output, operands legal
    g = _gemm_args(lib.calls[-1])
    assert g["ldc"] == 50264 and logits.shape == (T, V) and logits.stride() == (50264, 1)
    assert [c[0] for c in lib.calls] == ["edb_gemm_bf16"]
    lib.calls.clear()
    dl = torch.zeros(T, V, dtype=torch.bfloat16)      # row stride 50257: not a multiple of 8
    gemm._launch(dl, W, None)                         # dgrad: A staged into a padded buffer
    names = [c[0] for c in lib.calls]
    assert names == ["edb_box_copy_local", "edb_gemm_bf16"]
    g = _gemm_args(lib.calls[-1])
    assert g["lda"] == 50264 and g["a_k"] == 1 and g["K"] == V
    assert gemm.stats()["padded_operands"] == 1
    lib.calls.clear()
    # the cross-entropy kernel hands over a gradient that already has a legal stride: no staging
    dl_padded = torch.zeros(T, 50264, dtype=torch.bfloat16)[:, :V]
    gemm._launch(dl_padded, W, None)
    gemm._launch(dl_padded.t(), x, None)              # wgrad: A = dl^T, MN-major view of the same buffer
    assert [c[0] for c in lib.calls] == ["edb_gemm_bf16", "edb_gemm_bf16"]
    g = _gemm_args(lib.calls[-1])
    assert (g["M"], g["K"], g["a_k"], g["lda"]) == (V, T, 0, 50264)


def test_shapes_the_kernel_does_not_take(lib):
    a = torch.zeros(8, 1, dtype=torch.bfloat16)
    assert gemm._launch(a, torch.zeros(1, 8, dtype=torch.bfloat16), None) is None   # degenerate strides
    s = torch.zeros(8, 16, dtype=torch.bfloat16)[:, ::2]                            # no unit stride
    assert gemm._launch(s, torch.zeros(8, 8, dtype=torch.bfloat16), None) is None
    # bias needs N % 8 == 0
    assert gemm._launch(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 12, dtype=torch.bfloat16),
                        torch.zeros(12, dtype=torch.bfloat16)) is None
    # CPU tensors never reach the kernel through the public entry point: ATen, counted
    out = gemm.mm(torch.ones(4, 4, dtype=torch.bfloat16), torch.ones(4, 4, dtype=torch.bfloat16))
    assert gemm.stats()["aten_mm"] == 1 and float(out[0, 0]) == 4.0


def _overlapping_layouts(M, K):
    """[M, K] operands whose rows overlap: expanded (strides (0, 1)), its MN-major mirror (1, 0),
    and rows 64 elements apart with K = 512."""
    bf = torch.bfloat16
    return {"expanded_rows": torch.zeros(K, dtype=bf).expand(M, K),
            "expanded_cols": torch.zeros(M, 1, dtype=bf).expand(M, K),
            "overlapping": torch.zeros(M * 64 + K, dtype=bf).as_strided((M, K), (64, 1))}


@pytest.mark.parametrize("layout", ["expanded_rows", "expanded_cols", "overlapping"])
def test_overlapping_rows_never_reach_the_lib(lib, layout):
    """A TMA descriptor describes a matrix whose rows do not overlap: `_prepare` must not hand over
    ld < row length, which the backward of sum(dim=0) (an expanded gradient) would otherwise give."""
    M, K, N = 64, 512, 64
    a = _overlapping_layouts(M, K)[layout]
    for unit_dim in (0, 1):
        p = gemm._prepare(a, unit_dim)
        assert p is None or p[2] >= p[0].shape[1], (unit_dim, p and p[2])
    b = torch.zeros(K, N, dtype=torch.bfloat16)
    gemm._launch(a, b, None)                                            # as A
    gemm._launch(torch.zeros(N, M, dtype=torch.bfloat16), a, None)     # as B
    for name, args in lib.calls:
        if name == "edb_gemm_bf16":
            g = _gemm_args((name, args))
            assert g["lda"] >= (g["K"] if g["a_k"] else g["M"]), g
            assert g["ldb"] >= (g["K"] if g["b_k"] else g["N"]), g


@pytest.mark.parametrize("op", ["mm_add", "mm_gelu_bwd"])
def test_epilogue_operand_with_overlapping_rows_takes_the_unfused_path(lib, monkeypatch, op):
    """An expanded residual / pre-activation (stride(0) == 0 < N) is not a layout the epilogue reads:
    the GEMM runs plain and ATen applies the elementwise op."""
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    M, K, N = 64, 32, 48
    a = torch.zeros(M, K, dtype=torch.bfloat16)
    b = torch.zeros(K, N, dtype=torch.bfloat16)
    aux = torch.ones(N, dtype=torch.bfloat16).expand(M, N)
    out = getattr(gemm, op)(a, b, aux)
    assert out.shape == (M, N)
    assert [c[0] for c in lib.calls] == ["edb_gemm_bf16"], lib.calls
    # a dense operand still goes through the epilogue
    lib.calls.clear()
    getattr(gemm, op)(a, b, aux.contiguous())
    assert [c[0] for c in lib.calls] == ["edb_gemm_epi_bf16"]


def test_views_of_a_narrowed_gemm_output_are_reshapes():
    """gemm.mm returns an output with N % 8 != 0 as a narrowed view of a padded buffer; a `view` the
    graph took of the contiguous traced output (here: flattening a bias-free Linear(16, 3) head) must
    still work on it, and views of outputs with N % 8 == 0 stay views."""
    from torch.fx.experimental.proxy_tensor import make_fx
    from easydist_b200 import lowering
    aten = torch.ops.aten

    def padded_mm(a, b):          # what gemm.mm returns on the GPU for N % 8 != 0
        n = b.shape[1]
        out = torch.full((a.shape[0], (n + 7) // 8 * 8), float("nan"), dtype=a.dtype)
        out[:, :n] = a @ b
        return out[:, :n]

    for n_out in (3, 8):
        f = lambda x, w: torch.nn.functional.linear(x, w).reshape(-1)
        x = torch.randn(2, 4, 16, dtype=torch.bfloat16)
        w = torch.randn(n_out, 16, dtype=torch.bfloat16)
        gm = make_fx(f, tracing_mode="fake")(x, w)
        lowering.dispatch_compute(gm)
        targets = [nd.target for nd in gm.graph.nodes if nd.op == "call_function"]
        assert gemm.mm in targets
        views = [t for t in targets if t in (aten.view.default, aten._unsafe_view.default)]
        if n_out % 8:
            assert aten.reshape.default in targets and len(views) == 1, targets   # the input's view stays
        else:
            assert aten.reshape.default not in targets, targets
        for nd in gm.graph.nodes:
            if nd.target is gemm.mm:
                nd.target = padded_mm
        gm.recompile()
        assert torch.equal(gm(x, w), f(x, w))
