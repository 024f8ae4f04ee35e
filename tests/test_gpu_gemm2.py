"""k_gemm2_bf16 (the plain single-GPU GEMM: register-budgeted warpgroups, per-warpgroup epilogue)
against k_gemm_bf16 on the same operands.

Both kernels accumulate every output element in the same order and round at the same points, so the
comparison is torch.equal, over the whole destination buffer including the guard bands around C.
The `gemm2` option selects the kernel: 0 = k_gemm_bf16, 1 = k_gemm2_bf16.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

LAYOUTS = [(True, True), (True, False), (False, True), (False, False)]  # (A K-major, B K-major)
LAYOUT_IDS = ["a_k-b_k", "a_k-b_n", "a_m-b_k", "a_m-b_n"]
KINDS = ["none", "bias", "add", "gelu_bwd"]
EPI_ADD, EPI_GELU_BWD = 1, 2


@pytest.fixture(scope="module")
def rt():
    from easydist_b200 import runtime
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    r = runtime.init(rank=0, world=1, device=0, heap_bytes=2 << 30) \
        if not runtime.is_initialized() else runtime.get_runtime()
    old = r.get_option("gemm2")
    yield r
    r.set_option("gemm2", old)


def _shapes():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {
        "qkv": (4096, 3072, 1024),
        "fc_dgrad": (4096, 1024, 4096),
        "lm_head": (4096, 50257, 1024),       # N % 8 != 0: C and an MN-major B carry a padded ld
        "tails": (384, 264, 200),
        "odd_m_tiles": (128 * 5 + 1, 512, 200),
        "one_tile": (100, 200, 136),
        "waves": (128 * math.ceil(3 * sms / 10) + 72, 2560, 392),  # > 3 tiles per CTA, 7 k-blocks
    }


def _r8(x):
    return (x + 7) // 8 * 8


def _operand(rows, cols, major_is_cols, scale=1.0):
    """[rows, cols] values stored with unit stride along cols (major_is_cols) or along rows; the
    other stride is rounded up to 8 elements.  Returns (storage, ld)."""
    if major_is_cols:
        t = torch.zeros(rows, _r8(cols), device="cuda", dtype=torch.bfloat16)
        t[:, :cols] = (torch.randn(rows, cols, device="cuda") * scale).bfloat16()
    else:
        t = torch.zeros(cols, _r8(rows), device="cuda", dtype=torch.bfloat16)
        t[:, :rows] = (torch.randn(cols, rows, device="cuda") * scale).bfloat16()
    return t, t.stride(0)


class Case:
    def __init__(self, M, N, K, a_k, b_k, kind):
        self.M, self.N, self.K, self.a_k, self.b_k, self.kind = M, N, K, a_k, b_k, kind
        self.A, self.lda = _operand(M, K, a_k)
        self.B, self.ldb = _operand(N, K, b_k, scale=0.05)
        self.ldc = _r8(N) + 16
        self.sentinel = (torch.arange((M + 2) * self.ldc, device="cuda") % 251 - 125) \
            .bfloat16().view(M + 2, self.ldc)
        self.buf = self.sentinel.clone()
        self.bias = torch.randn(N, device="cuda").bfloat16() if kind in ("bias", "add") else None
        self.aux = None
        if kind in ("add", "gelu_bwd"):
            self.aux = (torch.randn(M, N + 8, device="cuda") * 2.0).bfloat16()[:, :N]

    def launch(self, rt):
        from easydist_b200._lib import check
        C = self.buf[1:self.M + 1]
        bias = self.bias.data_ptr() if self.bias is not None else None
        M, N, K = self.M, self.N, self.K
        if self.aux is not None:
            op = EPI_ADD if self.kind == "add" else EPI_GELU_BWD
            check(rt.lib.edb_gemm_epi_bf16(C.data_ptr(), self.A.data_ptr(), self.B.data_ptr(), bias,
                                           self.aux.data_ptr(), self.aux.stride(0), op, M, N, K,
                                           self.lda, self.ldb, self.ldc, int(self.a_k), int(self.b_k),
                                           0, 0, None, None, None, None, None, rt.stream()))
        else:
            check(rt.lib.edb_gemm_bf16(C.data_ptr(), self.A.data_ptr(), self.B.data_ptr(), bias, M, N,
                                       K, self.lda, self.ldb, self.ldc, int(self.a_k), int(self.b_k),
                                       0, rt.stream()))

    def run(self, rt, stage):
        """The destination buffer (guard bands included) after one launch at `stage`."""
        rt.set_option("gemm2", stage)
        self.buf.copy_(self.sentinel)
        n0 = rt.launch_count()
        self.launch(rt)
        assert rt.launch_count() - n0 == 1
        torch.cuda.synchronize()
        return self.buf.clone()

    def run_graph(self, rt, stage):
        rt.set_option("gemm2", stage)
        self.buf.copy_(self.sentinel)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.launch(rt)
        self.buf.copy_(self.sentinel)  # whatever the capture did, the replay alone must produce C
        g.replay()
        torch.cuda.synchronize()
        return self.buf.clone()


@pytest.mark.parametrize("shape", ["qkv", "fc_dgrad", "lm_head", "tails", "odd_m_tiles", "one_tile",
                                   "waves"])
@pytest.mark.parametrize("a_k,b_k", LAYOUTS, ids=LAYOUT_IDS)
def test_gemm2_bits_equal_gemm(rt, a_k, b_k, shape):
    """Every layout and epilogue: k_gemm2_bf16 writes the bits k_gemm_bf16 writes and leaves the
    guard bands alone, eagerly and replayed from a CUDA graph."""
    M, N, K = _shapes()[shape]
    torch.manual_seed(11)
    for kind in (KINDS if N % 8 == 0 else ["none"]):
        c = Case(M, N, K, a_k, b_k, kind)
        want = c.run(rt, 0)
        # an N that is not a multiple of 8 owns its row up to the next multiple (gemm.mm allocates
        # C that way): a TMA store clips at 16 bytes there and zeroes the columns in between
        guard = torch.ones_like(want, dtype=torch.bool)
        guard[1:M + 1, :_r8(N)] = False
        touched = (want.view(torch.int16) != c.sentinel.view(torch.int16)) & guard
        assert not touched.any(), (shape, kind, int(touched.sum()), touched.nonzero()[:8].tolist())
        assert not torch.equal(want[1:M + 1, :N], c.sentinel[1:M + 1, :N])
        got = c.run(rt, 1)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (shape, kind)
        got = c.run_graph(rt, 1)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (shape, kind, "graph")


def _kernels_of(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.key for e in prof.key_averages() if "gemm" in e.key]


def test_gemm2_takes_only_plain_256_wide_launches(rt):
    """By kernel name: a plain 256-wide launch runs k_gemm2_bf16 unless the option says 0; a forced
    tile width, a split-K shape and a K of more than 256 k-blocks keep k_gemm_bf16."""
    torch.manual_seed(12)
    plain = Case(1024, 1024, 512, True, True, "none")
    split = Case(1024, 1024, 1024, True, True, "none")  # 32 tiles, 16 k-blocks: split-K
    long_k = Case(4096, 1024, 64 * 257, True, True, "none")
    rt.set_option("gemm2", 1)
    names = _kernels_of(lambda: plain.launch(rt))
    assert len(names) == 1 and "k_gemm2_bf16" in names[0], names
    names = _kernels_of(lambda: long_k.launch(rt))
    assert len(names) == 1 and "k_gemm_bf16" in names[0], names
    names = _kernels_of(lambda: split.launch(rt))
    assert any("k_gemm_bf16" in n for n in names) and not any("k_gemm2_bf16" in n for n in names), names
    for bn in (128, 256):
        rt.set_option("gemm_force_bn", bn)
        try:
            names = _kernels_of(lambda: plain.launch(rt))
        finally:
            rt.set_option("gemm_force_bn", 0)
        assert len(names) == 1 and "k_gemm_bf16" in names[0], (bn, names)
    rt.set_option("gemm2", 0)
    names = _kernels_of(lambda: plain.launch(rt))
    assert len(names) == 1 and "k_gemm_bf16" in names[0], names
    rt.set_option("gemm2", 1)
