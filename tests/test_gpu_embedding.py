"""The embedding kernels (edb_embed.cu) on one H100: the forward bit for bit against aten.embedding
(+ aten.add for GPT-2's two tables) over dtypes, table sizes, widths, row counts and id dtypes; the
backward against the float64 bound of tests/embed_ref.py, its bits across runs and under CUDA-graph
capture; the in-place mode touching only the indexed rows; out-of-range ids; the counted ATen path;
and small GPT-2 and Llama models trained through the compiled path against vanilla fp32 PyTorch."""
import pytest
import torch

from tests import embed_ref as E

pytestmark = pytest.mark.gpu
aten = torch.ops.aten
GUARD = 4096  # elements of guard band on each side of an output


@pytest.fixture(scope="module")
def rt():
    from easydist_b200 import runtime
    from easydist_b200.device_mesh import set_device_mesh
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    r = runtime.init(rank=0, world=1, device=0, heap_bytes=2 << 30) \
        if not runtime.is_initialized() else runtime.get_runtime()
    set_device_mesh([0], ["dp"], rank=0)
    return r


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _ids(n, V, dtype, seed):
    return torch.randint(0, V, (n,), device="cuda", generator=_gen(seed)).to(dtype)


def _guarded(shape, dtype, fill):
    """A tensor of `shape` inside a buffer whose GUARD elements on either side hold `fill`."""
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + 2 * GUARD,), fill, dtype=dtype, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(shape)


def _guard_intact(buf, fill):
    return bool((buf[:GUARD] == fill).all()) and bool((buf[-GUARD:] == fill).all())


def _same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(
        a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


# ---- forward ---------------------------------------------------------------------------------------

FWD = [(V, C) for V in (1, 7, 50304) for C in (8, 64, 768, 1024, 4096)] + [(512, 12), (1000, 129)]


@pytest.mark.parametrize("V,C", FWD)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_forward_is_bit_identical_to_aten(rt, V, C, dtype):
    from easydist_b200 import embed
    W = torch.randn(V, C, device="cuda", generator=_gen(V + C)).to(dtype)
    embed.reset_stats()
    for n, idt in ((1, torch.int64), (333, torch.int32), (16384 if C <= 1024 else 2048, torch.int64)):
        idx = _ids(n, V, idt, n)
        assert _same_bits(embed.embedding_fwd(W, idx), aten.embedding(W, idx.long())), (n, idt)
    st = embed.stats()
    assert st["edb_embed_fwd"] == 3 and st["aten_embed"] == 0, st


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("idt", [torch.int32, torch.int64])
@pytest.mark.parametrize("B,T,C", [(8, 512, 1024), (1, 1, 8), (3, 7, 12)])
def test_two_table_forward_is_bit_identical_to_aten(rt, dtype, idt, B, T, C):
    from easydist_b200 import embed
    V, Vp = 50257, 1024
    W = torch.randn(V, C, device="cuda", generator=_gen(1)).to(dtype)
    P = torch.randn(Vp, C, device="cuda", generator=_gen(2)).to(dtype)
    idx = _ids(B * T, V, idt, 3).view(B, T)
    pos = torch.arange(T, device="cuda", dtype=idt)
    want = aten.add(aten.embedding(W, idx.long()), aten.embedding(P, pos.long()))
    buf, y = _guarded((B, T, C), dtype, 7.0)
    embed.reset_stats()
    got = embed.embedding_fwd(W, idx, P, pos)
    y.copy_(got)
    assert _same_bits(got, want) and _guard_intact(buf, 7.0)
    assert embed.stats()["edb_embed_fwd"] == 1


# ---- backward --------------------------------------------------------------------------------------

BWD = [  # (name, V, C, rows, ids)
    ("random", 50304, 1024, 4096, None),
    ("random_wide", 32000, 4096, 2048, None),
    ("one_id", 1000, 64, 16384, "one"),
    ("distinct", 50304, 128, 16384, "distinct"),
    ("scalar_path", 777, 129, 3000, None),
    ("tiny", 1, 8, 5, None),
]


def _bwd_inputs(V, C, rows, kind, dtype, idt, seed):
    g = _gen(seed)
    dy = torch.randn(rows, C, device="cuda", generator=g).to(dtype)
    if kind == "one":
        idx = torch.full((rows,), V // 2, device="cuda", dtype=idt)
    elif kind == "distinct":
        idx = torch.randperm(V, device="cuda", generator=g)[:rows].to(idt)
    else:
        idx = torch.randint(0, V, (rows,), device="cuda", generator=g).to(idt)
    return dy, idx


def _check_dense(got, dy, idx, V, pad, dtype):
    S, A, k = E.bwd_ref(dy, idx, V)
    if 0 <= pad < V:
        assert bool((got[pad] == 0).all())
        S[pad], A[pad], k[pad] = 0.0, 0.0, 0.0
    r = E.worst(got, S, E.bwd_bound(S, A, k, dtype))
    assert r <= 1.0, r


@pytest.mark.parametrize("name,V,C,rows,kind", BWD, ids=[b[0] for b in BWD])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_backward_within_the_bound_and_repeatable(rt, name, V, C, rows, kind, dtype):
    from easydist_b200 import embed
    for idt, pad in ((torch.int64, -1), (torch.int32, V // 2)):
        dy, idx = _bwd_inputs(V, C, rows, kind, dtype, idt, seed=rows + C)
        buf, out = _guarded((V, C), dtype, 3.0)
        embed.reset_stats()
        g1 = embed.embedding_bwd(dy, idx, V, pad)
        out.copy_(g1)
        _check_dense(g1, dy, idx, V, pad, dtype)
        assert _same_bits(g1, embed.embedding_bwd(dy, idx, V, pad))
        assert _guard_intact(buf, 3.0)
        assert embed.stats()["edb_embed_bwd"] == 2 and embed.stats()["aten_embed"] == 0


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("kind", [None, "one"])
def test_accumulate_touches_only_the_indexed_rows(rt, dtype, kind):
    from easydist_b200 import embed
    V, C, rows, pad = 5000, 1024, 4096, 17
    dy, idx = _bwd_inputs(V, C, rows, kind, dtype, torch.int64, seed=5)
    idx[::97] = pad
    hit = torch.zeros(V, dtype=torch.bool, device="cuda")
    hit[idx] = True
    hit[pad] = False
    sentinel = float("nan")
    buf, acc = _guarded((V, C), dtype, -9.0)
    acc.copy_(torch.randn(V, C, device="cuda", generator=_gen(6)).to(dtype) * 4)
    acc[~hit] = sentinel
    before = acc.clone()
    embed.reset_stats()
    out = embed.embedding_bwd_acc_(acc, dy, idx, pad)
    assert out.data_ptr() == acc.data_ptr() and embed.stats()["edb_embed_bwd_acc"] == 1
    assert _guard_intact(buf, -9.0)
    assert bool(torch.isnan(acc[~hit]).all())  # every other row: untouched
    S, A, k = E.bwd_ref(dy, idx, V)
    r = E.worst(acc, before.double() + S, E.acc_bound(before, S, A, k, dtype), rows=hit)
    assert r <= 1.0, r
    # the bits repeat
    again = before.clone()
    embed.embedding_bwd_acc_(again, dy, idx, pad)
    assert _same_bits(acc, again)


def test_accumulate_on_a_padded_row_stride(rt):
    """The LM-head GEMM returns a [V, C] view of a buffer with padded rows when C % 8 != 0."""
    from easydist_b200 import embed
    V, C, rows = 300, 12, 1000
    dy, idx = _bwd_inputs(V, C, rows, None, torch.bfloat16, torch.int64, seed=9)
    base = torch.randn(V, 16, device="cuda").bfloat16()
    acc = base[:, :C]
    want = (acc.float() + embed.embedding_bwd(dy, idx, V).float()).bfloat16()
    embed.embedding_bwd_acc_(acc, dy, idx)
    assert torch.equal(acc, want)


def test_out_of_range_ids_are_skipped(rt):
    """Fed to the kernels only: ATen's device-side assert would fault on them."""
    from easydist_b200 import embed
    V, C = 100, 64
    for dtype in (torch.bfloat16, torch.float32):
        W = torch.randn(V, C, device="cuda").to(dtype)
        idx = torch.tensor([0, -1, V, 5, 1 << 40, -(1 << 40), V - 1], device="cuda")
        ok = (idx >= 0) & (idx < V)
        y = embed.embedding_fwd(W, idx)
        assert torch.equal(y[ok], W[idx[ok]]) and bool((y[~ok] == 0).all())
        dy = torch.randn(idx.numel(), C, device="cuda").to(dtype)
        g = embed.embedding_bwd(dy, idx, V)
        want = torch.zeros(V, C, device="cuda", dtype=dtype)
        want[idx[ok]] = dy[ok]
        assert torch.equal(g, want)
        acc = torch.ones(V, C, device="cuda", dtype=dtype)
        embed.embedding_bwd_acc_(acc, dy, idx)
        assert torch.equal(acc, (torch.ones_like(acc).float() + want.float()).to(dtype))


def test_cuda_graph_capture_gives_the_eager_bits(rt):
    from easydist_b200 import embed
    V, C, rows = 50304, 1024, 4096
    W = torch.randn(V, C, device="cuda").bfloat16()
    P = torch.randn(1024, C, device="cuda").bfloat16()
    dy, idx = _bwd_inputs(V, C, rows, None, torch.bfloat16, torch.int64, seed=12)
    pos = torch.arange(512, device="cuda")
    acc0 = torch.randn(V, C, device="cuda").bfloat16()
    acc = acc0.clone()

    def step():
        acc.copy_(acc0)
        return [embed.embedding_fwd(W, idx.view(8, 512), P, pos), embed.embedding_bwd(dy, idx, V, 3),
                embed.embedding_bwd_acc_(acc, dy, idx, 3).clone()]

    eager = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize()
    assert all(_same_bits(a, b) for a, b in zip(eager, captured))


def test_what_the_kernels_do_not_take_runs_the_counted_aten_path(rt):
    from easydist_b200 import embed
    V, C = 64, 32
    W = torch.randn(C, V, device="cuda").bfloat16().t()  # a strided table
    idx = _ids(10, V, torch.int64, 1)
    dy = torch.randn(10, C, device="cuda").half()  # another dtype
    acc = torch.randn(C, V, device="cuda").bfloat16().t()  # rows not contiguous
    dyb = torch.randn(10, C, device="cuda").bfloat16()
    embed.reset_stats()
    assert torch.equal(embed.embedding_fwd(W, idx), aten.embedding(W, idx))
    assert torch.equal(embed.embedding_bwd(dy, idx, V), aten.embedding_dense_backward(dy, idx, V, -1, False))
    want = acc + aten.embedding_dense_backward(dyb, idx, V, -1, False)
    embed.embedding_bwd_acc_(acc, dyb, idx)
    assert torch.equal(acc, want)
    st = embed.stats()
    assert st["aten_embed"] == 3 and st["edb_embed_fwd"] == st["edb_embed_bwd"] == 0, st
    # an unaligned but contiguous table runs the kernel's scalar path
    buf = torch.randn(V * C + 1, device="cuda").bfloat16()
    Wu = buf[1:].view(V, C)
    assert torch.equal(embed.embedding_fwd(Wu, idx), aten.embedding(Wu, idx))
    assert embed.stats()["edb_embed_fwd"] == 1


# ---- compiled steps --------------------------------------------------------------------------------

def _train(rt, model_fn, cfg, dtype, cuda_graph, want_nodes):
    from easydist_b200 import embed
    from easydist_b200.api import easydist_compile
    from easydist_b200.workloads import gpt2_train_step, synthetic_tokens
    from tools import parity as P
    torch.manual_seed(0)
    model = model_fn().to(device="cuda", dtype=dtype)
    state = {k: v.detach().clone() for k, v in model.state_dict().items()}
    mk_opt = lambda ps: torch.optim.SGD(ps, lr=1e-3, momentum=0.9, foreach=True)
    opt = mk_opt(model.parameters())
    step = easydist_compile(gpt2_train_step, parallel_mode="ddp", tracing_mode="fake",
                            cuda_graph=cuda_graph)
    calls = 4
    embed.reset_stats()
    batches = [synthetic_tokens(cfg, 4, 64, seed=1000 * b) for b in range(calls)]
    losses = [float(step(tok.cuda(), tgt.cuda(), model, opt)) for tok, tgt in batches]
    info = step.compiled_func.info
    assert info["embed_nodes"] == want_nodes, info
    sched = ([0, 0] if cuda_graph else [0]) + list(range(1, calls))
    steps = [[batches[b]] for b in sched]
    ref_l, ref_p, ref_s = P.vanilla_run(model_fn, state, steps, mk_opt, torch.float32, "cuda")
    idx = [1 if cuda_graph else 0] + list(range(2 if cuda_graph else 1, len(sched)))
    rtol = 1e-4 if dtype == torch.float32 else 3e-2
    for got, i in zip(losses, idx):
        assert abs(got - ref_l[i][0]) <= rtol * abs(ref_l[i][0]), (losses, ref_l)
    got_p, got_s = P.compiled_state(step.compiled_func, ref_p, ref_s, 1)
    if dtype == torch.float32:
        res = P.compare(got_p, got_s, ref_p, ref_s, low_precision=False)
        assert res["assert_close_violation"] <= 1.0, res
    else:
        _, van_p, van_s = P.vanilla_run(model_fn, state, steps, mk_opt, torch.bfloat16, "cuda")
        van = P.compare({k: v.bfloat16() for k, v in van_p.items()},
                        {k: {kk: vv.bfloat16() for kk, vv in st.items()} for k, st in van_s.items()},
                        ref_p, ref_s, low_precision=True)
        res = P.compare(got_p, got_s, ref_p, ref_s, low_precision=True)
        assert res["state_rel_l2"] <= max(2e-2, 2.0 * van["state_rel_l2"]), (res, van)
        assert res["param_max_ulp"] <= max(2.0, 2.0 * van["param_max_ulp"]), (res, van)
    return embed.stats()


CASES = [(torch.float32, False), (torch.float32, True), (torch.bfloat16, False), (torch.bfloat16, True)]


@pytest.mark.parametrize("dtype,cuda_graph", CASES)
def test_small_gpt2_trains_like_vanilla_with_native_embeddings(rt, dtype, cuda_graph):
    from easydist_b200.workloads import GPT2, GPT2Config
    cfg = GPT2Config(2, 4, 256, vocab_size=1000, block_size=64)
    st = _train(rt, lambda: GPT2(cfg), cfg, dtype, cuda_graph, (1, 2))
    assert st["aten_embed"] == 0 and st["edb_embed_fwd"] > 0, st
    # bf16: the tied gradient is added in place into the LM-head GEMM's output; fp32 GEMMs are not
    # the native kernel, so the dense variant and the add run
    assert (st["edb_embed_bwd_acc"] > 0) == (dtype == torch.bfloat16), st


@pytest.mark.parametrize("dtype,cuda_graph", CASES)
def test_small_llama_trains_like_vanilla_with_native_embeddings(rt, dtype, cuda_graph):
    from easydist_b200.workloads import Llama, LlamaConfig
    cfg = LlamaConfig(n_layer=2, n_head=4, n_embd=256, ffn=688, vocab_size=512, block_size=64)
    st = _train(rt, lambda: Llama(cfg), cfg, dtype, cuda_graph, (1, 1))
    assert st["aten_embed"] == 0 and st["edb_embed_fwd"] > 0 and st["edb_embed_bwd"] > 0, st
