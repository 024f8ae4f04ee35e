"""The attention kernels (edb_attn.cu) on one H100: forward and backward against the float64 bounds
of tests/attn_ref.py over head dims, lengths, batch and head counts, causal and not, and the layouts
a traced graph hands them, each no less accurate than ATen's flash attention on the same inputs;
their bits across runs; guard bands and row gaps around every output; CUDA-graph capture; the
counted ATen path (other dtypes and head dims, misaligned and broadcast inputs, non-positive
scales); small GPT-2 and Llama models trained through the compiled path under deterministic
algorithms against vanilla fp32 PyTorch; and the bits of such a step across two compilations."""
import ctypes

import pytest
import torch

from tests import attn_ref as R

pytestmark = pytest.mark.gpu
aten = torch.ops.aten
GUARD = 4096


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


def _aten(q, k, v, dout, causal):
    r = aten._scaled_dot_product_flash_attention.default(q, k, v, 0.0, causal)
    g = aten._scaled_dot_product_flash_attention_backward.default(
        dout, q, k, v, r[0], r[1], r[2], r[3], r[4], r[5], 0.0, causal, r[6], r[7])
    return r[0], r[1], *g


def _native(q, k, v, dout, causal):
    from easydist_b200 import attn
    attn.reset_stats()
    out, lse = attn.attention_fwd(q, k, v, causal)
    dq, dk, dv = attn.attention_bwd(dout, q, k, v, out, lse, causal)
    assert attn.stats() == {"edb_attn_fwd": 1, "edb_attn_bwd": 1, "aten_attn_fwd": 0,
                            "aten_attn_bwd": 0}
    return out, lse, dq, dk, dv


SHAPES = [(hd, T) for hd in (64, 128) for T in (1, 17, 64, 127, 128, 129, 512, 2048)]
LAYOUTS = ["split", "contiguous", "transposed", "offset"]


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("hd,T", SHAPES)
def test_within_the_float64_bound_and_no_worse_than_aten(rt, hd, T, causal, layout):
    B, H = (1, 2) if T >= 2048 else ((3, 5) if T <= 129 else (2, 3))
    q, k, v, dout = R.inputs(B, H, T, hd, seed=T * 7 + hd + causal, layout=layout, device="cuda")
    r = R.reference(q, k, v, dout, causal)
    got = _native(q, k, v, dout, causal)
    ref = _aten(q, k, v, dout, causal)
    assert torch.allclose(got[1].double(), r["lse"], rtol=0, atol=1e-4)
    bounds = (R.fwd_bound(r), *R.bwd_bound(r))
    for name, g, a, want, bound in zip(("out", "dq", "dk", "dv"), got[:1] + got[2:], ref[:1] + ref[2:],
                                       (r["out"], r["dq"], r["dk"], r["dv"]), bounds):
        err = (g.double() - want).abs()
        assert float((err / bound).max()) <= 1.0, (name, float((err / bound).max()))
        # the same rounding points as FlashAttention-2: the mean error may differ by noise only
        aerr = (a.double() - want).abs()
        assert float(err.mean()) <= 1.25 * float(aerr.mean()) + 1e-7, (name, float(err.mean()),
                                                                        float(aerr.mean()))


@pytest.mark.parametrize("hd", [64, 128])
def test_two_runs_are_bit_identical(rt, hd):
    for causal in (True, False):
        q, k, v, dout = R.inputs(2, 4, 1000, hd, seed=hd, layout="split", device="cuda")
        a = _native(q, k, v, dout, causal)
        b = _native(q, k, v, dout, causal)
        for x, y in zip(a, b):
            assert torch.equal(x, y)


def _gapped(B, H, T, hd, dtype, fill):
    """A [B, H, T, hd] view whose rows are hd + 16 apart inside a buffer with GUARD elements of
    `fill` on either side; every element the view does not cover holds `fill`."""
    w = hd + 16 if dtype == torch.bfloat16 else 8
    n = B * H * T * w
    buf = torch.full((n + 2 * GUARD,), fill, dtype=dtype, device="cuda")
    full = buf[GUARD:GUARD + n].view(B, H, T, w)
    return buf, full, (full[..., :hd] if dtype == torch.bfloat16 else full[..., :1].squeeze(-1))


def _untouched(buf, full, hd):
    nan = torch.isnan
    outside = torch.cat([buf[:GUARD], buf[-GUARD:]])
    gaps = full[..., hd:] if full.dtype == torch.bfloat16 else full[..., 1:]
    return bool(nan(outside).all()) and bool(nan(gaps).all())


@pytest.mark.parametrize("hd", [64, 128])
def test_outputs_stay_inside_their_rows(rt, hd):
    """Outputs written through strides with gaps between rows, guard bands on either side: the
    kernels write exactly the elements of their views, with the values of contiguous outputs."""
    from easydist_b200 import _lib
    B, H, T, causal = 2, 3, 129, True
    q, k, v, dout = R.inputs(B, H, T, hd, seed=11, layout="split", device="cuda")
    want = _native(q, k, v, dout, causal)
    bufs = [_gapped(B, H, T, hd, torch.bfloat16, float("nan")) for _ in range(4)]
    lbuf = _gapped(B, H, T, hd, torch.float32, float("nan"))
    out, dq, dk, dv = (b[2] for b in bufs)
    lse = lbuf[2]
    lib = _lib.load()
    st = lambda *ts: [s for t in ts for s in t.stride()[:3]]
    stream = torch.cuda.current_stream().cuda_stream
    scale = hd ** -0.5
    _lib.check(lib.edb_attn_fwd(out.data_ptr(), lse.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(),
                                B, H, T, hd, _lib.i64_array(st(q, k, v, out) + list(lse.stride())),
                                scale, 1, stream))
    nbytes = ctypes.c_size_t()
    _lib.check(lib.edb_attn_bwd_workspace(B, H, T, ctypes.byref(nbytes)))
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device="cuda")
    _lib.check(lib.edb_attn_bwd(dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), dout.data_ptr(), q.data_ptr(),
                                k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(), ws.data_ptr(),
                                B, H, T, hd,
                                _lib.i64_array(st(dout, q, k, v, out, dq, dk, dv) + list(lse.stride())),
                                scale, 1, stream))
    torch.cuda.synchronize()
    for (buf, full, view), w in zip(bufs, (want[0], want[2], want[3], want[4])):
        assert torch.equal(view, w)
        assert _untouched(buf, full, hd)
    assert torch.equal(lse, want[1]) and _untouched(lbuf[0], lbuf[1], hd)


def test_cuda_graph_replay_gives_the_eager_bits(rt):
    from easydist_b200 import attn
    q, k, v, dout = R.inputs(2, 4, 300, 64, seed=5, layout="split", device="cuda")
    want = _native(q, k, v, dout, True)
    statics = [t.clone() for t in (q, k, v, dout)]
    for t in statics:
        t.zero_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        attn.attention_fwd(*statics[:3], True)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out, lse = attn.attention_fwd(*statics[:3], True)
        grads = attn.attention_bwd(statics[3], *statics[:3], out, lse, True)
    for dst, src in zip(statics, (q, k, v, dout)):
        dst.copy_(src)
    g.replay()
    torch.cuda.synchronize()
    for got, w in zip((out, lse, *grads), want):
        assert torch.equal(got, w)


def _aten_cudnn(q, k, v, dout, causal):
    r = aten._scaled_dot_product_cudnn_attention.default(q, k, v, None, True, 0.0, causal)
    g = aten._scaled_dot_product_cudnn_attention_backward.default(
        dout, q, k, v, r[0], r[1], r[6], r[7], None, None, None, q.shape[2], q.shape[2], 0.0, causal)
    return r[0], r[1], *g


def test_the_cudnn_pair_off_the_kernel_runs_cudnn(rt):
    from easydist_b200 import attn
    q, k, v, dout = R.inputs(2, 3, 77, 96, seed=2, device="cuda")
    attn.reset_stats()
    out, lse = attn.attention_fwd(q, k, v, True, aten_op="cudnn")
    grads = attn.attention_bwd(dout, q, k, v, out, lse, True, aten_op="cudnn")
    assert attn.stats() == {"edb_attn_fwd": 0, "edb_attn_bwd": 0, "aten_attn_fwd": 1, "aten_attn_bwd": 1}
    for got, w in zip((out, lse, *grads), _aten_cudnn(q, k, v, dout, True)):
        assert torch.equal(got, w)


@pytest.mark.parametrize("case", ["fp16", "hd96", "unaligned"])
def test_what_the_kernels_do_not_take_runs_the_counted_aten_path(rt, case):
    from easydist_b200 import attn
    hd = 96 if case == "hd96" else 64
    q, k, v, dout = R.inputs(2, 3, 77, hd, seed=1, device="cuda")
    if case == "fp16":
        q, k, v, dout = (t.half() for t in (q, k, v, dout))
    if case == "unaligned":
        q, k, v = (torch.empty(t.numel() + 4, dtype=t.dtype, device="cuda")[4:].view(t.shape).copy_(t)
                   for t in (q, k, v))
    attn.reset_stats()
    out, lse = attn.attention_fwd(q, k, v, True)
    grads = attn.attention_bwd(dout, q, k, v, out, lse, True)
    assert attn.stats() == {"edb_attn_fwd": 0, "edb_attn_bwd": 0, "aten_attn_fwd": 1, "aten_attn_bwd": 1}
    # ATen's flash kernels need aligned pointers: the reference runs on aligned copies
    want = _aten(*(t.clone() for t in (q, k, v, dout)), True)
    for got, w in zip((out, lse, *grads), want):
        assert torch.equal(got, w)


@pytest.mark.parametrize("scale", [0.0, -0.125])
def test_a_non_positive_scale_runs_the_counted_aten_path(rt, scale):
    """The online softmax shifts by the row maximum of the raw scores, right for scale > 0 only."""
    from easydist_b200 import attn
    q, k, v, dout = R.inputs(2, 3, 77, 64, seed=3, device="cuda")
    attn.reset_stats()
    out, lse = attn.attention_fwd(q, k, v, True, scale)
    grads = attn.attention_bwd(dout, q, k, v, out, lse, True, scale)
    assert attn.stats() == {"edb_attn_fwd": 0, "edb_attn_bwd": 0, "aten_attn_fwd": 1, "aten_attn_bwd": 1}
    r = aten._scaled_dot_product_flash_attention.default(q, k, v, 0.0, True, scale=scale)
    g = aten._scaled_dot_product_flash_attention_backward.default(
        dout, q, k, v, r[0], r[1], r[2], r[3], r[4], r[5], 0.0, True, r[6], r[7], scale=scale)
    for got, w in zip((out, lse, *grads), (r[0], r[1], *g)):  # ATen's NaNs included
        assert torch.allclose(got, w, rtol=0, atol=0, equal_nan=True)


def test_broadcast_inputs_run_the_counted_aten_path(rt):
    """q, k, v expanded along B and H (stride 0) are not read through tensor maps."""
    from easydist_b200 import attn
    q, k, v, dout = R.inputs(1, 1, 77, 64, seed=4, device="cuda")
    q, k, v = (t.expand(2, 3, 77, 64) for t in (q, k, v))
    dout = dout.expand(2, 3, 77, 64).contiguous()
    attn.reset_stats()
    out, lse = attn.attention_fwd(q, k, v, True)
    grads = attn.attention_bwd(dout, q, k, v, out, lse, True)
    assert attn.stats() == {"edb_attn_fwd": 0, "edb_attn_bwd": 0, "aten_attn_fwd": 1, "aten_attn_bwd": 1}
    want = _aten(*(t.contiguous() for t in (q, k, v, dout)), True)
    for got, w in zip((out, lse, *grads), want):
        assert torch.equal(got, w)


# ---- compiled steps --------------------------------------------------------------------------------

class _Deterministic:
    """torch.use_deterministic_algorithms(True, warn_only=True) inside, restored on exit: the
    request under which the compiled steps run attention on edb_attn.cu."""

    def __enter__(self):
        self.was = (torch.are_deterministic_algorithms_enabled(),
                    torch.is_deterministic_algorithms_warn_only_enabled())
        torch.use_deterministic_algorithms(True, warn_only=True)

    def __exit__(self, *exc):
        torch.use_deterministic_algorithms(self.was[0], warn_only=self.was[1])


def _train(model_fn, cfg, cuda_graph):
    from easydist_b200 import attn
    from easydist_b200.api import easydist_compile
    from easydist_b200.workloads import gpt2_train_step, synthetic_tokens
    from tools import parity as P
    torch.manual_seed(0)
    model = model_fn().to(device="cuda", dtype=torch.bfloat16)
    state = {k: v.detach().clone() for k, v in model.state_dict().items()}
    mk_opt = lambda ps: torch.optim.SGD(ps, lr=1e-3, momentum=0.9, foreach=True)
    opt = mk_opt(model.parameters())
    step = easydist_compile(gpt2_train_step, parallel_mode="ddp", tracing_mode="fake",
                            cuda_graph=cuda_graph)
    calls = 4
    attn.reset_stats()
    batches = [synthetic_tokens(cfg, 4, 64, seed=1000 * b) for b in range(calls)]
    with _Deterministic():
        losses = [float(step(tok.cuda(), tgt.cuda(), model, opt)) for tok, tgt in batches]
    info = step.compiled_func.info
    assert info["attn_nodes"] == (cfg.n_layer, cfg.n_layer), info
    gm = step.compiled_func.graph
    left = [n for n in gm.graph.nodes if n.op == "call_function" and "attention" in str(n.target)
            and n.target not in (attn.attention_fwd, attn.attention_bwd)]
    assert not left, left
    sched = ([0, 0] if cuda_graph else [0]) + list(range(1, calls))
    steps = [[batches[b]] for b in sched]
    ref_l, ref_p, ref_s = P.vanilla_run(model_fn, state, steps, mk_opt, torch.float32, "cuda")
    idx = [1 if cuda_graph else 0] + list(range(2 if cuda_graph else 1, len(sched)))
    for got, i in zip(losses, idx):
        assert abs(got - ref_l[i][0]) <= 3e-2 * abs(ref_l[i][0]), (losses, ref_l)
    got_p, got_s = P.compiled_state(step.compiled_func, ref_p, ref_s, 1)
    _, van_p, van_s = P.vanilla_run(model_fn, state, steps, mk_opt, torch.bfloat16, "cuda")
    van = P.compare({k: v.bfloat16() for k, v in van_p.items()},
                    {k: {kk: vv.bfloat16() for kk, vv in st.items()} for k, st in van_s.items()},
                    ref_p, ref_s, low_precision=True)
    res = P.compare(got_p, got_s, ref_p, ref_s, low_precision=True)
    assert res["state_rel_l2"] <= max(2e-2, 2.0 * van["state_rel_l2"]), (res, van)
    assert res["param_max_ulp"] <= max(2.0, 2.0 * van["param_max_ulp"]), (res, van)
    st = attn.stats()
    assert st["aten_attn_fwd"] == 0 and st["aten_attn_bwd"] == 0, st
    assert st["edb_attn_fwd"] > 0 and st["edb_attn_bwd"] > 0, st


@pytest.mark.parametrize("cuda_graph", [False, True])
def test_small_gpt2_trains_like_vanilla_with_native_attention(rt, cuda_graph):
    from easydist_b200.workloads import GPT2, GPT2Config
    cfg = GPT2Config(2, 4, 256, vocab_size=1000, block_size=64)
    _train(lambda: GPT2(cfg), cfg, cuda_graph)


@pytest.mark.parametrize("cuda_graph", [False, True])
def test_small_llama_trains_like_vanilla_with_native_attention(rt, cuda_graph):
    from easydist_b200.workloads import Llama, LlamaConfig
    cfg = LlamaConfig(n_layer=2, n_head=4, n_embd=256, ffn=688, vocab_size=512, block_size=64)
    _train(lambda: Llama(cfg), cfg, cuda_graph)


def test_a_deterministic_step_repeats_its_bits(rt):
    """The reason the rewrite exists: under deterministic algorithms two compilations of the
    GPT-2 step from the same weights, fed the same batches, give bit-identical losses, weights and
    momentum buffers."""
    from easydist_b200 import attn
    from easydist_b200.api import easydist_compile
    from easydist_b200.workloads import GPT2, GPT2Config, gpt2_train_step, synthetic_tokens
    cfg = GPT2Config(2, 4, 256, vocab_size=1000, block_size=128)
    batches = [synthetic_tokens(cfg, 4, 128, seed=b) for b in range(3)]
    runs = []
    for _ in range(2):
        torch.manual_seed(0)
        model = GPT2(cfg).to(device="cuda", dtype=torch.bfloat16)
        opt = torch.optim.SGD(model.parameters(), lr=1e-3, momentum=0.9, foreach=True)
        step = easydist_compile(gpt2_train_step, parallel_mode="ddp", tracing_mode="fake",
                                cuda_graph=False)
        attn.reset_stats()
        with _Deterministic():
            losses = [step(tok.cuda(), tgt.cuda(), model, opt).detach().clone() for tok, tgt in batches]
        assert attn.stats()["edb_attn_bwd"] == 3 * cfg.n_layer, attn.stats()
        params, _, states = step.compiled_func.get_state()
        runs.append((losses, {k: v.detach().clone() for k, v in params.items()},
                     {k: {kk: vv.detach().clone() for kk, vv in st.items()} for k, st in states.items()}))
    (l0, p0, s0), (l1, p1, s1) = runs
    assert all(torch.equal(a, b) for a, b in zip(l0, l1))
    for k in p0:
        assert torch.equal(p0[k], p1[k]), k
        for kk in s0[k]:
            assert torch.equal(s0[k][kk], s1[k][kk]), (k, kk)
