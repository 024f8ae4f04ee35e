"""The RoPE kernel (edb_rope.cu) on one H100: bit for bit against the ATen chains of both RoPE forms,
forward and backward, over head dims, sequence lengths, input and output layouts and unaligned
operands; guard bands; CUDA-graph capture; the counted ATen path for what the kernel does not take;
and a small Llama of either form trained through the compiled path against vanilla fp32 PyTorch."""
import ctypes

import pytest
import torch

from tests import rope_forms as RF

pytestmark = pytest.mark.gpu


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


def _offset(t, off):
    """A copy of t whose storage starts `off` elements into its allocation (same strides)."""
    if off == 0:
        return t
    buf = torch.empty(t.numel() + off, dtype=t.dtype, device=t.device)
    out = buf[off:].view(t.shape) if t.is_contiguous() else None
    if out is None:  # the transposed view: [B, T, H, hd] storage
        out = buf[off:].view(t.transpose(1, 2).shape).transpose(1, 2)
    out.copy_(t)
    return out


def _inputs(B, H, T, hd, dtype, layout, off, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if layout == "transposed":  # the projection output viewed as [B, H, T, hd]
        x = (torch.randn(B, T, H, hd, device="cuda", generator=g) * 3).to(dtype).transpose(1, 2)
    else:
        x = (torch.randn(B, H, T, hd, device="cuda", generator=g) * 3).to(dtype)
    dy = torch.randn(B, H, T, hd, device="cuda", generator=g).to(dtype)
    cos, sin = RF.tables(T, hd, dtype, "cuda")
    return tuple(_offset(t, off) for t in (x, dy, cos, sin))


def _chains(x, dy, cos, sin):
    """(forward, gradient) of both forms through ATen / autograd."""
    outs = []
    for fn in (RF.rope_half_split, RF.rope_rotate_half):
        xx = x.detach().clone().requires_grad_(True)
        y = fn(xx, cos, sin)
        y.backward(dy)
        outs.append((y.detach(), xx.grad))
    return outs


def _same_bits(a, b):
    it = torch.int16 if a.dtype == torch.bfloat16 else torch.int32
    return a.shape == b.shape and torch.equal(a.contiguous().view(it), b.contiguous().view(it))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("T", [1, 7, 2048])
@pytest.mark.parametrize("hd", [6, 16, 64, 128, 256])
def test_rope_kernel_equals_aten_chains(rt, hd, T, dtype):
    """hd 6 takes the scalar path; offset 1 puts x, dy and both tables one element past 16-byte
    alignment (scalar path); both output layouts of the forward and of the backward."""
    from easydist_b200 import rope
    B, H = (4, 32) if hd <= 128 else (2, 16)
    rope.reset_stats()
    calls = 0
    for layout in ("contiguous", "transposed"):
        for off in (0, 1):
            x, dy, cos, sin = _inputs(B, H, T, hd, dtype, layout, off, seed=hd * 7 + T + off)
            (ya, ga), (yb, gb) = _chains(x, dy, cos, sin)
            y = rope.rope(x, cos, sin)
            y_strided = rope.rope(x, cos, sin, False, stride=list(x.stride()))
            g = rope.rope(dy, cos, sin, True)
            g_t = rope.rope(dy, cos, sin, True, transposed=True)
            calls += 4
            ctx = (layout, off)
            assert y.is_contiguous() and y_strided.stride() == x.stride(), ctx
            assert g_t.is_contiguous() and g_t.shape == (B, T, H, hd), ctx
            for want in (ya, yb):
                assert _same_bits(y, want) and _same_bits(y_strided, want), ctx
            for want in (ga, gb):
                assert _same_bits(g, want), ctx
                assert _same_bits(g_t, want.transpose(1, 2).contiguous()), ctx
    st = rope.stats()
    assert st["aten_rope"] == 0 and st["edb_rope_fwd"] + st["edb_rope_bwd"] == calls, st


def _call(y, x, cos, sin, ys, inverse=0, half=None):
    from easydist_b200 import _lib, norm
    B, H, T, hd = x.shape
    xs = (ctypes.c_int64 * 3)(*x.stride()[:3])
    yv = (ctypes.c_int64 * 3)(*ys)
    return _lib.load().edb_rope(y.data_ptr(), x.data_ptr(), cos.data_ptr(), sin.data_ptr(), B, H, T,
                                hd // 2 if half is None else half, xs, yv, cos.stride(0), inverse,
                                norm._DT[x.dtype], torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("hd", [6, 128])
def test_rope_writes_stay_inside_outputs(rt, hd, dtype):
    """Outputs at offsets 0 and 1 inside buffers whose guard bands hold NaN, in the [B, H, T, hd]
    and the [B, T, H, hd] layout."""
    B, H, T, pad = 3, 5, 37, 4096
    for layout in ("contiguous", "transposed"):
        for off in (0, 1):
            x, dy, cos, sin = _inputs(B, H, T, hd, dtype, "transposed", 0, seed=hd + off)
            (want, _), _ = _chains(x, dy, cos, sin)
            n = x.numel()
            buf = torch.full((n + 2 * pad + off,), float("nan"), dtype=dtype, device="cuda")
            inner = buf[pad + off:pad + off + n]
            if layout == "contiguous":
                y = inner.view(B, H, T, hd)
            else:
                y = inner.view(B, T, H, hd).transpose(1, 2)
            assert _call(y, x, cos, sin, y.stride()[:3]) == 0
            torch.cuda.synchronize()
            assert torch.isnan(buf[:pad + off]).all() and torch.isnan(buf[pad + off + n:]).all()
            assert _same_bits(y, want), (layout, off)


def test_rope_rejects_malformed_arguments(rt):
    from easydist_b200 import _lib
    x, dy, cos, sin = _inputs(2, 2, 8, 16, torch.bfloat16, "contiguous", 0, seed=1)
    y = torch.full_like(x, float("nan"))
    ok = list(y.stride()[:3])
    for kw, ys in (({"half": 0}, ok), ({"half": 257}, ok), ({}, [-1, 0, 0])):
        assert _call(y, x, cos, sin, ys, **kw) in (_lib.EDB_E_INVALID, _lib.EDB_E_UNSUPPORTED), kw
    assert _call(x, x, cos, sin, ok) == _lib.EDB_E_INVALID  # y aliases x
    torch.cuda.synchronize()
    assert torch.isnan(y).all()


def test_unsupported_arguments_take_the_counted_aten_path(rt):
    from easydist_b200 import rope
    cases = []
    x, _, cos, sin = _inputs(2, 3, 5, 520, torch.bfloat16, "contiguous", 0, seed=2)
    cases.append((x, cos, sin))  # head dim above 512
    x, _, cos, sin = _inputs(2, 3, 5, 32, torch.float32, "contiguous", 0, seed=3)
    cases.append((torch.repeat_interleave(x, 2, dim=-1)[..., ::2], cos, sin))  # last-dim stride 2
    for x, cos, sin in cases:
        rope.reset_stats()
        y, g = rope.rope(x, cos, sin), rope.rope(x, cos, sin, True)
        assert torch.equal(y, RF.rope_half_split(x, cos, sin))
        assert torch.equal(g, rope._chain(x, cos, sin, True))
        assert rope.stats() == {"edb_rope_fwd": 0, "edb_rope_bwd": 0, "aten_rope": 2}
    # an odd head dim has no [T, hd/2] table: the counted ATen path raises what the chain raises
    _, _, cos, sin = _inputs(2, 3, 5, 8, torch.bfloat16, "contiguous", 0, seed=4)
    x = torch.randn(2, 3, 5, 7, device="cuda").bfloat16()
    rope.reset_stats()
    with pytest.raises(RuntimeError):
        rope.rope(x, cos[:, :3], sin[:, :3])
    assert rope.stats()["aten_rope"] == 1 and rope.stats()["edb_rope_fwd"] == 0


def test_cuda_graph_capture_gives_the_eager_bits(rt):
    from easydist_b200 import rope
    runs = []
    for dtype in (torch.bfloat16, torch.float32):
        x, dy, cos, sin = _inputs(4, 32, 2048, 128, dtype, "transposed", 0, seed=11)
        xo, dyo, co, so = _inputs(2, 4, 7, 6, dtype, "contiguous", 1, seed=12)

        def step():
            return [rope.rope(x, cos, sin), rope.rope(x, cos, sin, False, stride=list(x.stride())),
                    rope.rope(dy, cos, sin, True), rope.rope(dy, cos, sin, True, transposed=True),
                    rope.rope(xo, co, so), rope.rope(dyo, co, so, True, transposed=True)]

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
        runs.append(all(_same_bits(a, b) for a, b in zip(eager, captured)))
    assert all(runs), runs


# ---- end to end -------------------------------------------------------------------------------

@pytest.mark.parametrize("form", RF.FORMS)
@pytest.mark.parametrize("dtype,cuda_graph", [(torch.float32, False), (torch.float32, True),
                                              (torch.bfloat16, False), (torch.bfloat16, True)])
def test_small_llama_trains_like_vanilla_with_native_rope(rt, form, dtype, cuda_graph):
    """As tests/test_gpu_rms_swiglu.py: losses and every parameter / optimizer state against vanilla
    fp32 PyTorch (fp32: the reference's assert_close; bf16: calibrated by vanilla bf16)."""
    from easydist_b200 import rope
    from easydist_b200.api import easydist_compile
    from easydist_b200.workloads import LlamaConfig, gpt2_train_step, synthetic_tokens
    from tools import parity as P
    cfg = LlamaConfig(n_layer=2, n_head=4, n_embd=256, ffn=688, vocab_size=512, block_size=64)
    make = lambda: RF.llama(cfg, form)
    torch.manual_seed(0)
    model = make().to(device="cuda", dtype=dtype)
    state = {k: v.detach().clone() for k, v in model.state_dict().items()}
    mk_opt = lambda ps: torch.optim.SGD(ps, lr=1e-3, momentum=0.9, foreach=True)
    opt = mk_opt(model.parameters())
    step = easydist_compile(gpt2_train_step, parallel_mode="ddp", tracing_mode="fake",
                            cuda_graph=cuda_graph)
    calls = 4
    rope.reset_stats()
    batches = [synthetic_tokens(cfg, 4, 64, seed=1000 * b) for b in range(calls)]
    losses = [float(step(tok.cuda(), tgt.cuda(), model, opt)) for tok, tgt in batches]
    info = step.compiled_func.info
    assert info["rope_nodes"] == (4, 4), info
    sched = ([0, 0] if cuda_graph else [0]) + list(range(1, calls))
    steps = [[batches[b]] for b in sched]
    ref_l, ref_p, ref_s = P.vanilla_run(make, state, steps, mk_opt, torch.float32, "cuda")
    idx = [1 if cuda_graph else 0] + list(range(2 if cuda_graph else 1, len(sched)))
    rtol = 1e-4 if dtype == torch.float32 else 3e-2
    for got, i in zip(losses, idx):
        assert abs(got - ref_l[i][0]) <= rtol * abs(ref_l[i][0]), (losses, ref_l)
    got_p, got_s = P.compiled_state(step.compiled_func, ref_p, ref_s, 1)
    if dtype == torch.float32:
        res = P.compare(got_p, got_s, ref_p, ref_s, low_precision=False)
        assert res["assert_close_violation"] <= 1.0, res
    else:
        _, van_p, van_s = P.vanilla_run(make, state, steps, mk_opt, torch.bfloat16, "cuda")
        van = P.compare({k: v.bfloat16() for k, v in van_p.items()},
                        {k: {kk: vv.bfloat16() for kk, vv in st.items()} for k, st in van_s.items()},
                        ref_p, ref_s, low_precision=True)
        res = P.compare(got_p, got_s, ref_p, ref_s, low_precision=True)
        assert res["state_rel_l2"] <= max(2e-2, 2.0 * van["state_rel_l2"]), (res, van)
        assert res["param_max_ulp"] <= max(2.0, 2.0 * van["param_max_ulp"]), (res, van)
    st = rope.stats()
    assert st["aten_rope"] == 0 and st["edb_rope_fwd"] > 0 and st["edb_rope_bwd"] > 0, st
