"""RMSNorm and SwiGLU kernels (edb_rms.cu) on one H100: RMSNorm against a float64 evaluation of the
same formula under the bounds derived in tests/rms_ref.py, SwiGLU bit for bit against the ATen chains
it replaces, CUDA-graph capture, and a small Llama trained through the compiled path against vanilla
fp32 PyTorch."""
import pytest
import torch
import torch.nn as nn

from tests import rms_ref as R

pytestmark = pytest.mark.gpu
aten = torch.ops.aten


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


def _inputs(rows, H, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(rows, H, device="cuda", generator=g) * 2 + 0.1).to(dtype)
    w = (torch.randn(H, device="cuda", generator=g) * 0.5 + 1).to(dtype)
    dy = torch.randn(rows, H, device="cuda", generator=g).to(dtype)
    add = torch.randn(rows, H, device="cuda", generator=g).to(dtype)
    return x, w, dy, add


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("rows", [1, 7, 4096, 16384])
@pytest.mark.parametrize("H", [64, 256, 1024, 4096, 5120, 8192, 16384])
def test_rms_norm_kernels_within_float64_bound(rt, H, rows, dtype):
    from easydist_b200 import norm
    x, w, dy, add = _inputs(rows, H, dtype, seed=H + rows)
    eps = 1e-5
    norm.reset_stats()
    for mode in (R.CAST, R.FUSED):
        y, rstd = norm.rms_norm_fwd(x, w, eps, mode)
        y64, r64, nhat, flip = R.forward_ref(x, w, eps, mode)
        assert rstd.shape == (rows, 1) and rstd.dtype == torch.float32
        assert R.worst(rstd, r64, R.rstd_bound(x, r64)) <= 1.0, (mode, "rstd")
        assert R.worst(y, y64, R.forward_bound(x, w, y64, nhat, flip, mode)) <= 1.0, (mode, "y")
        for a, mask in ((None, [True, True]), (add, [True, True]), (add, [True, False])):
            dx, dw = norm.rms_norm_bwd(dy, x, rstd, w, mode, mask, _add=a)
            dx64, dw64, M, S = R.backward_ref(dy, x, w, r64, mode, a)
            assert R.worst(dx, dx64, R.dx_bound(x, dx64, M, a)) <= 1.0, (mode, a is not None, "dx")
            if not mask[1]:
                assert dw is None
                continue
            assert R.worst(dw, dw64, R.dw_bound(dy, x, dw64, S, flip, nhat, mode)) <= 1.0, (mode, "dw")
            _, dw2 = norm.rms_norm_bwd(dy, x, rstd, w, mode, mask, _add=a)
            assert torch.equal(dw, dw2), "dw is not deterministic"
    st = norm.stats()
    # per mode: three backward calls plus the two repeats of the determinism check
    assert st["aten_rms"] == 0 and st["edb_rms_fwd"] == 2 and st["edb_rms_bwd"] == 10, st


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("H", [64, 1024, 4096, 16384])
def test_rms_norm_writes_stay_inside_outputs(rt, H, dtype):
    """Every output sits inside a buffer whose guard bands (before and after) hold a NaN pattern."""
    from easydist_b200 import _lib, norm
    from ctypes import byref, c_size_t
    rows, pad = 37, 4096
    x, w, dy, add = _inputs(rows, H, dtype, seed=3)
    lib = _lib.load()
    code = norm._DT[dtype]
    st = torch.cuda.current_stream().cuda_stream

    def guarded(n, dt):
        buf = torch.full((n + 2 * pad,), float("nan"), dtype=dt, device="cuda")
        return buf, buf[pad:pad + n]

    ybuf, y = guarded(rows * H, dtype)
    rbuf, rstd = guarded(rows, torch.float32)
    _lib.check(lib.edb_rms_norm_fwd(y.data_ptr(), rstd.data_ptr(), x.data_ptr(), w.data_ptr(), rows, H,
                                    1e-5, R.CAST, code, st))
    dxbuf, dx = guarded(rows * H, dtype)
    dwbuf, dw = guarded(H, dtype)
    nbytes = c_size_t()
    _lib.check(lib.edb_rms_norm_bwd_workspace(H, byref(nbytes)))
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device="cuda")
    _lib.check(lib.edb_rms_norm_bwd(dx.data_ptr(), dw.data_ptr(), dy.data_ptr(), x.data_ptr(),
                                    rstd.data_ptr(), w.data_ptr(), add.data_ptr(), ws.data_ptr(), rows,
                                    H, R.CAST, code, st))
    torch.cuda.synchronize()
    for buf, inner in ((ybuf, y), (rbuf, rstd), (dxbuf, dx), (dwbuf, dw)):
        assert torch.isnan(buf[:pad]).all() and torch.isnan(buf[-pad:]).all()
        assert not torch.isnan(inner).any()


def test_rms_norm_unsupported_width_takes_the_counted_aten_path(rt):
    from easydist_b200 import norm
    for H, dtype in ((20000, torch.float32), (60, torch.bfloat16), (16392, torch.bfloat16)):
        x, w, dy, _ = _inputs(5, H, dtype, seed=1)
        norm.reset_stats()
        y, rstd = norm.rms_norm_fwd(x, w, 1e-5, R.CAST)
        dx, dw = norm.rms_norm_bwd(dy, x, rstd, w, R.CAST, [True, True])
        want_y, want_r = norm._rms_fwd_chain(x, w, 1e-5)
        want_dx, want_dw = norm._rms_bwd_chain(dy, x, want_r, w, [True, True], None)
        assert torch.equal(y, want_y) and torch.equal(dx, want_dx) and torch.equal(dw, want_dw)
        st = norm.stats()
        assert st["aten_rms"] == 2 and st["edb_rms_fwd"] == 0 and st["edb_rms_bwd"] == 0, st


def _swiglu_chain(gate, up, dy):
    out = aten.mul.Tensor(aten.silu.default(gate), up)
    dup = aten.mul.Tensor(dy, aten.silu.default(gate))
    dgate = aten.silu_backward.default(aten.mul.Tensor(dy, up), gate)
    return out, dgate, dup


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("n,offset", [(8 * 11008, 0), (4096 * 11008 + 5, 0), (1000003, 0), (7, 0),
                                      (65536, 1), (12345, 3)])
def test_swiglu_kernels_equal_aten_chains(rt, dtype, n, offset):
    """offset > 0: every operand starts `offset` elements into its allocation (not 16-byte aligned)."""
    from easydist_b200 import act
    g = torch.Generator(device="cuda").manual_seed(n)
    gate, up, dy = (torch.randn(n + offset, device="cuda", generator=g).mul(4).to(dtype)[offset:]
                    for _ in range(3))
    act.reset_stats()
    out = act.swiglu_fwd(gate, up)
    dgate, dup = act.swiglu_bwd(dy, gate, up)
    want_out, want_dgate, want_dup = _swiglu_chain(gate, up, dy)
    assert torch.equal(out, want_out)
    assert torch.equal(dgate, want_dgate)
    assert torch.equal(dup, want_dup)
    st = act.stats()
    assert st["edb_swiglu_fwd"] == 1 and st["edb_swiglu_bwd"] == 1 and st["aten_swiglu"] == 0, st


def test_cuda_graph_capture_gives_the_eager_bits(rt):
    from easydist_b200 import act, norm
    runs = []
    for dtype in (torch.bfloat16, torch.float32):
        x, w, dy, add = _inputs(4096, 4096, dtype, seed=11)
        gate, up, gdy = (t.reshape(-1)[:4096 * 1000 + 3] for t in (x, dy, add))

        def step(x=x, w=w, dy=dy, add=add, gate=gate, up=up, gdy=gdy):
            outs = []
            for mode in (R.CAST, R.FUSED):
                y, rstd = norm.rms_norm_fwd(x, w, 1e-5, mode)
                outs += [y, rstd, *norm.rms_norm_bwd(dy, x, rstd, w, mode, [True, True], _add=add)]
            outs.append(act.swiglu_fwd(gate, up))
            outs += list(act.swiglu_bwd(gdy, gate, up))
            return outs

        eager = step()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step()  # warm-up on the capture stream (workspaces allocated)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            captured = step()
        graph.replay()
        torch.cuda.synchronize()
        runs.append(all(torch.equal(a, b) for a, b in zip(eager, captured)))
    assert all(runs), runs


# ---- end to end -------------------------------------------------------------------------------

def _small_llama_cfg():
    from easydist_b200.workloads import LlamaConfig
    return LlamaConfig(n_layer=2, n_head=4, n_embd=256, ffn=688, vocab_size=512, block_size=64)


def _llama_with_torch_rmsnorm(cfg):
    """The same model with every RMSNorm replaced by torch.nn.RMSNorm (same parameter names)."""
    from easydist_b200.workloads import Llama, RMSNorm
    m = Llama(cfg)
    for mod in list(m.modules()):
        for name, child in list(mod.named_children()):
            if isinstance(child, RMSNorm):
                setattr(mod, name, nn.RMSNorm(cfg.n_embd, eps=cfg.eps))
    return m


@pytest.mark.parametrize("variant", ["workloads", "nn.RMSNorm"])
@pytest.mark.parametrize("dtype,cuda_graph", [(torch.float32, False), (torch.float32, True),
                                              (torch.bfloat16, False), (torch.bfloat16, True)])
def test_small_llama_trains_like_vanilla_on_native_kernels(rt, variant, dtype, cuda_graph):
    """As tests/test_gpu_train.py for GPT-2: losses and every parameter / optimizer state against
    vanilla fp32 PyTorch (fp32: the reference's assert_close; bf16: calibrated by vanilla bf16)."""
    from easydist_b200 import act, norm
    from easydist_b200.api import easydist_compile
    from easydist_b200.workloads import Llama, gpt2_train_step, synthetic_tokens
    from tools import parity as P
    cfg = _small_llama_cfg()
    make = (lambda: Llama(cfg)) if variant == "workloads" else (lambda: _llama_with_torch_rmsnorm(cfg))
    torch.manual_seed(0)
    model = make().to(device="cuda", dtype=dtype)
    state = {k: v.detach().clone() for k, v in model.state_dict().items()}
    mk_opt = lambda ps: torch.optim.SGD(ps, lr=1e-3, momentum=0.9, foreach=True)
    opt = mk_opt(model.parameters())
    step = easydist_compile(gpt2_train_step, parallel_mode="ddp", tracing_mode="fake",
                            cuda_graph=cuda_graph)
    calls = 4
    norm.reset_stats()
    act.reset_stats()
    batches = [synthetic_tokens(cfg, 4, 64, seed=1000 * b) for b in range(calls)]
    losses = [float(step(tok.cuda(), tgt.cuda(), model, opt)) for tok, tgt in batches]
    info = step.compiled_func.info
    assert info["rms_norm_nodes"] == (5, 5) and info["swiglu_nodes"] == (2, 2), info
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
    st, ast = norm.stats(), act.stats()
    assert st["aten_rms"] == 0 and st["edb_rms_fwd"] > 0 and st["edb_rms_bwd"] > 0, st
    assert ast["aten_swiglu"] == 0 and ast["edb_swiglu_fwd"] > 0 and ast["edb_swiglu_bwd"] > 0, ast
