"""The gradient-clipping kernels (edb_clip.cu, edb_sgd_momentum_scaled) on H100s: the sum of squares
within the bound of tests/clip_ref.py over mixed tensor lists (tiny to 50257x1024, > 300 tensors,
unaligned operands, transposed views), NORM = T(sqrt(RAW)), determinism, guard bands, CUDA-graph
capture and error statuses; the scale kernels bit for bit against ATen's mul_ (+ the SGD chain); a
small Llama trained with clipping through the compiled path against vanilla fp32 PyTorch; and a
zero3 step with clipping on 2 GPUs."""
import ctypes
import os
import sys

import pytest
import torch

from tests import clip_ref as R

pytestmark = pytest.mark.gpu
aten = torch.ops.aten
SIZES = [1, 7, 8, 4095, (1 << 20) + 3, 50257 * 1024]


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


def _tensor(n, dtype, seed, off=0, scale=1.0):
    """n random elements starting `off` elements into their allocation."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.empty(n + off, dtype=dtype, device="cuda")
    buf[off:] = (torch.randn(n, generator=g, device="cuda") * scale).to(dtype)
    return buf[off:]


def _mixed(dtype):
    ts = [_tensor(n, dtype, i) for i, n in enumerate(SIZES)]
    ts += [_tensor(n, dtype, 100 + i, off=1) for i, n in enumerate(SIZES[:5])]  # 1 element off 16 B
    ts.append(_tensor(1024 * 4096, dtype, 7).view(1024, 4096).t())             # weight-gradient view
    ts.append(_tensor(64 * 48, dtype, 8, off=3).view(64, 48).t())
    return ts


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_sumsq_within_the_bound_and_norm_is_its_sqrt(rt, dtype):
    from easydist_b200 import clip
    ts = _mixed(dtype)
    clip.reset_stats()
    raw = clip.grad_sumsq(ts)
    assert raw.dtype == torch.float32 and R.worst(raw.cpu().double(), ts) <= 1.0
    norms = clip.grad_norms(ts)
    assert norms.dtype == dtype and torch.equal(norms, torch.sqrt(raw).to(dtype))
    assert torch.equal(clip.grad_sumsq(ts), raw)  # deterministic
    assert clip.stats() == {"edb_sumsq": 3, "aten_sumsq": 0, "edb_scale": 0, "aten_scale": 0}


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_sumsq_over_330_tensors(rt, dtype):
    from easydist_b200 import clip
    g = torch.Generator().manual_seed(3)
    sizes = torch.randint(1, 70000, (330,), generator=g).tolist()
    ts = [_tensor(n, dtype, i, off=i % 3, scale=0.1 + i % 5) for i, n in enumerate(sizes)]
    raw = clip.grad_sumsq(ts)
    assert R.worst(raw.cpu().double(), ts) <= 1.0
    assert torch.equal(clip.grad_norms(ts), torch.sqrt(raw).to(dtype))


def _raw_call(ts, out, ws, mode, dtype_code):
    from easydist_b200 import _lib
    from easydist_b200.optim import _ptr_array
    return _lib.load().edb_grad_sumsq(len(ts), _ptr_array(ts), _lib.i64_array([t.numel() for t in ts]),
                                      out, ws, mode, dtype_code, torch.cuda.current_stream().cuda_stream)


def test_guard_bands_and_error_statuses(rt):
    from easydist_b200 import _lib
    ts = _mixed(torch.bfloat16)
    code = _lib.DTYPE_CODES["bfloat16"]
    nbytes = ctypes.c_size_t()
    assert _lib.load().edb_grad_sumsq_workspace(len(ts), _lib.i64_array([t.numel() for t in ts]),
                                                code, ctypes.byref(nbytes)) == 0
    ws = torch.full((nbytes.value // 4 + 64,), 7.0, device="cuda")
    out = torch.full((len(ts) + 64,), -3.0, device="cuda")
    assert _raw_call(ts, out[32:].data_ptr(), ws[32:].data_ptr(), 0, code) == 0
    torch.cuda.synchronize()
    assert (out[:32] == -3.0).all() and (out[32 + len(ts):] == -3.0).all()
    assert (ws[:32] == 7.0).all() and (ws[32 + nbytes.value // 4:] == 7.0).all()
    assert R.worst(out[32:32 + len(ts)].cpu().double(), ts) <= 1.0
    lib = _lib.load()
    before = lib.edb_launch_count()
    assert _raw_call(ts, out.data_ptr(), ws.data_ptr(), 5, code) == _lib.EDB_E_INVALID
    assert _raw_call(ts, out.data_ptr(), None, 0, code) == _lib.EDB_E_INVALID
    assert _raw_call(ts, out.data_ptr(), ws.data_ptr(), 0, _lib.DTYPE_CODES["int32"]) == \
        _lib.EDB_E_UNSUPPORTED
    bad = lib.edb_grad_sumsq(1, (ctypes.c_void_p * 1)(ts[0].data_ptr()), _lib.i64_array([-1]),
                             out.data_ptr(), ws.data_ptr(), 0, code, None)
    assert bad == _lib.EDB_E_INVALID
    assert lib.edb_multi_scale_(1, (ctypes.c_void_p * 1)(ts[0].data_ptr()), _lib.i64_array([1]), None,
                                code, None) == _lib.EDB_E_INVALID
    assert lib.edb_launch_count() == before


def test_cuda_graph_capture_gives_the_eager_bits(rt):
    from easydist_b200 import clip
    ts = _mixed(torch.bfloat16) + _mixed(torch.float32)
    bf, f32 = ts[:len(ts) // 2], ts[len(ts) // 2:]

    def step():
        return [clip.grad_sumsq(bf), clip.grad_norms(bf), clip.grad_sumsq(f32), clip.grad_norms(f32)]

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
    assert all(torch.equal(a, b) for a, b in zip(eager, captured))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_scale_kernels_match_aten_mul_(rt, dtype):
    from easydist_b200 import clip, optim
    coef = torch.tensor(0.3171, device="cuda").to(dtype)
    sizes = [1, 7, 8, 4095, (1 << 20) + 3, 50257 * 1024 // 4]
    # multi_scale_: aligned and unaligned tensors, against the per-tensor mul_
    ts = [_tensor(n, dtype, i, off=i % 2) for i, n in enumerate(sizes)]
    want = [t.clone().mul_(coef) for t in ts]
    clip.reset_stats()
    clip.scale_(ts, coef)
    assert all(torch.equal(a, b) for a, b in zip(ts, want))
    # a view that is not dense takes the counted ATen path
    big = _tensor(64 * 64, dtype, 9).view(64, 64)[:, :32]
    w2 = big.clone().mul_(coef)
    clip.scale_([big], coef)
    assert torch.equal(big, w2) and clip.stats()["edb_scale"] == 1 and clip.stats()["aten_scale"] == 1
    # sgd_momentum_(grad_scale=c) against mul_ + the three ATen ops; one unaligned tensor takes the
    # counted ATen path
    params = [_tensor(n, dtype, 10 + i) for i, n in enumerate(sizes)]
    grads = [_tensor(n, dtype, 20 + i) for i, n in enumerate(sizes)]
    bufs = [_tensor(n, dtype, 30 + i) for i, n in enumerate(sizes)]
    params.append(_tensor(1000, dtype, 40, off=1))
    grads.append(_tensor(1000, dtype, 41))
    bufs.append(_tensor(1000, dtype, 42))
    rp, rg, rb = [t.clone() for t in params], [t.clone() for t in grads], [t.clone() for t in bufs]
    for g in rg:
        g.mul_(coef)
    aten._foreach_mul_.Scalar(rb, 0.9)
    aten._foreach_add_.List(rb, rg, alpha=1.0)
    aten._foreach_add_.List(rp, rb, alpha=-0.01)
    g_before = [g.clone() for g in grads]
    optim.reset_stats()
    optim.sgd_momentum_(params, grads, bufs, 0.9, 1.0, -0.01, grad_scale=coef)
    assert all(torch.equal(a, b) for a, b in zip(params, rp))
    assert all(torch.equal(a, b) for a, b in zip(bufs, rb))
    assert all(torch.equal(a, b) for a, b in zip(grads, g_before))  # gradients are not written
    assert optim.stats() == {"edb_sgd": 1, "aten_sgd": 1}


# ---- end to end -------------------------------------------------------------------------------

MAX_NORM = 0.2


def _clipped(opt_cls):
    class Clipped(opt_cls):
        """The vanilla reference: clip_grad_norm_ in front of every step."""

        def step(self, closure=None):
            torch.nn.utils.clip_grad_norm_([p for g in self.param_groups for p in g["params"]],
                                           MAX_NORM)
            return super().step(closure)
    return Clipped


def clipped_train_step(tokens, targets, model, opt):
    loss = model(tokens, targets)
    loss.backward()
    torch.nn.utils.clip_grad_norm_(model.parameters(), MAX_NORM)
    opt.step()
    opt.zero_grad(True)
    return loss


@pytest.mark.parametrize("kind", ["sgd", "adamw"])
@pytest.mark.parametrize("dtype,cuda_graph", [(torch.float32, False), (torch.float32, True),
                                              (torch.bfloat16, False), (torch.bfloat16, True)])
def test_small_llama_trains_like_vanilla_with_clipping(rt, kind, dtype, cuda_graph):
    """As tests/test_gpu_rope.py, with clip_grad_norm_ active (the total norm is above MAX_NORM):
    losses and every parameter / optimizer state against vanilla fp32 PyTorch."""
    from easydist_b200 import clip
    from easydist_b200.api import easydist_compile
    from easydist_b200.workloads import Llama, LlamaConfig, synthetic_tokens
    from tools import parity as P
    cfg = LlamaConfig(n_layer=2, n_head=4, n_embd=256, ffn=688, vocab_size=512, block_size=64)
    make = lambda: Llama(cfg)
    torch.manual_seed(0)
    model = make().to(device="cuda", dtype=dtype)
    n_params = len(list(model.parameters()))
    state = {k: v.detach().clone() for k, v in model.state_dict().items()}
    if kind == "sgd":
        mk = lambda cls: (lambda ps: cls(ps, lr=1e-2, momentum=0.9, foreach=True))
        base = torch.optim.SGD
    else:
        # Adam normalises every element's update, so where v is at noise level the update differs by
        # O(lr) for any difference in summation order: lr 1e-4 keeps that inside atol 1e-5
        mk = lambda cls: (lambda ps: cls(ps, lr=1e-4, weight_decay=0.05, fused=True))
        base = torch.optim.AdamW
    opt = mk(base)(model.parameters())
    step = easydist_compile(clipped_train_step, parallel_mode="ddp", tracing_mode="fake",
                            cuda_graph=cuda_graph)
    calls = 4
    clip.reset_stats()
    batches = [synthetic_tokens(cfg, 4, 64, seed=1000 * b) for b in range(calls)]
    losses = [float(step(tok.cuda(), tgt.cuda(), model, opt)) for tok, tgt in batches]
    info = step.compiled_func.info
    assert info["clip_nodes"] == (n_params, n_params), info
    sched = ([0, 0] if cuda_graph else [0]) + list(range(1, calls))
    steps = [[batches[b]] for b in sched]
    mk_ref = mk(_clipped(base))
    ref_l, ref_p, ref_s = P.vanilla_run(make, state, steps, mk_ref, torch.float32, "cuda")
    idx = [1 if cuda_graph else 0] + list(range(2 if cuda_graph else 1, len(sched)))
    rtol = 1e-4 if dtype == torch.float32 else 3e-2
    for got, i in zip(losses, idx):
        assert abs(got - ref_l[i][0]) <= rtol * abs(ref_l[i][0]), (losses, ref_l)
    got_p, got_s = P.compiled_state(step.compiled_func, ref_p, ref_s, 1)
    if dtype == torch.float32:
        res = P.compare(got_p, got_s, ref_p, ref_s, low_precision=False)
        assert res["assert_close_violation"] <= 1.0, res
    else:
        _, van_p, van_s = P.vanilla_run(make, state, steps, mk_ref, torch.bfloat16, "cuda")
        van = P.compare({k: v.bfloat16() for k, v in van_p.items()},
                        {k: {kk: vv.bfloat16() for kk, vv in st.items()} for k, st in van_s.items()},
                        ref_p, ref_s, low_precision=True)
        res = P.compare(got_p, got_s, ref_p, ref_s, low_precision=True)
        assert res["state_rel_l2"] <= max(2e-2, 2.0 * van["state_rel_l2"]), (res, van)
        assert res["param_max_ulp"] <= max(2.0, 2.0 * van["param_max_ulp"]), (res, van)
    st = clip.stats()
    assert st["aten_sumsq"] == 0 and st["edb_sumsq"] > 0, st
    assert st["aten_scale"] == 0 and (st["edb_scale"] > 0) == (kind == "adamw"), st


def test_zero3_with_clipping_on_two_gpus():
    """torchrun on 2 GPUs: the zero3 step of a small Llama with clipping against vanilla fp32, and the
    parameters bit-identical across the ranks (tests/clip_zero3_worker.py)."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from tests._procs import run_torchrun
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    rc, out, err = run_torchrun(os.path.join(root, "tests", "clip_zero3_worker.py"), 2, env, 900,
                                root, sys.executable)
    assert rc == 0 and "CLIP_ZERO3_OK" in out, (out[-3000:], err[-3000:])
