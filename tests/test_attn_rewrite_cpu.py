"""lowering.fuse_attention on the traced GPT-2 and Llama steps and on hand-built graphs of ATen's
CUDA flash pair: what is matched, what is left alone, and that the rewritten graph computes exactly
what the unrewritten one does.  On CPU attn.attention_fwd / attention_bwd run the `_for_cpu` ops the
nodes called, so the results are bit-identical.  The kernels are checked by
tests/test_gpu_attention.py."""
import collections
import operator

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from easydist_b200 import api, attn, lowering, workloads
from easydist_b200.device_mesh import set_device_mesh
from tests import gloo_ops

aten = torch.ops.aten
FWD_CUDA, FWD_CPU, FWD_CUDNN = attn.FWD_OPS["flash"], attn.FWD_OPS["cpu"], attn.FWD_OPS["cudnn"]
BWD_CUDA, BWD_CPU, BWD_CUDNN = attn.BWD_OPS["flash"], attn.BWD_OPS["cpu"], attn.BWD_OPS["cudnn"]


def _counts(gm):
    return collections.Counter(n.target for n in gm.graph.nodes if n.op == "call_function")


def _model(name):
    if name == "gpt2":
        cfg = workloads.GPT2_CONFIGS["gpt2-tiny"]
        return cfg, workloads.GPT2(cfg)
    cfg = workloads.LLAMA_CONFIGS["llama-tiny"]
    return cfg, workloads.Llama(cfg)


def _compiled(name):
    set_device_mesh([0], ["dp"], rank=0)
    torch.manual_seed(0)
    cfg, model = _model(name)
    model = model.bfloat16()
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, foreach=True)
    tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, 0)
    c = api._compile_dp(workloads.gpt2_train_step, "ddp", "fake", (tok, tgt, model, opt), {},
                        ops=gloo_ops, native=False)
    return c, model, opt, cfg


@pytest.mark.parametrize("name", ["gpt2", "llama"])
def test_step_rewritten_graph_is_bit_identical(name):
    c, model, opt, cfg = _compiled(name)
    plain, pmodel, popt, _ = _compiled(name)
    gm = c.graph
    if name == "llama":
        assert lowering.fuse_rope(gm) == (4, 4)
        assert lowering.fuse_rope(plain.graph) == (4, 4)
    assert lowering.fuse_attention(gm) == (2, 2)
    gm.graph.lint()
    after = _counts(gm)
    assert not (after[FWD_CPU] or after[BWD_CPU])
    assert after[attn.attention_fwd] == 2 and after[attn.attention_bwd] == 2
    for nd in gm.graph.nodes:
        if nd.target is attn.attention_fwd:
            assert nd.args[3] is True and nd.args[4] is None
            assert nd.kwargs["out_stride"] == list(nd.meta["val"][0].stride())
            assert nd.kwargs["lse_stride"] == list(nd.meta["val"][1].stride())
        if nd.target is attn.attention_bwd:
            assert nd.kwargs["strides"] == [list(t.stride()) for t in nd.meta["val"]]
    assert lowering.fuse_attention(gm) == (0, 0)
    attn.reset_stats()
    for i in range(3):
        tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, i)
        assert torch.equal(c(tok, tgt, model, opt), plain(tok, tgt, pmodel, popt))
    (p, _, st), (pp, _, pst) = c.get_state(), plain.get_state()
    for k in pp:
        assert torch.equal(p[k], pp[k]), k
        for kk, v in pst[k].items():
            assert torch.equal(st[k][kk], v), (k, kk)
    assert attn.stats() == {"edb_attn_fwd": 0, "edb_attn_bwd": 0, "aten_attn_fwd": 6, "aten_attn_bwd": 6}


@pytest.mark.parametrize("name", ["gpt2", "llama"])
@pytest.mark.parametrize("mode", ["ddp", "zero3"])
def test_rewrite_matches_the_data_parallel_graphs(mode, name):
    from easydist_b200.compile import GraphIO, trace_train_step
    torch.manual_seed(0)
    cfg, model = _model(name)
    model = model.bfloat16()
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, foreach=True)
    tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, 0)
    params, buffers, states, gm, _, _ = trace_train_step(workloads.gpt2_train_step,
                                                         (tok, tgt, model, opt), {}, "fake")
    io = GraphIO(gm, params, buffers, states)
    if mode == "ddp":
        lowering.transform_ddp(gm, io, [0, 1], gloo_ops, bucket_numel=0)
    else:
        lowering.transform_fsdp(gm, io, [0, 1], 0, True, gloo_ops, bucket_numel=0)
    if name == "llama":
        lowering.fuse_rope(gm)
    assert lowering.fuse_attention(gm) == (2, 2)
    gm.graph.lint()
    after = _counts(gm)
    assert not (after[FWD_CPU] or after[BWD_CPU])


@pytest.fixture
def deterministic():
    """torch.use_deterministic_algorithms(True, warn_only=True) for the test, restored after."""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


@pytest.mark.parametrize("det,env,want", [(False, None, (0, 0)), (False, "1", (0, 0)), (True, None, (2, 2)),
                                          (True, "1", (2, 2)), (True, "0", (0, 0))])
def test_rewrite_runs_for_steps_compiled_under_deterministic_algorithms(request, monkeypatch, det, env,
                                                                         want):
    """dispatch_compute rewrites attention only when the step asks for deterministic algorithms
    (ATen's attention backwards are then either not repeatable or slower), unless
    EDB_NATIVE_ATTN=0 turns the rewrite off."""
    c, *_ = _compiled("gpt2")
    if env is None:
        monkeypatch.delenv("EDB_NATIVE_ATTN", raising=False)
    else:
        monkeypatch.setenv("EDB_NATIVE_ATTN", env)
    if det:
        request.getfixturevalue("deterministic")
    counts = {}
    lowering.dispatch_compute(c.graph, counts)
    assert counts["attn"] == want
    assert _counts(c.graph)[FWD_CPU] == (2 if want == (0, 0) else 0)


def test_entry_points_refuse_what_the_kernels_cannot_compute():
    """A non-positive or non-finite scale (the softmax shifts by the row maximum of the raw scores)
    and broadcast (stride-0) views are EDB_E_UNSUPPORTED before anything is read or launched."""
    from easydist_b200 import _lib
    lib = _lib.load()
    B, H, T, hd = 2, 3, 64, 64
    ok = [H * T * hd, T * hd, hd] * 4 + [H * T, T, 1]
    p = 1 << 20  # aligned, never dereferenced
    for scale, st in ((0.0, ok), (-0.125, ok), (float("inf"), ok), (float("nan"), ok),
                      (0.125, [0] + ok[1:]), (0.125, ok[:4] + [0] + ok[5:])):
        rc = lib.edb_attn_fwd(p, p, p, p, p, B, H, T, hd, _lib.i64_array(st), scale, 1, None)
        assert rc == _lib.EDB_E_UNSUPPORTED, (scale, st)
    bst = [H * T * hd, T * hd, hd] * 8 + [H * T, T, 1]
    for scale, st in ((0.0, bst), (0.125, bst[:6] + [0] + bst[7:])):
        rc = lib.edb_attn_bwd(p, p, p, p, p, p, p, p, p, p, B, H, T, hd, _lib.i64_array(st), scale, 1,
                              None)
        assert rc == _lib.EDB_E_UNSUPPORTED, (scale, st)


# ---- hand-built graphs: the CUDA flash pair, which CPU tracing cannot produce ------------------------

def _flash_graph(fwd_args=(0.0, True), fwd_kwargs=None, bwd=True, lse_reader=False, bwd_causal=True):
    """q, k, v -> ATen's CUDA flash forward (9 getitems) -> its backward, as AOT autograd traces
    them, with fake CUDA meta values; q, k, v are the c_attn split views."""
    B, H, T, hd = 2, 4, 33, 64
    mode = FakeTensorMode(allow_non_fake_inputs=True)
    with mode:
        qkv = torch.empty(B, T, 3 * H * hd, dtype=torch.bfloat16, device="cuda")
        views = [t.view(B, T, H, hd).transpose(1, 2) for t in qkv.split(H * hd, dim=2)]
        dout = torch.empty(B, H, T, hd, dtype=torch.bfloat16, device="cuda")
        fv = FWD_CUDA(*views, *fwd_args, **(fwd_kwargs or {}))
        bv = BWD_CUDA(dout, *views, fv[0], fv[1], fv[2], fv[3], fv[4], fv[5], 0.0, bwd_causal,
                      fv[6], fv[7])
    g = torch.fx.Graph()
    q, k, v, d = (g.placeholder(n) for n in ("q", "k", "v", "dout"))
    for nd, val in zip((q, k, v, d), (*views, dout)):
        nd.meta["val"] = val
    f = g.call_function(FWD_CUDA, (q, k, v, *fwd_args), dict(fwd_kwargs or {}))
    f.meta["val"] = fv
    gi = []
    for i in range(9):
        n = g.call_function(operator.getitem, (f, i))
        n.meta["val"] = fv[i]
        gi.append(n)
    outs = [gi[0]]
    if bwd:
        b = g.call_function(BWD_CUDA, (d, q, k, v, gi[0], gi[1], gi[2], gi[3], gi[4], gi[5], 0.0,
                                       bwd_causal, gi[6], gi[7]))
        b.meta["val"] = bv
        for i in range(3):
            n = g.call_function(operator.getitem, (b, i))
            n.meta["val"] = bv[i]
            outs.append(n)
    if lse_reader:
        outs.append(g.call_function(aten.exp.default, (gi[1],)))
    for n in gi[2:]:
        if not n.users:
            g.erase_node(n)
    g.output(tuple(outs))
    return torch.fx.GraphModule(torch.nn.Module(), g), fv, bv


def test_cuda_flash_pair_is_rewritten_with_its_argument_layout():
    gm, fv, bv = _flash_graph()
    assert lowering.fuse_attention(gm) == (1, 1)
    gm.graph.lint()
    nodes = {n.target: n for n in gm.graph.nodes if n.op == "call_function"}
    assert FWD_CUDA not in nodes and BWD_CUDA not in nodes
    f, b = nodes[attn.attention_fwd], nodes[attn.attention_bwd]
    q, k, v, d = [n for n in gm.graph.nodes if n.op == "placeholder"]
    assert f.args == (q, k, v, True, None)
    assert f.kwargs == {"out_stride": list(fv[0].stride()), "lse_stride": list(fv[1].stride()),
                        "aten_op": "flash"}
    assert len(f.meta["val"]) == 2 and f.meta["val"][0] is fv[0] and f.meta["val"][1] is fv[1]
    out, lse = sorted((u for u in f.users), key=lambda u: u.args[1])
    assert [u.args[1] for u in (out, lse)] == [0, 1]
    assert b.args == (d, q, k, v, out, lse, True, None)
    assert b.kwargs == {"strides": [list(t.stride()) for t in bv], "aten_op": "flash"}
    assert b.meta["val"] is bv


def test_a_forward_without_a_gradient_is_rewritten_alone():
    gm, fv, _ = _flash_graph(bwd=False)
    assert lowering.fuse_attention(gm) == (1, 0)
    assert _counts(gm)[attn.attention_fwd] == 1


@pytest.mark.parametrize("case", ["dropout", "debug_mask", "lse_reader", "other_causal", "mask"])
def test_unsupported_cases_are_left_alone(case):
    if case == "mask":
        c, *_ = _compiled("gpt2")
        fwd = next(n for n in c.graph.graph.nodes if n.target == FWD_CPU)
        fwd.kwargs = {"attn_mask": fwd.args[0]}
        assert lowering.fuse_attention(c.graph) == (1, 1)
        assert _counts(c.graph)[FWD_CPU] == 1
        return
    kw = {}
    if case == "dropout":
        kw["fwd_args"] = (0.1, True)
    elif case == "debug_mask":
        kw["fwd_args"] = (0.0, True, True)
    elif case == "lse_reader":
        kw["lse_reader"] = True
    else:
        kw["bwd_causal"] = False
    gm, _, _ = _flash_graph(**kw)
    before = _counts(gm)
    assert lowering.fuse_attention(gm) == (0, 0)
    assert _counts(gm) == before


def test_cudnn_pair_is_rewritten_with_its_argument_layout():
    """The pair SDPA traces to on the H100: cuDNN's forward (attn_bias None, compute_log_sumexp) with
    its [B, H, T, 1] logsumexp, and the backward reading the philox getitems."""
    B, H, T, hd = 2, 4, 33, 64
    with FakeTensorMode(allow_non_fake_inputs=True):
        qkv = torch.empty(B, T, 3 * H * hd, dtype=torch.bfloat16, device="cuda")
        views = [t.view(B, T, H, hd).transpose(1, 2) for t in qkv.split(H * hd, dim=2)]
        dout = torch.empty(B, H, T, hd, dtype=torch.bfloat16, device="cuda")
        fv = FWD_CUDNN(*views, None, True, 0.0, True)
        bv = BWD_CUDNN(dout, *views, fv[0], fv[1], fv[6], fv[7], None, None, None, T, T, 0.0, True)
    g = torch.fx.Graph()
    q, k, v, d = (g.placeholder(n) for n in ("q", "k", "v", "dout"))
    f = g.call_function(FWD_CUDNN, (q, k, v, None, True, 0.0, True))
    f.meta["val"] = fv
    gi = {}
    for i in (0, 1, 6, 7):
        gi[i] = g.call_function(operator.getitem, (f, i))
        gi[i].meta["val"] = fv[i]
    b = g.call_function(BWD_CUDNN, (d, q, k, v, gi[0], gi[1], gi[6], gi[7], None, None, None, T, T, 0.0,
                                    True))
    b.meta["val"] = bv
    outs = [gi[0]] + [g.call_function(operator.getitem, (b, i)) for i in range(3)]
    g.output(tuple(outs))
    gm = torch.fx.GraphModule(torch.nn.Module(), g)
    assert lowering.fuse_attention(gm) == (1, 1)
    gm.graph.lint()
    assert not (_counts(gm)[FWD_CUDNN] or _counts(gm)[BWD_CUDNN])
    assert f.target is attn.attention_fwd and f.args == (q, k, v, True, None)
    assert f.kwargs == {"out_stride": list(fv[0].stride()), "lse_stride": list(fv[1].stride()),
                        "aten_op": "cudnn"}
    assert tuple(fv[1].shape) == (B, H, T, 1)
    assert b.target is attn.attention_bwd and b.args == (d, q, k, v, gi[0], gi[1], True, None)
    assert b.kwargs == {"strides": [list(t.stride()) for t in bv], "aten_op": "cudnn"}
    assert sorted(u.args[1] for u in f.users) == [0, 1]
