"""lowering.fuse_rms_norm / fuse_swiglu on the traced Llama step: what is matched, what is left
alone, and that the rewritten graph computes exactly what the unrewritten one does.  On CPU the
norm.rms_norm_* / act.swiglu_* callables run their ATen restatement of the replaced chain, so the
results are bit-identical; the kernels themselves are checked by tests/test_gpu_rms_swiglu.py."""
import operator
import os

import pytest
import torch
import torch.distributed as dist

from easydist_b200 import act, api, lowering, norm, workloads
from easydist_b200.device_mesh import set_device_mesh
from tests import gloo_ops
from tests._procs import run_world

aten = torch.ops.aten
GONE = (aten.rsqrt.default, aten.silu.default, aten.silu_backward.default)


def _targets(gm):
    return [n.target for n in gm.graph.nodes if n.op == "call_function"]


def _compiled(dtype, seed=0):
    set_device_mesh([0], ["dp"], rank=0)
    cfg = workloads.LLAMA_CONFIGS["llama-tiny"]
    torch.manual_seed(seed)
    model = workloads.Llama(cfg).to(dtype)
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, foreach=True)
    tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, 0)
    c = api._compile_dp(workloads.gpt2_train_step, "ddp", "fake", (tok, tgt, model, opt), {},
                        ops=gloo_ops, native=False)
    return c, model, opt, cfg


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_llama_step_rewritten_graph_is_bit_identical(dtype):
    c, model, opt, cfg = _compiled(dtype)
    plain, pmodel, popt, _ = _compiled(dtype)
    gm = c.graph
    before = _targets(gm)
    assert before.count(aten.rsqrt.default) == 5 and before.count(aten.silu.default) == 2
    assert lowering.fuse_rms_norm(gm) == (5, 5)
    assert lowering.fuse_swiglu(gm) == (2, 2)
    gm.graph.lint()
    after = _targets(gm)
    assert not [t for t in GONE if t in after]
    assert after.count(norm.rms_norm_fwd) == 5 and after.count(norm.rms_norm_bwd) == 5
    assert after.count(act.swiglu_fwd) == 2 and after.count(act.swiglu_bwd) == 2
    # the norms of the blocks fold the running residual gradient; the first one (final norm, whose
    # input has no other gradient path) has none
    bwd = [n for n in gm.graph.nodes if n.op == "call_function" and n.target is norm.rms_norm_bwd]
    assert sum("_add" in n.kwargs for n in bwd) == 4
    if dtype == torch.bfloat16:  # the fp32 copies of x, rstd^3, the pieces' casts ... are gone
        assert len(after) < len(before) - 100
    assert lowering.fuse_rms_norm(gm) == (0, 0) and lowering.fuse_swiglu(gm) == (0, 0)
    norm.reset_stats()
    act.reset_stats()
    for i in range(3):
        tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, i)
        assert torch.equal(c(tok, tgt, model, opt), plain(tok, tgt, pmodel, popt))
    (p, _, st), (pp, _, pst) = c.get_state(), plain.get_state()
    for name in pp:
        assert torch.equal(p[name], pp[name]), name
        for k, v in pst[name].items():  # momentum buffers: the accumulated gradients
            assert torch.equal(st[name][k], v), (name, k)
    assert norm.stats()["aten_rms"] == 30 and act.stats()["aten_swiglu"] == 12


@pytest.mark.parametrize("mode", ["ddp", "zero3"])
def test_rewrites_match_the_data_parallel_graphs(mode):
    """After the ddp / zero3 transforms (zero3: every weight is a gathered view) all chains still
    match."""
    from easydist_b200.compile import GraphIO, trace_train_step
    cfg = workloads.LLAMA_CONFIGS["llama-tiny"]
    torch.manual_seed(0)
    model = workloads.Llama(cfg).bfloat16()
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, foreach=True)
    tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, 0)
    params, buffers, states, gm, _, _ = trace_train_step(workloads.gpt2_train_step,
                                                         (tok, tgt, model, opt), {}, "fake")
    io = GraphIO(gm, params, buffers, states)
    if mode == "ddp":
        lowering.transform_ddp(gm, io, [0, 1], gloo_ops, bucket_numel=0)
    else:
        lowering.transform_fsdp(gm, io, [0, 1], 0, True, gloo_ops, bucket_numel=0)
    assert lowering.fuse_rms_norm(gm) == (5, 5)
    assert lowering.fuse_swiglu(gm) == (2, 2)
    gm.graph.lint()
    assert not [t for t in GONE if t in _targets(gm)]


def _add_reader(gm, pick):
    """Give the node `pick` selects an extra (userless) reader."""
    nd = pick(gm)
    with gm.graph.inserting_after(nd):
        gm.graph.call_function(aten.neg.default, (nd,))


def _first(gm, target, k=0):
    return [n for n in gm.graph.nodes if n.op == "call_function" and n.target == target][k]


@pytest.mark.parametrize("case", ["normed_extra_user", "rstd_extra_user", "eps_dim_differs",
                                  "sum_dim_differs", "silu_third_user"])
def test_chains_with_extra_readers_or_other_shapes_are_left_alone(case):
    c, *_ = _compiled(torch.bfloat16)
    gm = c.graph
    if case == "normed_extra_user":  # the bf16 normed tensor: rsqrt -> mul(x.float(), rstd) -> _to_copy
        def normed(g):
            n32 = next(u for u in _first(g, aten.rsqrt.default).users if u.target == aten.mul.Tensor)
            return next(iter(n32.users))
        _add_reader(gm, normed)
    elif case == "rstd_extra_user":
        _add_reader(gm, lambda g: _first(g, aten.rsqrt.default, 2))
    elif case == "eps_dim_differs":  # the backward divides by another width than the forward averages
        dv = _first(gm, aten.div.Scalar, 1)
        dv.args = (dv.args[0], dv.args[1] + 1)
    elif case == "sum_dim_differs":  # the backward's sum(g*x) over another dim than the forward mean
        s = [n for n in gm.graph.nodes if n.op == "call_function" and n.target == aten.sum.dim_IntList
             and n.args[1] == [2]][0]
        s.args = (s.args[0], [1], True)
    if case == "silu_third_user":
        _add_reader(gm, lambda g: _first(g, aten.silu.default))
        assert lowering.fuse_swiglu(gm) == (1, 1)
        assert _targets(gm).count(aten.silu.default) == 1
    else:
        assert lowering.fuse_rms_norm(gm) == (4, 4)
        assert _targets(gm).count(aten.rsqrt.default) == 1


def test_fused_rms_norm_nodes_are_retargeted_with_the_gradient_add_folded():
    """aten._fused_rms_norm(_backward) (F.rms_norm / nn.RMSNorm on CUDA) -> norm.fused_rms_norm(_backward),
    add(dx, g) -> _add=g."""
    # built by hand: on CPU tensors F.rms_norm decomposes before it reaches these ops
    g = torch.fx.Graph()
    x, w, dy, res = (g.placeholder(n) for n in ("x", "w", "dy", "res"))
    fw = g.call_function(aten._fused_rms_norm.default, (x, [64], w, 1e-5))
    y, r = (g.call_function(operator.getitem, (fw, i)) for i in range(2))
    bw = g.call_function(aten._fused_rms_norm_backward.default, (dy, x, [64], r, w, [True, True]))
    dx, dw = (g.call_function(operator.getitem, (bw, i)) for i in range(2))
    out = g.call_function(aten.add.Tensor, (dx, res))
    g.output((y, out, dw))
    for nd in (dx, res, out):
        nd.meta["val"] = torch.empty(4, 8, 64)
    gm = torch.fx.GraphModule(torch.nn.Module(), g)
    assert lowering.fuse_rms_norm(gm) == (1, 1)
    gm.graph.lint()
    after = _targets(gm)
    assert norm.fused_rms_norm in after and norm.fused_rms_norm_backward in after
    assert aten.add.Tensor not in after
    bw = _first(gm, norm.fused_rms_norm_backward)
    assert bw.kwargs["_add"].op == "placeholder"


def _dp_worker(rank, world, port, mode, q):
    os.environ["OMP_NUM_THREADS"] = "1"
    torch.set_num_threads(1)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    set_device_mesh(list(range(world)), ["dp"], rank=rank)
    cfg = workloads.LLAMA_CONFIGS["llama-tiny"]
    torch.manual_seed(0)
    model, ref = workloads.Llama(cfg), workloads.Llama(cfg)
    ref.load_state_dict(model.state_dict())
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, foreach=True)
    ropt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9, foreach=True)
    g = torch.Generator().manual_seed(5)
    toks = [torch.randint(0, cfg.vocab_size, (world * 2, 33), generator=g) for _ in range(3)]
    sl = slice(rank * 2, (rank + 1) * 2)
    compiled = api._compile_dp(workloads.gpt2_train_step, mode, "fake",
                               (toks[0][sl, :-1].contiguous(), toks[0][sl, 1:].contiguous(), model, opt),
                               {}, ops=gloo_ops, native=False)
    n_rms, n_sw = lowering.fuse_rms_norm(compiled.graph), lowering.fuse_swiglu(compiled.graph)
    ok, msg = (n_rms == (5, 5) and n_sw == (2, 2)), f"rewrites: rms {n_rms} swiglu {n_sw}"
    for t in toks:
        loss = compiled(t[sl, :-1].contiguous(), t[sl, 1:].contiguous(), model, opt)
        rloss = workloads.gpt2_train_step(t[:, :-1].contiguous(), t[:, 1:].contiguous(), ref, ropt)
        la = loss.detach().clone()
        dist.all_reduce(la)
        la /= world
        if not torch.allclose(la, rloss.detach(), rtol=1e-4, atol=1e-5):
            ok, msg = False, f"loss {la} vs {rloss}"
    params = compiled.named_parameters()
    for name, p_ref in ref.named_parameters():
        p = params[name]
        if p.shape != p_ref.shape:
            parts = [torch.empty_like(p) for _ in range(world)]
            dist.all_gather(parts, p.contiguous())
            p = torch.cat(parts).view(p_ref.shape)
        if not torch.allclose(p, p_ref.detach(), rtol=1e-4, atol=1e-5):
            ok, msg = False, f"param {name} differs by {(p - p_ref).abs().max()}"
    if rank == 0:
        q.put((ok, msg))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("mode", ["ddp", "zero3"])
def test_tiny_llama_dp_with_rewrites_matches_vanilla(mode):
    ok, msg = run_world(_dp_worker, 2, lambda r, port, q: (r, 2, port, mode, q), timeout=300)
    assert ok, msg
