"""Gradient-norm clipping (`torch.nn.utils.clip_grad_norm_`, norm_type 2) in compiled steps:
lowering.fuse_grad_clip at world 1, and the zero2 / zero3 transforms, which take the norms of the
gradient shards.  On CPU the clip ops run the replaced ATen ops op for op, so the rewritten step is
bit-identical to the unrewritten one; the kernels are checked by tests/test_gpu_clip.py."""
import collections
import os

import pytest
import torch
import torch.distributed as dist

from easydist_b200 import api, clip, lowering, optim, workloads
from easydist_b200.device_mesh import set_device_mesh
from tests import gloo_ops
from tests._procs import run_world

aten = torch.ops.aten
ACTIVE, INACTIVE = 0.02, 1e4  # max_norm: coefficient < 1 / clamped to 1


def clipped_step(max_norm):
    def step(tokens, targets, model, opt):
        loss = model(tokens, targets)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm)
        opt.step()
        opt.zero_grad(True)
        return loss
    return step


def _model(name, dtype):
    torch.manual_seed(0)
    if name in workloads.LLAMA_CONFIGS:
        cfg = workloads.LLAMA_CONFIGS[name]
        return cfg, workloads.Llama(cfg).to(dtype)
    cfg = workloads.GPT2_CONFIGS[name]
    return cfg, workloads.GPT2(cfg).to(dtype)


def _make_opt(kind, params):
    if kind == "sgd":
        return torch.optim.SGD(params, lr=0.05, momentum=0.9, foreach=True)
    return torch.optim.AdamW(params, lr=1e-3, weight_decay=0.05, fused=True)


def _compiled(name, dtype, max_norm=ACTIVE, kind="sgd"):
    set_device_mesh([0], ["dp"], rank=0)
    cfg, model = _model(name, dtype)
    opt = _make_opt(kind, model.parameters())
    tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, 0)
    c = api._compile_dp(clipped_step(max_norm), "ddp", "fake", (tok, tgt, model, opt), {},
                        ops=gloo_ops, native=False)
    return c, model, opt, cfg


def _counts(gm):
    return collections.Counter(n.target for n in gm.graph.nodes if n.op == "call_function")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("name", ["llama-tiny", "gpt2-tiny"])
def test_world1_rewrite_is_bit_identical(name, dtype):
    c, model, opt, cfg = _compiled(name, dtype)
    plain, pmodel, popt, _ = _compiled(name, dtype)
    n_params = len(list(model.parameters()))
    gm = c.graph
    assert lowering.fuse_optimizer_updates(gm) == 1
    assert lowering.fuse_optimizer_updates(plain.graph) == 1
    assert lowering.fuse_grad_clip(gm) == (n_params, n_params)
    gm.graph.lint()
    after = _counts(gm)
    assert after[aten.linalg_vector_norm.default] == 1 and after[aten.mul_.Tensor] == 0, after
    assert after[clip.grad_norms] == 1 and after[aten.stack.default] == 0
    sgd = next(n for n in gm.graph.nodes if n.op == "call_function" and n.target is optim.sgd_momentum_)
    assert sgd.kwargs["grad_scale"].target == aten.clamp.default
    assert lowering.fuse_grad_clip(gm) == (0, 0)
    clip.reset_stats()
    for i in range(3):
        tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, i)
        assert torch.equal(c(tok, tgt, model, opt), plain(tok, tgt, pmodel, popt))
    (p, _, st), (pp, _, pst) = c.get_state(), plain.get_state()
    for name_ in pp:
        assert torch.equal(p[name_], pp[name_]), name_
        for k, v in pst[name_].items():
            assert torch.equal(st[name_][k], v), (name_, k)
    assert clip.stats()["aten_sumsq"] == 3


def test_unfused_optimizer_gets_one_scale_node():
    """AdamW(fused=True) is not fused here: the T mul_ become one clip.scale_ in front of it."""
    c, model, opt, cfg = _compiled("llama-tiny", torch.bfloat16, kind="adamw")
    plain, pmodel, popt, _ = _compiled("llama-tiny", torch.bfloat16, kind="adamw")
    n_params = len(list(model.parameters()))
    assert lowering.fuse_grad_clip(c.graph) == (n_params, n_params)
    assert _counts(c.graph)[clip.scale_] == 1
    for i in range(3):
        tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, i)
        assert torch.equal(c(tok, tgt, model, opt), plain(tok, tgt, pmodel, popt))
    for name_, v in plain.named_parameters().items():
        assert torch.equal(c.named_parameters()[name_], v), name_


def test_extra_reader_of_a_gradient_blocks_the_fold():
    """A node behind the mul_ reads the gradient: folding the scale into the SGD node would leave that
    reader with the unscaled values, so the mul_ nodes become a scale_ node (in place) instead."""
    c, model, opt, cfg = _compiled("llama-tiny", torch.bfloat16)
    gm = c.graph
    lowering.fuse_optimizer_updates(gm)
    mul = next(n for n in gm.graph.nodes if n.op == "call_function" and n.target == aten.mul_.Tensor)
    g = mul.args[0]
    sgd = next(n for n in gm.graph.nodes if n.op == "call_function" and n.target is optim.sgd_momentum_)
    with gm.graph.inserting_after(sgd):
        gm.graph.call_function(aten.neg.default, (g,))
    n_params = len(list(model.parameters()))
    assert lowering.fuse_grad_clip(gm) == (n_params, n_params)
    assert "grad_scale" not in sgd.kwargs and _counts(gm)[clip.scale_] == 1


def test_coefficient_of_another_dtype_is_left_alone():
    c, model, opt, cfg = _compiled("llama-tiny", torch.bfloat16)
    gm = c.graph
    clamp = next(n for n in gm.graph.nodes if n.op == "call_function" and n.target == aten.clamp.default)
    clamp.meta["val"] = clamp.meta["val"].float()
    n_params = len(list(model.parameters()))
    assert lowering.fuse_grad_clip(gm) == (n_params, 0)
    assert _counts(gm)[aten.mul_.Tensor] == n_params


def test_switch_leaves_the_graph_alone(monkeypatch):
    n = len(list(_model("llama-tiny", torch.float32)[1].parameters()))
    for env, want in (("0", (0, 0)), ("1", (n, n))):
        c, *_ = _compiled("llama-tiny", torch.bfloat16)
        monkeypatch.setenv("EDB_NATIVE_CLIP", env)
        counts = {}
        lowering.dispatch_compute(c.graph, counts)
        assert counts["clip"] == want


def _traced(step):
    from easydist_b200.compile import GraphIO, trace_train_step
    cfg, model = _model("llama-tiny", torch.bfloat16)
    opt = _make_opt("sgd", model.parameters())
    tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, 0)
    params, buffers, states, gm, _, _ = trace_train_step(step, (tok, tgt, model, opt), {}, "fake")
    return gm, GraphIO(gm, params, buffers, states)


@pytest.mark.parametrize("kwargs", [dict(norm_type=float("inf")), dict(error_if_nonfinite=True)])
def test_unsupported_forms_still_raise_in_zero3(kwargs):
    def step(tokens, targets, model, opt):
        loss = model(tokens, targets)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 1.0, **kwargs)
        opt.step()
        opt.zero_grad(True)
        return loss
    with pytest.raises(Exception) as e:
        gm, io = _traced(step)
        lowering.transform_fsdp(gm, io, [0, 1], 0, True, gloo_ops, bucket_numel=0)
    assert isinstance(e.value, (NotImplementedError, RuntimeError)), e.value


def test_zero3_graph_with_clipping_passes_the_epoch_protocol_check(monkeypatch):
    """The zero3 graph lowered as in test_prefetch_schedule_cpu._lowered_zero3_graph, with clipping:
    the all-reduce of the shards' sums of squares gets its static buffers and sits between the
    barrier in front of the optimizer and the end barrier."""
    monkeypatch.setenv("EDB_EPOCH", "1")
    from easydist_b200.api import _flat_inputs
    from easydist_b200.compile import GraphIO, trace_train_step
    from tests.test_dp_cpu import make_opt, train_step_clipped
    from tests.test_prefetch_schedule_cpu import Deep
    torch.manual_seed(0)
    n, me = 4, 1
    model = Deep(layers=2).bfloat16()
    opt = make_opt("sgd", model.parameters())
    x = torch.randn(64, 256).bfloat16()
    params, buffers, named_states, gm, module, o = trace_train_step(train_step_clipped,
                                                                   (x, model, opt), {}, "fake")
    io = GraphIO(gm, params, buffers, named_states)
    ranks = list(range(n))
    _, shard_info = lowering.transform_fsdp(gm, io, ranks, me, True, gloo_ops, bucket_numel=2048)
    with torch.no_grad():
        params = {k: v.detach() for k, v in params.items()}
        for ph, name in zip(io.param_ph, io.param_names):
            if ph.name in shard_info:
                params[name] = torch.chunk(params[name].flatten(), n)[me].contiguous()
        flat_states, spec = torch.utils._pytree.tree_flatten(named_states)
        for i, ph in enumerate(io.state_ph):
            if ph.name in shard_info and isinstance(flat_states[i], torch.Tensor):
                flat_states[i] = torch.chunk(flat_states[i].detach().flatten(), n)[me].contiguous()
        named_states = torch.utils._pytree.tree_unflatten(flat_states, spec)
        lowering.propagate_local_meta(gm, [t.detach() if isinstance(t, torch.Tensor) else t for t in
                                           _flat_inputs(params, buffers, named_states, (x, model, opt), {})])
    rt = gloo_ops.FakeSymmRuntime()
    lowering.fuse_collective_gemms(gm, io, rt, ranks, gloo_ops, my_index=me)
    lowering.reinplace_optimizer_updates(gm)
    lowering.assign_static_buffers(gm, rt, gloo_ops, push=True)
    lowering.ensure_end_barrier(gm, ranks, gloo_ops)
    counts = {}
    lowering.dispatch_compute(gm, counts)
    rep = lowering.verify_epoch_protocol(gm, gloo_ops, n)
    assert rep["ok"] and rep["barriers"] == 2, rep
    nodes = list(gm.graph.nodes)
    ar = [i for i, nd in enumerate(nodes) if nd.op == "call_function"
          and nd.target is gloo_ops.all_reduce_start and nd.args[1] == "sum"]
    assert len(ar) == 1 and "_buf" in nodes[ar[0]].kwargs and nodes[ar[0]].kwargs.get("_push") == 1
    barriers = [i for i, nd in enumerate(nodes) if nd.op == "call_function"
                and nd.target is gloo_ops.epoch_barrier]
    assert barriers[0] < ar[0] < barriers[1]
    # the four 2-D/bias parameters of 2048+ elements are sharded, the rest replicated
    assert counts["clip"][1] > 0


def _gather(t, full_shape, world):
    if tuple(t.shape) == tuple(full_shape):
        return t
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t.contiguous())
    return torch.cat(parts).view(full_shape)


def _run_case(rank, world, mode, kind, max_norm):
    """One clipped zero2 / zero3 run inside an initialised gloo job -> (ok, message, clip counts)."""
    set_device_mesh(list(range(world)), ["dp"], rank=rank)
    cfg, model = _model("llama-tiny", torch.float32)
    _, ref = _model("llama-tiny", torch.float32)
    opt, ropt = _make_opt(kind, model.parameters()), _make_opt(kind, ref.parameters())
    g = torch.Generator().manual_seed(5)
    toks = [torch.randint(0, cfg.vocab_size, (world * 2, 33), generator=g) for _ in range(3)]
    sl = slice(rank * 2, (rank + 1) * 2)
    # 4097: the norm weights and the 64x64 projections stay replicated (bucketed all-reduce), the
    # embedding, the MLP and the LM head are sharded
    compiled = api._compile_dp(clipped_step(max_norm), mode, "fake",
                               (toks[0][sl, :-1].contiguous(), toks[0][sl, 1:].contiguous(), model, opt),
                               {}, ops=gloo_ops, native=False, bucket_numel=4097)
    lowering.fuse_optimizer_updates(compiled.graph)
    n_clip = lowering.fuse_grad_clip(compiled.graph)
    ok, msg = True, ""
    for t in toks:
        loss = compiled(t[sl, :-1].contiguous(), t[sl, 1:].contiguous(), model, opt)
        rloss = ref(t[:, :-1].contiguous(), t[:, 1:].contiguous())
        rloss.backward()
        total = torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm)
        if (total > max_norm) != (max_norm == ACTIVE):
            ok, msg = False, f"clipping {'in' if max_norm == ACTIVE else ''}active: norm {total}"
        ropt.step()
        ropt.zero_grad(True)
        la = loss.detach().clone()
        dist.all_reduce(la)
        la /= world
        if not torch.allclose(la, rloss.detach(), rtol=1e-4, atol=1e-5):
            ok, msg = False, f"loss {la} vs {rloss}"
    params = compiled.named_parameters()
    states = compiled.get_state()[2]
    rstates = {n_: ropt.state[p] for n_, p in ref.named_parameters()}
    for name, p_ref in ref.named_parameters():
        p = params[name]
        full = _gather(p, p_ref.shape, world)
        if not torch.allclose(full, p_ref.detach(), rtol=1e-4, atol=1e-5):
            ok, msg = False, f"param {name} differs by {(full - p_ref).abs().max()}"
        # every rank holds the same bits: replicated parameters directly, sharded ones gathered
        peers = [torch.empty_like(full) for _ in range(world)]
        dist.all_gather(peers, full.contiguous())
        if not all(torch.equal(peers[0], x) for x in peers[1:]):
            ok, msg = False, f"param {name} differs across ranks"
        for k, v in rstates[name].items():
            if not isinstance(v, torch.Tensor) or v.dim() == 0:
                continue
            s = _gather(states[name][k], v.shape, world)
            if not torch.allclose(s, v, rtol=1e-4, atol=1e-5):
                ok, msg = False, f"state {name}.{k} differs by {(s - v).abs().max()}"
    return ok, msg, n_clip


def _batch_worker(rank, world, port, cases, q):
    """Every case in ONE gloo job (process start-up would otherwise dominate these tests)."""
    os.environ["OMP_NUM_THREADS"] = "1"
    torch.set_num_threads(1)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    results = {}
    for case in cases:
        try:
            results[case] = _run_case(rank, world, *case)
        except Exception as e:  # noqa: BLE001 — reported per case
            import traceback
            results[case] = (False, f"{type(e).__name__}: {e}\n{traceback.format_exc()[-1500:]}", None)
        dist.barrier()
    if rank == 0:
        q.put(results)
    dist.barrier()
    dist.destroy_process_group()


CASES = [(mode, kind, max_norm) for mode in ("zero2", "zero3") for kind in ("sgd", "adamw")
         for max_norm in (ACTIVE, INACTIVE)]


@pytest.fixture(scope="module")
def world2_results():
    return run_world(_batch_worker, 2, lambda r, port, q: (r, 2, port, CASES, q), timeout=600)


@pytest.mark.parametrize("max_norm", [ACTIVE, INACTIVE])
@pytest.mark.parametrize("kind", ["sgd", "adamw"])
@pytest.mark.parametrize("mode", ["zero2", "zero3"])
def test_zero_modes_with_clipping_match_vanilla(world2_results, mode, kind, max_norm):
    ok, msg, n_clip = world2_results[(mode, kind, max_norm)]
    assert ok, msg
    assert n_clip[0] == 0 and n_clip[1] > 0, n_clip  # norms already taken from the shards


def test_zero3_world4_with_clipping_matches_vanilla():
    case = ("zero3", "sgd", ACTIVE)
    res = run_world(_batch_worker, 4, lambda r, port, q: (r, 4, port, [case], q), timeout=300)
    ok, msg, n_clip = res[case]
    assert ok, msg
