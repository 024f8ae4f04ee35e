"""lowering.fuse_rope on the traced Llama step, in both RoPE forms: what is matched, what is left
alone, and that the rewritten graph computes exactly what the unrewritten one does.  On CPU rope.rope
runs the half-split ATen chain op for op, so the results are bit-identical only because both forms
and their backwards compute the same bits — which the first test pins down.  The kernel itself is
checked by tests/test_gpu_rope.py."""
import collections
import os

import pytest
import torch
import torch.distributed as dist

from easydist_b200 import api, lowering, rope, workloads
from easydist_b200.device_mesh import set_device_mesh
from tests import gloo_ops
from tests import rope_forms as RF
from tests._procs import run_world

aten = torch.ops.aten
GONE = (aten.cat.default, aten.sub.Tensor, aten.neg.default, aten.slice_backward.default)


def _counts(gm):
    return collections.Counter(n.target for n in gm.graph.nodes if n.op == "call_function")


def _compiled(dtype, form, seed=0):
    set_device_mesh([0], ["dp"], rank=0)
    cfg = workloads.LLAMA_CONFIGS["llama-tiny"]
    torch.manual_seed(seed)
    model = RF.llama(cfg, form).to(dtype)
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, foreach=True)
    tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, 0)
    c = api._compile_dp(workloads.gpt2_train_step, "ddp", "fake", (tok, tgt, model, opt), {},
                        ops=gloo_ops, native=False)
    return c, model, opt, cfg


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_both_forms_and_the_kernel_formula_are_bit_identical(dtype):
    """Forward and autograd gradient of the half-split and rotate_half forms, rope.formula (the
    kernel's arithmetic) and rope.rope (off the GPU: the ATen chain), on the transposed projection
    view, over 5 seeds."""
    B, H, T, hd = 2, 4, 64, 128
    cos, sin = RF.tables(T, hd, dtype)
    for seed in range(5):
        g = torch.Generator().manual_seed(seed)
        x = (torch.randn(B, T, H, hd, generator=g) * 3).to(dtype).transpose(1, 2)
        dy = torch.randn(B, H, T, hd, generator=g).to(dtype)
        outs = []
        for fn in (RF.rope_half_split, RF.rope_rotate_half):
            xx = x.detach().clone().requires_grad_(True)
            y = fn(xx, cos, sin)
            y.backward(dy)
            outs.append((y.detach(), xx.grad))
        (ya, ga), (yb, gb) = outs
        for want, inverse, src in ((ya, False, x), (ga, True, dy)):
            assert torch.equal(want, yb if not inverse else gb), (seed, inverse)
            assert torch.equal(want, rope.formula(src, cos, sin, inverse)), (seed, inverse)
            assert torch.equal(want, rope.rope(src, cos, sin, inverse)), (seed, inverse)
        # the layouts the rewrite asks for: the rotate_half forward's (x's) strides, and the
        # backward written as the [B, T, H, hd] tensor of transpose(1, 2).contiguous()
        y = rope.rope(x, cos, sin, False, stride=list(yb.stride()))
        assert torch.equal(y, ya) and y.stride() == yb.stride()
        t = rope.rope(dy, cos, sin, True, transposed=True)
        assert t.is_contiguous() and torch.equal(t, ga.transpose(1, 2).contiguous())


@pytest.mark.parametrize("form", RF.FORMS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_llama_step_rewritten_graph_is_bit_identical(dtype, form):
    c, model, opt, cfg = _compiled(dtype, form)
    plain, pmodel, popt, _ = _compiled(dtype, form)
    gm = c.graph
    before = _counts(gm)
    assert lowering.fuse_rope(gm) == (4, 4)
    gm.graph.lint()
    after = _counts(gm)
    assert not [t for t in GONE if after[t]], {t: after[t] for t in GONE}
    assert before[aten.clone.default] - after[aten.clone.default] == 4  # the backward clones
    assert after[rope.rope] == 8
    folded = [n for n in gm.graph.nodes if n.op == "call_function" and n.target is rope.rope
              and n.kwargs.get("transposed")]
    assert len(folded) == 4 and all(n.args[3] is True for n in folded)
    assert lowering.fuse_rope(gm) == (0, 0)
    rope.reset_stats()
    for i in range(3):
        tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, i)
        assert torch.equal(c(tok, tgt, model, opt), plain(tok, tgt, pmodel, popt))
    (p, _, st), (pp, _, pst) = c.get_state(), plain.get_state()
    for name in pp:
        assert torch.equal(p[name], pp[name]), name
        for k, v in pst[name].items():  # momentum buffers: the accumulated gradients
            assert torch.equal(st[name][k], v), (name, k)
    assert rope.stats()["aten_rope"] == 24


def test_switch_leaves_the_graph_alone(monkeypatch):
    for env, want in (("0", (0, 0)), ("1", (4, 4))):
        c, *_ = _compiled(torch.bfloat16, "half_split")
        before = _counts(c.graph)
        monkeypatch.setenv("EDB_NATIVE_ROPE", env)
        counts = {}
        lowering.dispatch_compute(c.graph, counts)
        after = _counts(c.graph)
        assert counts["rope"] == want
        assert (after[aten.cat.default], after[rope.rope]) == \
            ((before[aten.cat.default], 0) if env == "0" else (0, 8))


@pytest.mark.parametrize("form", RF.FORMS)
@pytest.mark.parametrize("mode", ["ddp", "zero3"])
def test_rewrite_matches_the_data_parallel_graphs(mode, form):
    from easydist_b200.compile import GraphIO, trace_train_step
    cfg = workloads.LLAMA_CONFIGS["llama-tiny"]
    torch.manual_seed(0)
    model = RF.llama(cfg, form).bfloat16()
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, foreach=True)
    tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, 0)
    params, buffers, states, gm, _, _ = trace_train_step(workloads.gpt2_train_step,
                                                         (tok, tgt, model, opt), {}, "fake")
    io = GraphIO(gm, params, buffers, states)
    if mode == "ddp":
        lowering.transform_ddp(gm, io, [0, 1], gloo_ops, bucket_numel=0)
    else:
        lowering.transform_fsdp(gm, io, [0, 1], 0, True, gloo_ops, bucket_numel=0)
    assert lowering.fuse_rope(gm) == (4, 4)
    gm.graph.lint()
    after = _counts(gm)
    assert not [t for t in GONE if after[t]]


def _first(gm, target, k=0):
    return [n for n in gm.graph.nodes if n.op == "call_function" and n.target == target][k]


def test_chain_with_an_extra_reader_is_left_alone():
    c, model, opt, cfg = _compiled(torch.bfloat16, "half_split")
    gm = c.graph
    sub = _first(gm, aten.sub.Tensor)
    with gm.graph.inserting_after(sub):
        gm.graph.call_function(aten.neg.default, (sub,))
    assert lowering.fuse_rope(gm) == (3, 4)
    assert _counts(gm)[aten.sub.Tensor] == 1


def test_fp32_tables_with_bf16_x_are_left_alone():
    """Tables of another dtype mean type promotion: the products are not rounded to x's dtype."""
    c, model, opt, cfg = _compiled(torch.bfloat16, "promoted_table")
    assert lowering.fuse_rope(c.graph) == (0, 0)
    assert _counts(c.graph)[aten.cat.default] == 4


@pytest.mark.parametrize("form", RF.FORMS)
def test_backward_without_the_clone_is_rewritten_without_the_fold(form):
    """The transpose behind the first backward result gets a second reader: that result is written
    in its own [B, H, T, hd] layout and the transpose and clone stay."""
    c, model, opt, cfg = _compiled(torch.bfloat16, form)
    plain, pmodel, popt, _ = _compiled(torch.bfloat16, form)
    gm = c.graph
    clone = next(n for n in gm.graph.nodes if n.op == "call_function" and n.target == aten.clone.default
                 and n.kwargs.get("memory_format") == torch.contiguous_format
                 and n.args[0].target == aten.transpose.int
                 and n.args[0].args[0].target == aten.add.Tensor)
    tr = clone.args[0]
    with gm.graph.inserting_after(tr):
        gm.graph.call_function(aten.neg.default, (tr,))
    n_clones = _counts(gm)[aten.clone.default]
    assert lowering.fuse_rope(gm) == (4, 4)
    assert n_clones - _counts(gm)[aten.clone.default] == 3
    src = tr.args[0]
    assert src.target is rope.rope and src.args[3] is True and "transposed" not in src.kwargs
    assert src.kwargs["stride"] == list(src.meta["val"].stride())
    for i in range(2):
        tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, i)
        assert torch.equal(c(tok, tgt, model, opt), plain(tok, tgt, pmodel, popt))


def _dp_worker(rank, world, port, mode, form, q):
    os.environ["OMP_NUM_THREADS"] = "1"
    torch.set_num_threads(1)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    set_device_mesh(list(range(world)), ["dp"], rank=rank)
    cfg = workloads.LLAMA_CONFIGS["llama-tiny"]
    torch.manual_seed(0)
    model, ref = RF.llama(cfg, form), RF.llama(cfg, form)
    ref.load_state_dict(model.state_dict())
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, foreach=True)
    ropt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9, foreach=True)
    g = torch.Generator().manual_seed(5)
    toks = [torch.randint(0, cfg.vocab_size, (world * 2, 33), generator=g) for _ in range(3)]
    sl = slice(rank * 2, (rank + 1) * 2)
    compiled = api._compile_dp(workloads.gpt2_train_step, mode, "fake",
                               (toks[0][sl, :-1].contiguous(), toks[0][sl, 1:].contiguous(), model, opt),
                               {}, ops=gloo_ops, native=False)
    n = lowering.fuse_rope(compiled.graph)
    ok, msg = n == (4, 4), f"rope rewrites {n}"
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


@pytest.mark.parametrize("form", RF.FORMS)
@pytest.mark.parametrize("mode", ["ddp", "zero3"])
def test_tiny_llama_dp_with_the_rewrite_matches_vanilla(mode, form):
    ok, msg = run_world(_dp_worker, 2, lambda r, port, q: (r, 2, port, mode, form, q), timeout=300)
    assert ok, msg
