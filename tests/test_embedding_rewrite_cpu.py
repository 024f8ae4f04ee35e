"""lowering.fuse_embedding on the traced GPT-2 and Llama steps: what is matched, what is left alone,
and that the rewritten graph computes exactly what the unrewritten one does.  On CPU the embed ops
run the ATen ops they replace, op for op, so the steps are bit-identical.  The in-place fold of the
tied gradient needs the LM-head weight gradient to come from gemm.mm, so these tests retarget the
graph's aten.mm nodes to gemm.mm (which runs aten.mm off the GPU) as dispatch_compute does for bf16.
The kernels themselves are checked by tests/test_gpu_embedding.py."""
import collections
import os

import pytest
import torch
import torch.distributed as dist

from easydist_b200 import api, embed, gemm, lowering, workloads
from easydist_b200.device_mesh import set_device_mesh
from tests import gloo_ops
from tests._procs import run_world

aten = torch.ops.aten
GONE = (aten.embedding.default, aten.embedding_dense_backward.default)


def _counts(gm):
    return collections.Counter(n.target for n in gm.graph.nodes if n.op == "call_function")


def _model(name, dtype):
    torch.manual_seed(0)
    if name.startswith("gpt2"):
        cfg = workloads.GPT2_CONFIGS[name]
        return workloads.GPT2(cfg).to(dtype), cfg
    cfg = workloads.LLAMA_CONFIGS[name]
    return workloads.Llama(cfg).to(dtype), cfg


def _compiled(name, dtype, mode="ddp"):
    set_device_mesh([0], ["dp"], rank=0)
    model, cfg = _model(name, dtype)
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, foreach=True)
    tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, 0)
    c = api._compile_dp(workloads.gpt2_train_step, mode, "fake", (tok, tgt, model, opt), {},
                        ops=gloo_ops, native=False)
    return c, model, opt, cfg


def _native_mm(gm):
    for nd in gm.graph.nodes:
        if nd.op == "call_function" and nd.target == aten.mm.default:
            nd.target = gemm.mm
    gm.recompile()


WANT = {"gpt2-tiny": (1, 2), "llama-tiny": (1, 1)}


@pytest.mark.parametrize("name", ["gpt2-tiny", "llama-tiny"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_rewritten_step_is_bit_identical(name, dtype):
    c, model, opt, cfg = _compiled(name, dtype)
    plain, pmodel, popt, _ = _compiled(name, dtype)
    gm = c.graph
    _native_mm(gm)
    n_add = _counts(gm)[aten.add.Tensor]
    assert lowering.fuse_embedding(gm) == WANT[name]
    gm.graph.lint()
    after = _counts(gm)
    assert not [t for t in GONE if after[t]]
    if name == "gpt2-tiny":  # wte + wpe, and the tied add, are gone
        assert after[embed.embedding_bwd_acc_] == 1 and after[embed.embedding_bwd] == 1
        assert n_add - after[aten.add.Tensor] == 2
        fwd = next(n for n in gm.graph.nodes if n.target is embed.embedding_fwd)
        assert len(fwd.args) == 4
    assert lowering.fuse_embedding(gm) == (0, 0)
    embed.reset_stats()
    for i in range(3):
        tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, i)
        assert torch.equal(c(tok, tgt, model, opt), plain(tok, tgt, pmodel, popt))
    (p, _, st), (pp, _, pst) = c.get_state(), plain.get_state()
    for k in pp:
        assert torch.equal(p[k], pp[k]), k
        for kk, v in pst[k].items():
            assert torch.equal(st[k][kk], v), (k, kk)
    assert embed.stats()["aten_embed"] == 3 * sum(WANT[name])


@pytest.mark.parametrize("name", ["gpt2-tiny", "llama-tiny"])
@pytest.mark.parametrize("mode", ["ddp", "zero3"])
def test_dispatch_leaves_no_aten_embedding(name, mode, monkeypatch):
    """The bf16 graphs dispatch_compute lowers at world 1 (zero3 is what bench.py compiles)."""
    for env, want in (("0", (0, 0)), ("1", WANT[name])):
        monkeypatch.setenv("EDB_NATIVE_EMBED", env)
        c, *_ = _compiled(name, torch.bfloat16, mode)
        counts = {}
        lowering.dispatch_compute(c.graph, counts)
        after = _counts(c.graph)
        assert counts["embed"] == want
        if env == "1":
            assert not [t for t in GONE if after[t]]
            assert after[embed.embedding_bwd_acc_] == (name == "gpt2-tiny")
        else:
            assert after[aten.embedding.default] > 0


def test_extra_reader_of_the_lm_gradient_blocks_the_fold():
    c, model, opt, cfg = _compiled("gpt2-tiny", torch.bfloat16)
    plain, pmodel, popt, _ = _compiled("gpt2-tiny", torch.bfloat16)
    gm = c.graph
    _native_mm(gm)
    bwd = [n for n in gm.graph.nodes if n.target == aten.embedding_dense_backward.default]
    add = next(iter(u for b in bwd for u in b.users if u.target == aten.add.Tensor))
    x = next(a for a in add.args if a not in bwd)
    with gm.graph.inserting_after(x):
        gm.graph.call_function(aten.neg.default, (x,))
    assert lowering.fuse_embedding(gm) == (1, 2)
    after = _counts(gm)
    assert after[embed.embedding_bwd_acc_] == 0 and after[embed.embedding_bwd] == 2
    gm.recompile()
    for i in range(2):
        tok, tgt = workloads.synthetic_tokens(cfg, 2, 32, i)
        assert torch.equal(c(tok, tgt, model, opt), plain(tok, tgt, pmodel, popt))


def test_scale_grad_by_freq_is_left_alone():
    c, *_ = _compiled("llama-tiny", torch.bfloat16)
    gm = c.graph
    bwd = next(n for n in gm.graph.nodes if n.target == aten.embedding_dense_backward.default)
    bwd.args = tuple(bwd.args[:4]) + (True,)
    assert lowering.fuse_embedding(gm) == (1, 0)
    assert _counts(gm)[aten.embedding_dense_backward.default] == 1


def _dp_worker(rank, world, port, mode, q):
    os.environ["OMP_NUM_THREADS"] = "1"
    torch.set_num_threads(1)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    set_device_mesh(list(range(world)), ["dp"], rank=rank)
    cfg = workloads.GPT2_CONFIGS["gpt2-tiny"]
    torch.manual_seed(0)
    model, ref = workloads.GPT2(cfg), workloads.GPT2(cfg)
    ref.load_state_dict(model.state_dict())
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, foreach=True)
    ropt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9, foreach=True)
    g = torch.Generator().manual_seed(5)
    toks = [torch.randint(0, cfg.vocab_size, (world * 2, 33), generator=g) for _ in range(3)]
    sl = slice(rank * 2, (rank + 1) * 2)
    compiled = api._compile_dp(workloads.gpt2_train_step, mode, "fake",
                               (toks[0][sl, :-1].contiguous(), toks[0][sl, 1:].contiguous(), model, opt),
                               {}, ops=gloo_ops, native=False)
    _native_mm(compiled.graph)
    n = lowering.fuse_embedding(compiled.graph)
    left = [t for t in GONE if _counts(compiled.graph)[t]]
    ok, msg = n == (1, 2) and not left, f"embedding rewrites {n}, left {left}"
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
            p = torch.cat(parts)[:p_ref.numel()].view(p_ref.shape)
        if not torch.allclose(p, p_ref.detach(), rtol=1e-4, atol=1e-5):
            ok, msg = False, f"param {name} differs by {(p - p_ref).abs().max()}"
    if rank == 0:
        q.put((ok, msg))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("mode", ["ddp", "zero2", "zero3"])
def test_tiny_gpt2_dp_with_the_rewrite_matches_vanilla(mode):
    ok, msg = run_world(_dp_worker, 2, lambda r, port, q: (r, 2, port, mode, q), timeout=300)
    assert ok, msg
