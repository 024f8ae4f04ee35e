"""Auto-SPMD with a RECORDED plan: graph + plan solved by the unmodified reference (annotation,
MetaIR, AutoFlow ILP) in the CPU container and stored as tests/golden/auto_foo_mesh*.json by
tests/ref/auto_worker.py.  Here — with no reference in sight — the bundle is lowered by
easydist_b200.lowering.sharding_transform and executed over gloo; results must match vanilla
PyTorch (the reference's comparator, rtol 1e-4 / atol 1e-5).  The same bundles are executed on
real GPUs by tests/mgpu_worker.py."""
import os
import sys

import pytest
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests._procs import run_world  # noqa: E402
GOLDEN = os.path.join(ROOT, "tests", "golden")


class Foo(torch.nn.Module):
    def __init__(self, d=64):
        super().__init__()
        self.norm = torch.nn.LayerNorm(d)
        self.linear = torch.nn.Linear(d, d)

    def forward(self, x):
        return self.linear(self.norm(x)).relu()


def train_step(input, model, opt):
    out = model(input)
    loss = out.mean()
    loss.backward()
    opt.step()
    opt.zero_grad()
    return out


def run_bundle(rank, world, mesh_shape, ops, native, device, planner="GREEDY"):
    """Shared by the CPU test and the GPU worker.  Returns (ok, message, comm histogram).
    `planner`: the reshard planner the lowering uses (the solved plan does not depend on it)."""
    import numpy as np
    from easydist_b200 import api
    from easydist_b200.device_mesh import set_device_mesh
    names = [f"spmd{i}" for i in range(len(mesh_shape))]
    set_device_mesh(np.arange(world).reshape(mesh_shape), names, rank=rank)
    tag = "x".join(str(v) for v in mesh_shape)
    bundle = open(os.path.join(GOLDEN, f"auto_foo_mesh{tag}.json")).read()
    torch.manual_seed(42)
    model = Foo().to(device)
    ref = Foo().to(device)
    ref.load_state_dict(model.state_dict())
    opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9, foreach=True)
    ropt = torch.optim.SGD(ref.parameters(), lr=0.1, momentum=0.9, foreach=True)
    g = torch.Generator().manual_seed(7)
    batches = [torch.randn(16, 64, generator=g).to(device) for _ in range(3)]
    compiled = api.compile_from_bundle(bundle, (batches[0], model, opt), {}, ops=ops, native=native,
                                       planner=planner)
    ok, msg = True, ""
    for b in batches:
        out = compiled(b, model, opt)
        want = train_step(b, ref, ropt)
        if out.shape != want.shape or not torch.allclose(out, want.detach(), rtol=1e-4, atol=1e-5):
            ok, msg = False, f"output differs: {(out - want).abs().max() if out.shape == want.shape else out.shape}"
    return ok, msg, compiled.info["comm_nodes"]


def _worker(rank, world, mesh_shape, port, q, bucket="0", planner="GREEDY"):
    os.environ["OMP_NUM_THREADS"] = "1"
    os.environ["EDB_BUCKET_COMM"] = bucket
    torch.set_num_threads(1)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank,
                            world_size=world)
    import numpy as np
    from tests import gloo_ops
    gloo_ops.init_groups(np.arange(world).reshape(mesh_shape))
    ok, msg, hist = run_bundle(rank, world, mesh_shape, gloo_ops, False, "cpu", planner=planner)
    if rank == 0:
        q.put((ok, msg, hist))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("planner,want", [
    # the reference's own lowering of this plan with that planner (tests/ref/auto_worker.py with
    # EDB_TEST_MESH=2x2 EDB_PLANNER=<planner> EDB_SAMEPLAN=1, `hist_ref_same_plan`); P2P's
    # histogram equals GREEDY's on this plan, REPLICATE gathers instead of all-to-all
    ("REPLICATE", {"all_gather_start": 45, "scatter_wrapper": 27, "reduce_scatter_start": 1,
                   "all_reduce_start": 5, "all_to_all_start": 0}),
    ("P2P", {"all_gather_start": 37, "scatter_wrapper": 19, "reduce_scatter_start": 1,
             "all_reduce_start": 5, "all_to_all_start": 2}),
])
def test_recorded_reference_plan_lowers_like_the_reference_with_other_planners(planner, want):
    """The drop-in lowering with the REPLICATE and P2P reshard planners on a 2x2 mesh: the plan
    the reference solved, lowered by this backend, matches vanilla PyTorch and has the same
    communication structure as the reference's lowering of that plan."""
    ok, msg, hist = run_world(_worker, 4, lambda r, port, q: (r, 4, (2, 2), port, q, "0", planner),
                              timeout=240)
    assert ok, msg
    for k, v in want.items():
        assert hist.get(k, 0) == v, (k, hist)


@pytest.mark.parametrize("mesh_shape", [(2,), (2, 2)])
def test_recorded_reference_plan_lowers_and_matches_vanilla(mesh_shape):
    world = 1
    for v in mesh_shape:
        world *= v
    ok, msg, hist = run_world(_worker, world, lambda r, port, q: (r, world, mesh_shape, port, q),
                              timeout=240)
    assert ok, msg
    # the communication structure the reference's own lowering produced for these plans
    want = {(2,): {"all_gather_start": 26, "all_reduce_start": 3, "scatter_wrapper": 13,
                   "all_to_all_start": 2},
            (2, 2): {"all_gather_start": 37, "scatter_wrapper": 19, "reduce_scatter_start": 1,
                     "all_reduce_start": 5, "all_to_all_start": 2}}[mesh_shape]
    for k, v in want.items():
        assert hist.get(k, 0) == v, (k, hist)


@pytest.mark.parametrize("mesh_shape", [(2,), (2, 2)])
def test_bucketed_small_collectives_match_vanilla(mesh_shape):
    """EDB_BUCKET_COMM=1 (lowering.bucket_small_comm, the analogue of the reference's comm_group
    pass): the same recorded plans with their small all-reduces / dim-0 all-gathers bucketed still
    reproduce vanilla PyTorch, with fewer collectives."""
    world = 1
    for v in mesh_shape:
        world *= v
    ok, msg, hist = run_world(_worker, world,
                              lambda r, port, q: (r, world, mesh_shape, port, q, "1"), timeout=240)
    assert ok, msg
    plain = {(2,): (26, 3), (2, 2): (37, 5)}[mesh_shape]
    assert hist.get("all_gather_start", 0) < plain[0], hist
    assert hist.get("all_reduce_start", 0) <= plain[1], hist


def _close(got, want, rtol, atol, floor_rms=1e-6):
    """fp32: the reference's comparator (assert_close semantics).  `rtol=None` = low precision
    (bf16 replay of a plan): partial products are rounded before they are summed across ranks, so
    single elements differ by ulps of the *tensor's* scale; compare the relative L2 error (`atol`)."""
    if got.shape != want.shape:
        return False
    if rtol is None:
        # floor_rms: tensors far below the scale of their peers are rounding noise (gradients that
        # are zero analytically, e.g. the key bias under softmax) and are compared against that scale
        den = max(float(want.float().norm()), floor_rms * want.numel() ** 0.5)
        return float((got.float() - want.float()).norm()) <= atol * den
    return torch.allclose(got, want, rtol=rtol, atol=atol)


def run_c1_bundle(rank, world, ops, native, device, steps=2, tag=None, bundle_file=None,
                  gpt=(4, 1024, 32), batch=None, seq=128, vanilla_ranks=None,
                  dtype=torch.float32, rtol=1e-4, atol=1e-5):
    """SURVEY.md config 1 (the reference's examples/torch/gpt_train.py model: GPT depth 4, dim
    1024, 32 heads, batch 4 x 128, fp32, world 2) with the plan the reference's solver produced for
    it (tests/golden/auto_gpt_c1_mesh2.json.gz, recorded by tests/ref/auto_worker.py with
    EDB_MODEL=gpt EDB_GPT=4,1024,32,4,128).  Returns (ok, message, comm histogram)."""
    import gzip
    import numpy as np
    from easydist_b200 import api
    from easydist_b200.device_mesh import get_device_mesh as get_mesh, set_device_mesh
    from easydist_b200.workloads import EmbeddingGPT, embedding_gpt_train_step
    tag = tag or str(world)                      # "2", "4", "8" (1-D meshes) or "2x2"
    mesh_shape = tuple(int(v) for v in tag.split("x"))
    set_device_mesh(np.arange(world).reshape(mesh_shape), [f"spmd{i}" for i in range(len(mesh_shape))],
                    rank=rank)
    # other bundles of the same model family (tools/validate_bundle.py): file, (depth, dim, heads),
    # batch and sequence length they were solved for
    bundle = gzip.open(bundle_file or os.path.join(GOLDEN, f"auto_gpt_c1_mesh{tag}.json.gz"), "rt").read()
    torch.manual_seed(42)
    model = EmbeddingGPT(*gpt).to(device=device, dtype=dtype)
    # vanilla_ranks: the ranks that hold the vanilla model and compare (all by default; big models on
    # one host: rank 0 only — the others still take part in the gathers)
    check = vanilla_ranks is None or rank in vanilla_ranks
    ref = EmbeddingGPT(*gpt).to(device=device, dtype=dtype) if check else model
    if check:
        ref.load_state_dict(model.state_dict())
    opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9, foreach=True)
    ropt = torch.optim.SGD(ref.parameters(), lr=0.1, momentum=0.9, foreach=True) if check else None
    g = torch.Generator().manual_seed(7)
    if batch is None:
        batch = 8 if tag == "8" else 4            # the (8,) plan was solved for a batch of 8
    batches = [torch.randn(batch, seq, gpt[1], generator=g).to(device=device, dtype=dtype)
               for _ in range(steps)]
    # EDB_TEST_AUTO_PF=1 (CPU): the parameter-prefetch rewrite of the product path too, with the
    # stand-in runtime of tests/gloo_ops.py (offsets only; `gathered` is a real gloo all-gather)
    fake_rt = ops.FakeSymmRuntime() if (not native and os.environ.get("EDB_TEST_AUTO_PF") == "1") else None
    compiled = api.compile_from_bundle(bundle, (batches[0], model, opt), {}, ops=ops, native=native,
                                       fuse_rt=fake_rt)
    ok, msg = True, ""
    for b in batches:
        out = compiled(b, model, opt)
        if not check:
            continue
        want = embedding_gpt_train_step(b, ref, ropt)
        if not _close(out, want.detach(), rtol, atol):
            ok, msg = False, f"output differs by {(out - want).abs().max()}"
    # the reference's comparator (tests/test_torch/test_spmd.py:97-113): every parameter and every
    # optimizer state, re-assembled from the shards the plan left on each rank
    mesh = get_mesh()
    env = compiled.graph._edb_shard_env
    phs = [n for n in compiled.graph.graph.nodes if n.op == "placeholder"]
    params, _, named_states = compiled.get_state()
    flat_states, _ = torch.utils._pytree.tree_flatten(named_states)
    names = list(params) + [f"state{i}" for i in range(len(flat_states))]
    locals_ = list(params.values()) + flat_states
    ph_of = phs[:len(params)] + phs[len(params) + len(compiled.get_state()[1]):
                                     len(params) + len(compiled.get_state()[1]) + len(flat_states)]
    if check:
        ref_states, _ = torch.utils._pytree.tree_flatten(
            {n: ropt.state[p] for n, p in ref.named_parameters()})
        wants = [p.detach() for p in ref.parameters()] + ref_states
    else:
        wants = list(locals_)
    rms = lambda t: float(t.float().pow(2).mean().sqrt())
    n_par = len(params)
    floors = [1e-2 * max([rms(w) for w in grp if isinstance(w, torch.Tensor)] + [1e-30])
              for grp in (wants[:n_par], wants[n_par:])]
    for i, (name, loc, ph, want_t) in enumerate(zip(names, locals_, ph_of, wants)):
        if not isinstance(loc, torch.Tensor) or not isinstance(want_t, torch.Tensor):
            continue
        full = loc.detach()
        strat = env.get(ph.name)
        if strat is not None:
            for mdim in reversed(range(len(strat))):
                sp = strat[mdim]
                if sp.is_shard():
                    grp = mesh.ranks_along(mdim)
                    full = ops.all_gather_end(ops.all_gather_start(full.contiguous(), sp.dim, grp),
                                              sp.dim, grp)
        if check and not _close(full, want_t, rtol, atol, floors[0 if i < n_par else 1]):
            ok, msg = False, f"{name} {tuple(want_t.shape)} differs: " + (
                f"max abs {float((full - want_t).abs().max()):.3e}, rel L2 "
                f"{float((full.float() - want_t.float()).norm() / want_t.float().norm().clamp_min(1e-30)):.3e}"
                                                    if full.shape == want_t.shape else
                                                    f"{tuple(full.shape)} vs {tuple(want_t.shape)}")
    return ok, msg, compiled.info["comm_nodes"]


def _c1_worker(rank, world, port, q, localize="0", auto_pf="0"):
    os.environ["OMP_NUM_THREADS"] = "2"
    os.environ["EDB_LOCALIZE_OPT"] = localize
    os.environ["EDB_TEST_AUTO_PF"] = auto_pf
    torch.set_num_threads(2)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank,
                            world_size=world)
    import numpy as np
    from tests import gloo_ops
    gloo_ops.init_groups(np.arange(world).reshape((world,)))
    ok, msg, hist = run_c1_bundle(rank, world, gloo_ops, False, "cpu")
    if rank == 0:
        q.put((ok, msg, hist))
    dist.barrier()
    dist.destroy_process_group()


def test_config1_gpt_plan_from_the_reference_solver_matches_vanilla():
    ok, msg, hist = run_world(_c1_worker, 2, lambda r, port, q: (r, 2, port, q), timeout=600)
    assert ok, msg
    # what the reference's own lowering produces for this very plan (tests/ref/auto_worker.py,
    # EDB_SAMEPLAN=1: same_plan_equal=True)
    want = {"all_gather_start": 429, "scatter_wrapper": 197, "reduce_scatter_start": 8,
            "all_reduce_start": 17, "all_to_all_start": 52}
    for k, v in want.items():
        assert hist.get(k, 0) == v, (k, hist)


def _gpt_test_worker(rank, world, port, q):
    os.environ["OMP_NUM_THREADS"] = "1"
    torch.set_num_threads(1)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank,
                            world_size=world)
    import numpy as np
    from tests import gloo_ops
    gloo_ops.init_groups(np.arange(world).reshape((world,)))
    ok, msg, hist = run_c1_bundle(rank, world, gloo_ops, False, "cpu", steps=2,
                                  bundle_file=os.path.join(GOLDEN, "auto_gpt_test_mesh2.json.gz"),
                                  gpt=(2, 64, 4), batch=4, seq=32)
    if rank == 0:
        q.put((ok, msg, hist))
    dist.barrier()
    dist.destroy_process_group()


def test_reference_test_gpt_plan_lowers_like_the_reference():
    """The reference's own GPT test model (depth 2, dim 64, 4 heads; batch 4 x 32) with the plan its
    solver produced at mesh (2,) (recorded by tests/ref/auto_worker.py with EDB_MODEL=gpt
    EDB_SAMEPLAN=1): this backend's lowering matches vanilla PyTorch in outputs, every parameter and
    every momentum buffer, and has the communication structure of the reference's lowering of the
    same plan (`hist_ref_same_plan` of that run)."""
    ok, msg, hist = run_world(_gpt_test_worker, 2, lambda r, port, q: (r, 2, port, q), timeout=300)
    assert ok, msg
    want = {"all_gather_start": 215, "scatter_wrapper": 99, "reduce_scatter_start": 14,
            "all_reduce_start": 9, "all_to_all_start": 8}
    for k, v in want.items():
        assert hist.get(k, 0) == v, (k, hist)


def test_config1_optimizer_runs_on_shards_when_localized():
    """lowering.localize_foreach on the same plan: the optimizer's foreach ops run on the shards
    (the reference gathers every parameter / gradient / state in front of each of them and scatters
    the results back, SURVEY.md fact 5).  Results still equal vanilla — outputs, every parameter,
    every momentum buffer — with 2/3 of the all-gathers and all optimizer scatters gone."""
    ok, msg, hist = run_world(_c1_worker, 2, lambda r, port, q: (r, 2, port, q, "1"), timeout=600)
    assert ok, msg
    assert hist.get("all_gather_start", 0) <= 429 - 280, hist
    assert hist.get("scatter_wrapper", 0) <= 197 - 170, hist


def test_config1_parameter_gathers_become_prefetches():
    """The product structure executed on CPU: optimizer on shards AND the parameter-prefetch rewrite
    (lowering.prefetch_param_gathers with the stand-in runtime; `gathered` = a real gloo all-gather of
    the flat shard).  Weights the plan shards along dim 0 are read as views of their gathered buffer;
    weights it shards along dim 1 (gathers of t(W_shard) in front of the GEMMs) through one local
    permuted copy of the buffer — 68 of the 125 all-gathers become buffer reads, results still equal
    vanilla: outputs, every parameter, every momentum buffer."""
    ok, msg, hist = run_world(_c1_worker, 2, lambda r, port, q: (r, 2, port, q, "1", "1"), timeout=600)
    assert ok, msg
    assert hist.get("gathered") == 68 and hist.get("all_gather_start") == 57, hist
    assert hist.get("ag_prefetch") == 1 and hist.get("epoch_barrier") == 2, hist


@pytest.mark.parametrize("tag,mesh_shape,rank,want", [
    ("4", (4,), 3, {"all_gather_start": 429, "scatter_wrapper": 197, "reduce_scatter_start": 12,
                    "all_reduce_start": 17, "all_to_all_start": 24}),
    ("8", (8,), 5, {"all_gather_start": 437, "scatter_wrapper": 197, "reduce_scatter_start": 20,
                    "all_reduce_start": 17, "all_to_all_start": 24}),
    ("2x2", (2, 2), 2, {"all_gather_start": 675, "scatter_wrapper": 319, "reduce_scatter_start": 12,
                        "all_reduce_start": 54, "all_to_all_start": 95}),
])
def test_config1_plans_for_larger_meshes_lower_to_the_recorded_structure(tag, mesh_shape, rank, want):
    """The config-1 plans the reference solved for meshes (4,), (8,) and (2,2) (each verified against
    vanilla inside the reference's pipeline when it was recorded, tests/ref/auto_worker.py) lower —
    for an arbitrary rank of the mesh, in one process, nothing executed — to the communication
    structure recorded with them.  (Execution of these meshes is the GPU worker's job.)"""
    import gzip
    import numpy as np
    from easydist_b200 import api
    from easydist_b200.device_mesh import set_device_mesh
    from easydist_b200.workloads import EmbeddingGPT
    from tests import gloo_ops
    world = int(np.prod(mesh_shape))
    set_device_mesh(np.arange(world).reshape(mesh_shape), [f"spmd{i}" for i in range(len(mesh_shape))],
                    rank=rank)
    bundle = gzip.open(os.path.join(GOLDEN, f"auto_gpt_c1_mesh{tag}.json.gz"), "rt").read()
    torch.manual_seed(0)
    model = EmbeddingGPT(4, 1024, 32)
    opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9, foreach=True)
    batch = 8 if tag == "8" else 4
    compiled = api.compile_from_bundle(bundle, (torch.randn(batch, 128, 1024), model, opt), {},
                                       ops=gloo_ops, native=False)
    hist = compiled.info["comm_nodes"]
    for k, v in want.items():
        assert hist.get(k, 0) == v, (k, hist)
    # every parameter ended up with its local shard shape under the plan
    full = dict(model.named_parameters())
    assert any(p.shape != full[n].shape for n, p in compiled.named_parameters().items())


@pytest.mark.parametrize("name,gpt,world,rank,batch,seq,want", [
    ("gpt2small_s256_mesh2", (12, 768, 12), 2, 1, 4, 256,
     {"all_gather_start": 1285, "scatter_wrapper": 589, "reduce_scatter_start": 84,
      "all_reduce_start": 49, "all_to_all_start": 48}),
    ("gpt2small_s256_mesh8", (12, 768, 12), 8, 5, 8, 256,
     {"all_gather_start": 1309, "scatter_wrapper": 589, "reduce_scatter_start": 60,
      "all_reduce_start": 49, "all_to_all_start": 72}),
    # BASELINE.json configs[1]'s model size (GPT-2 medium: depth 24, dim 1024, 16 heads) in the
    # reference's own benchmark-GPT form, solved by the unmodified reference at world 2
    ("gpt2medium_s128_mesh2", (24, 1024, 16), 2, 0, 4, 128,
     {"all_gather_start": 2569, "scatter_wrapper": 1177, "reduce_scatter_start": 72,
      "all_reduce_start": 97, "all_to_all_start": 144}),
    # ... and at world 8 (capture-only recording: no reference-lowering histogram to compare with;
    # executed against vanilla with tools/validate_bundle.py)
    ("gpt2medium_s128_mesh8", (24, 1024, 16), 8, 3, 8, 128, None),
])
def test_gpt2_small_and_medium_size_plans_lower_to_the_recorded_structure_and_pass_the_static_check(
        name, gpt, world, rank, batch, seq, want, monkeypatch):
    """A GPT-2-small-sized model (the reference's benchmark GPT: depth 12, dim 768, 12 heads, batch
    4 x 256 at world 2, 8 x 256 at world 8; SURVEY.md 8(d) 'GPT-2 small variant') solved by the
    unmodified reference on meshes (2,) and (8,) and recorded with tests/ref/auto_worker.py (there:
    outputs and parameters == vanilla, and this lowering == the reference's lowering of the very same
    plan, e.g. mesh (2,): 1285 all-gathers, 589 scatters, 84 reduce-scatters, 49 all-reduces, 48
    all-to-alls).  Here, without the reference and without
    executing anything: (1) the bundle lowers to that structure; (2) with the product passes
    (optimizer on shards, parameter gathers as prefetches, push collectives, epoch barriers) two
    thirds of the all-gathers are gone and the static epoch-protocol check passes."""
    import gzip
    import numpy as np
    from easydist_b200 import api, lowering
    from easydist_b200.device_mesh import set_device_mesh
    from easydist_b200.workloads import EmbeddingGPT
    from tests import gloo_ops
    set_device_mesh(np.arange(world).reshape((world,)), ["spmd0"], rank=rank)
    bundle = gzip.open(os.path.join(GOLDEN, f"auto_{name}.json.gz"), "rt").read()

    def build():
        torch.manual_seed(0)
        model = EmbeddingGPT(*gpt)
        opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9, foreach=True)
        return api.compile_from_bundle(bundle, (torch.randn(batch, seq, gpt[1]), model, opt), {},
                                       ops=gloo_ops, native=False)

    if want is not None:
        monkeypatch.setenv("EDB_LOCALIZE_OPT", "0")
        hist = build().info["comm_nodes"]
        for k, v in want.items():
            assert hist.get(k, 0) == v, (k, hist)
    monkeypatch.setenv("EDB_LOCALIZE_OPT", "1")
    compiled = build()
    n_ag_localized = compiled.info["comm_nodes"].get("all_gather_start", 0)
    gm = compiled.graph
    params = compiled.get_state()[0]
    phs = [n for n in gm.graph.nodes if n.op == "placeholder"]
    auto_io = api._ParamIO(phs[:len(params)], list(params.keys()))
    rt = gloo_ops.FakeSymmRuntime()
    ranks = list(range(world))
    rehomed, n_pf = lowering.prefetch_param_gathers(gm, auto_io, rt, ranks, gloo_ops, my_index=rank)
    assert n_pf == len(rehomed) > 100
    lowering.insert_epoch_barriers(gm, ranks, gloo_ops)
    lowering.assign_static_buffers(gm, rt, gloo_ops, push=True)
    lowering.ensure_end_barrier(gm, ranks, gloo_ops)
    lowering.dispatch_compute(gm)
    after = lowering.count_nodes(gm, gloo_ops)
    n_ag_ref = want["all_gather_start"] if want else 3 * n_ag_localized
    assert after.get("all_gather_start", 0) < n_ag_ref // 3, after
    rep = lowering.verify_epoch_protocol(gm, gloo_ops, world)
    assert rep["ok"], rep["problems"]
