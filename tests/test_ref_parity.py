"""Reference-in-the-loop parity (needs the original easydist sources, EASYDIST_REFERENCE).  The unmodified
reference traces, annotates and solves; its lowering (A) and the drop-in
easydist_b200.lowering.sharding_transform (B) are run on the same plan and inputs over gloo and
compared with each other and with vanilla PyTorch — tests/ref/auto_worker.py.  Every case of
test_dropin_lowering_equals_reference_lowering has a recorded counterpart in
tests/test_auto_bundle_cpu.py (the reference's plan + its lowering's communication histogram,
replayed without the reference); the plugin-hook tests drive the reference's own decorator and
have none."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.refcompat import REFERENCE_ROOT  # noqa: E402
from tests._procs import run_torchrun  # noqa: E402
pytestmark = pytest.mark.refonly


@pytest.mark.parametrize("mesh,nproc,planner,model", [
    ("2", 2, "GREEDY", "foo"), ("2x2", 4, "GREEDY", "foo"),
    ("2x2", 4, "REPLICATE", "foo"), ("2x2", 4, "P2P", "foo"),
    ("2", 2, "GREEDY", "gpt"),   # the reference's GPT test model: views, expand, bmm
])
def test_dropin_lowering_equals_reference_lowering(mesh, nproc, planner, model):
    if not os.path.isdir(os.path.join(REFERENCE_ROOT, "easydist")):
        pytest.skip("original easydist sources not present (set EASYDIST_REFERENCE)")
    env = dict(os.environ, EDB_TEST_MESH=mesh, OMP_NUM_THREADS="1", EDB_PLANNER=planner,
               EDB_MODEL=model, EDB_SAMEPLAN="1")
    rc, out, err = run_torchrun(os.path.join(ROOT, "tests", "ref", "auto_worker.py"), nproc, env,
                                timeout=280, cwd=ROOT, python=sys.executable)
    line = next((l for l in out.splitlines() if l.startswith("AUTO_PARITY")), "")
    assert rc == 0 and "ok=True" in line, out[-2000:] + err[-3000:]
    # same communication structure as the reference's lowering OF THE VERY SAME PLAN (run A solves
    # again and the ILP may return another equal-cost plan, so its histogram is informative only)
    assert "same_plan_equal=True" in line, line


@pytest.mark.parametrize("mode", ["b200_ddp", "b200_zero3", "auto", "b200_auto", "auto+localize",
                                  "b200_auto+gpt"])
def test_plugin_hook_through_the_reference_decorator(mode):
    """Hook A of INTEGRATION.md: `easydist_b200.api.register()` adds the modes to the reference's
    registry (`register_parallel_method`, api.py:39-50); the REFERENCE's own `easydist_compile`
    decorator and CompiledFuncWrapper then drive this backend's compiled object (`.graph`,
    `.run_with_graph`, state accessors); "auto" = Hook B, the `sharding_transform` name rebound by
    the same call; "b200_auto" = Hook C: the reference's tracing + annotation + ILP produce the plan,
    this backend lowers AND executes it (its own EDCompiledFunc, no per-step distribute_tensor) —
    tests/ref/plugin_worker.py."""
    if not os.path.isdir(os.path.join(REFERENCE_ROOT, "easydist")):
        pytest.skip("original easydist sources not present (set EASYDIST_REFERENCE)")
    env = dict(os.environ, OMP_NUM_THREADS="1", EDB_PLUGIN_MODE=mode)
    if mode == "auto+localize":
        # Hook B with the optimizer localized: the REFERENCE's executor runs the rewritten graph
        env.update(EDB_PLUGIN_MODE="auto", EDB_LOCALIZE_OPT="1")
    cached = mode == "b200_auto"
    if mode == "b200_auto+gpt":
        # Hook C on the reference's GPT test model, with the product structure of the auto path
        # (optimizer on shards, parameter gathers rewritten to prefetched-buffer reads) executed by
        # this backend's EDCompiledFunc
        mode = "b200_auto"
        env.update(EDB_PLUGIN_MODE="b200_auto", EDB_PLUGIN_MODEL="gpt", EDB_LOCALIZE_OPT="1",
                   EDB_TEST_AUTO_PF="1")
    elif mode == "b200_auto":
        import tempfile
        env["EDB_PLAN_CACHE_DIR"] = tempfile.mkdtemp(prefix="edb_plan_cache_")
    rc, out, err = run_torchrun(os.path.join(ROOT, "tests", "ref", "plugin_worker.py"), 2, env,
                                timeout=280, cwd=ROOT, python=sys.executable)
    line = next((l for l in out.splitlines() if l.startswith("PLUGIN_PARITY")), "")
    assert rc == 0 and "ok=True" in line, out[-2000:] + err[-3000:]
    if mode.startswith("b200_"):
        # the object the reference's wrapper drives is THIS backend's executor
        assert "compiled=easydist_b200.compile.EDCompiledFunc" in line, line
    if env.get("EDB_TEST_AUTO_PF") == "1":
        assert "'ag_pf': 0" not in line and "'ag_pf'" in line, line   # the prefetch rewrite applied
    if cached:
        # ... and a second compilation took graph + plan from the plan cache (SURVEY f2)
        assert "plan_source=['solved', 'cache']" in line, line
