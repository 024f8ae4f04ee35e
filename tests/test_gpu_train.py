"""End-to-end train step through the compiled path on one H100 vs the oracle (CPU fp32
restatement of the same step).  bf16 GPU vs fp32 CPU: the loss trajectory must agree within 3e-2
relative (bf16 keeps 8 mantissa bits; the reference's own comparator uses rtol 1e-4 for fp32,
tests/test_torch/test_spmd.py:67, which is what the fp32 case below holds itself to)."""
import pytest
import torch

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


@pytest.mark.parametrize("dtype,cuda_graph,rtol", [(torch.float32, False, 1e-4),
                                                    (torch.float32, True, 1e-4),
                                                    (torch.bfloat16, False, 3e-2),
                                                    (torch.bfloat16, True, 3e-2)])
def test_gpt2_tiny_train_steps_match_oracle(rt, dtype, cuda_graph, rtol):
    """Loss of every call vs the oracle (CPU fp32 restatement), then the reference's comparator
    (tests/test_torch/test_spmd.py:97-113): EVERY parameter and EVERY optimizer state against
    vanilla fp32 PyTorch after the same optimisation steps — assert_close(rtol 1e-4, atol 1e-5)
    for fp32; for bf16 (8 mantissa bits) bf16-ulp / relative-L2 bounds calibrated by what vanilla
    bf16 eager PyTorch itself reaches against fp32 (tools/parity.py).  With a CUDA graph the first
    call performs TWO updates on the first batch (eager warm-up + first replay, exactly like the
    reference's wrapper, api.py:183-222) and returns the loss of the second; the vanilla schedule
    accounts for it."""
    from easydist_b200 import gemm, loss as loss_mod, optim as optim_mod
    from easydist_b200.api import easydist_compile
    from easydist_b200.workloads import GPT2, GPT2_CONFIGS, gpt2_train_step, synthetic_tokens
    from oracle import train_oracle
    from tools import parity as P
    cfg = GPT2_CONFIGS["gpt2-tiny"]
    torch.manual_seed(0)
    model = GPT2(cfg).to(device="cuda", dtype=dtype)
    state = {k: v.detach().clone() for k, v in model.state_dict().items()}
    mk_opt = lambda ps: torch.optim.SGD(ps, lr=1e-3, momentum=0.9, foreach=True)
    opt = mk_opt(model.parameters())
    step = easydist_compile(gpt2_train_step, parallel_mode="ddp", tracing_mode="fake",
                            cuda_graph=cuda_graph)
    calls = 4
    gemm.reset_stats()
    loss_mod.reset_stats()
    optim_mod.reset_stats()
    batches = [synthetic_tokens(cfg, 4, 64, seed=1000 * b) for b in range(calls)]
    losses = []
    for tok, tgt in batches:
        losses.append(float(step(tok.cuda(), tgt.cuda(), model, opt)))
    sched = ([0, 0] if cuda_graph else [0]) + list(range(1, calls))
    steps = [[batches[b]] for b in sched]
    ref_l, ref_p, ref_s = P.vanilla_run(lambda: GPT2(cfg), state, steps, mk_opt, torch.float32, "cuda")
    idx = [1 if cuda_graph else 0] + list(range(2 if cuda_graph else 1, len(sched)))
    for got, i in zip(losses, idx):
        assert abs(got - ref_l[i][0]) <= rtol * abs(ref_l[i][0]), (losses, ref_l)
    if not cuda_graph:
        # the oracle (CPU restatement) agrees with the GPU fp32 vanilla run it is checked against
        want, _ = train_oracle.train_losses("gpt2-tiny", cfg.attn, 4, 64, steps=calls, state_dict=state)
        for got, w in zip(losses, want):
            assert abs(got - w) <= rtol * abs(w), (losses, want)
    got_p, got_s = P.compiled_state(step.compiled_func, ref_p, ref_s, 1)
    if dtype == torch.float32:
        res = P.compare(got_p, got_s, ref_p, ref_s, low_precision=False)
        assert res["assert_close_violation"] <= 1.0, res
    else:
        _, van_p, van_s = P.vanilla_run(lambda: GPT2(cfg), state, steps, mk_opt, torch.bfloat16, "cuda")
        van = P.compare({k: v.bfloat16() for k, v in van_p.items()},
                        {k: {kk: vv.bfloat16() for kk, vv in st.items()} for k, st in van_s.items()},
                        ref_p, ref_s, low_precision=True)
        res = P.compare(got_p, got_s, ref_p, ref_s, low_precision=True)
        assert res["state_rel_l2"] <= max(2e-2, 2.0 * van["state_rel_l2"]), (res, van)
        assert res["param_max_ulp"] <= max(2.0, 2.0 * van["param_max_ulp"]), (res, van)
        assert gemm.stats()["edb_gemm"] > 0, "bf16 Linear layers must run on the native GEMM"
    st = loss_mod.stats()
    assert st["edb_ce_fwd"] > 0 and st["edb_ce_bwd"] > 0 and st["aten_ce"] == 0, st
    ost = optim_mod.stats()
    assert ost["edb_sgd"] > 0 and ost["aten_sgd"] == 0, ost
