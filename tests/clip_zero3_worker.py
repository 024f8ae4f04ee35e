"""torchrun worker of tests/test_gpu_clip.py::test_zero3_with_clipping_on_two_gpus: the zero3 step of a
small Llama with clip_grad_norm_ active, through easydist_compile (eager and CUDA graph), against
vanilla fp32 PyTorch on the same global batches, and the parameters bit-identical across ranks."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from easydist_b200 import runtime  # noqa: E402
from easydist_b200.api import easydist_compile  # noqa: E402
from easydist_b200.device_mesh import set_device_mesh  # noqa: E402
from easydist_b200.workloads import Llama, LlamaConfig, synthetic_tokens  # noqa: E402
from tests.test_gpu_clip import MAX_NORM, _clipped, clipped_train_step  # noqa: E402
from tools import parity as P  # noqa: E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rt = runtime.init(rank, world, local, heap_bytes=2 << 30)
    rt.set_option("spin_timeout_ms", 20000)
    set_device_mesh(list(range(world)), ["dp"], rank=rank)
    cfg = LlamaConfig(n_layer=2, n_head=4, n_embd=256, ffn=688, vocab_size=512, block_size=64)
    mk_opt = lambda ps: torch.optim.SGD(ps, lr=1e-2, momentum=0.9, foreach=True)
    mk_ref = lambda ps: _clipped(torch.optim.SGD)(ps, lr=1e-2, momentum=0.9, foreach=True)
    for cuda_graph in (False, True):
        torch.manual_seed(0)
        model = Llama(cfg).to(device="cuda", dtype=torch.bfloat16)
        state0 = {k: v.detach().clone() for k, v in model.state_dict().items()}
        opt = mk_opt(model.parameters())
        batches = [[synthetic_tokens(cfg, 2, 64, seed=500 + 100 * b + r) for r in range(world)]
                   for b in range(3)]
        step = easydist_compile(clipped_train_step, parallel_mode="zero3", tracing_mode="fake",
                                cuda_graph=cuda_graph)
        losses = [float(step(batches[b][rank][0].cuda(), batches[b][rank][1].cuda(), model, opt))
                  for b in range(3)]
        info = step.compiled_func.info
        assert info["clip_nodes"][1] > 0, info
        sched = ([0, 0] if cuda_graph else [0]) + [1, 2]
        steps = [batches[b] for b in sched]
        ref_l, ref_p, ref_s = P.vanilla_run(lambda: Llama(cfg), state0, steps, mk_ref, torch.float32, "cuda")
        _, van_p, van_s = P.vanilla_run(lambda: Llama(cfg), state0, steps, mk_ref, torch.bfloat16, "cuda")
        got_p, got_s = P.compiled_state(step.compiled_func, ref_p, ref_s, world)
        ours = P.compare(got_p, got_s, ref_p, ref_s, low_precision=True)
        van = P.compare({k: v.bfloat16() for k, v in van_p.items()},
                        {k: {kk: vv.bfloat16() for kk, vv in st.items()} for k, st in van_s.items()},
                        ref_p, ref_s, low_precision=True)
        idx = [1 if cuda_graph else 0, len(sched) - 2, len(sched) - 1]
        for got, i in zip(losses, idx):
            assert abs(got - ref_l[i][rank]) <= 2e-2 * abs(ref_l[i][rank]), (losses, ref_l)
        assert ours["state_rel_l2"] <= max(2e-2, 2.0 * van["state_rel_l2"]), (ours, van)
        assert ours["param_max_ulp"] <= max(2.0, 2.0 * van["param_max_ulp"]), (ours, van)
        for name, p in got_p.items():
            peers = [torch.empty_like(p) for _ in range(world)]
            dist.all_gather(peers, p.contiguous())
            assert all(torch.equal(peers[0], x) for x in peers[1:]), f"{name} differs across ranks"
    torch.cuda.synchronize()
    assert not any(rt.error_flags())
    dist.barrier()
    if rank == 0:
        print(f"CLIP_ZERO3_OK world={world} max_norm={MAX_NORM}", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
