"""Config 1 (the reference's examples/torch/gpt_train.py model: GPT depth 4 / dim 1024 / 32 heads,
fp32) in AUTO-SPMD mode on N GPUs: the plan is the one the reference's solver produced for this
mesh (tests/golden/auto_gpt_c1_mesh{N}.json.gz), lowered and executed by this backend.
Prints one JSON line (samples/s, ms/step, comm histogram).  EDB_BUCKET_COMM=1 buckets the small
collectives of the plan.

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/bench_c1_auto.py [--mesh 2x2]
"""
import argparse
import gzip
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

from easydist_b200 import api, runtime
from easydist_b200.device_mesh import set_device_mesh
from easydist_b200.workloads import EmbeddingGPT


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mesh", default="")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-cuda-graph", action="store_true")
    ap.add_argument("--bundle", default="",
                    help="another recorded graph + plan (graph_io bundle, .json or .json.gz) instead of "
                         "the config-1 golden bundles; give the model with --gpt")
    ap.add_argument("--gpt", default="", help="depth,dim,heads,batch,seq of the bundle's model")
    ap.add_argument("--dtype", default="fp32", choices=["fp32", "bf16"],
                    help="bf16: parameters and inputs in bf16 (the plan is dtype independent; the "
                         "Linear layers then run on the native wgmma GEMM)")
    run(ap.parse_args())


def run(args):
    """Also the body of `bench.py --mode auto` (args: mesh, steps, warmup, no_cuda_graph)."""
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    runtime.init(rank, world, local, heap_bytes=16 << 30)
    tag = args.mesh or str(world)
    mesh_shape = tuple(int(v) for v in tag.split("x"))
    set_device_mesh(np.arange(world).reshape(mesh_shape), [f"spmd{i}" for i in range(len(mesh_shape))],
                    rank=rank)
    golden = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
    custom = getattr(args, "bundle", "")
    depth, dim, heads, gbatch, seq = 4, 1024, 32, (8 if tag == "8" else 4), 128
    if custom:
        opener = gzip.open if custom.endswith(".gz") else open
        bundle = opener(custom, "rt").read()
        depth, dim, heads, gbatch, seq = (int(v) for v in args.gpt.split(","))
    else:
        bundle = gzip.open(os.path.join(golden, f"auto_gpt_c1_mesh{tag}.json.gz"), "rt").read()
    tdt = torch.bfloat16 if getattr(args, "dtype", "fp32") == "bf16" else torch.float32
    # parity first (outside the timed region): outputs, every parameter and every momentum buffer
    # vs vanilla PyTorch on the same batches (the reference's comparator, rtol 1e-4 / atol 1e-5)
    from easydist_b200 import reshard
    from tests.test_auto_bundle_cpu import run_c1_bundle
    if tdt != torch.float32:
        ok, msg = True, "parity leg runs in fp32 only (bf16: tools/validate_bundle.py --dtype bf16)"
    elif custom:
        ok, msg, _ = run_c1_bundle(rank, world, reshard, True, "cuda", steps=3, tag=tag,
                                   bundle_file=custom, gpt=(depth, dim, heads), batch=gbatch, seq=seq)
    else:
        ok, msg, _ = run_c1_bundle(rank, world, reshard, True, "cuda", steps=3, tag=tag)
    flag = torch.tensor([0.0 if ok else 1.0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MAX)
    parity_ok = bool(flag.item() == 0.0)
    if not ok:
        print(f"[rank {rank}] parity failed: {msg}", flush=True)
    torch.manual_seed(42)
    model = EmbeddingGPT(depth, dim, heads).cuda().to(tdt)
    opt = torch.optim.SGD(model.parameters(), lr=1e-3, momentum=0.9, foreach=True)
    batch = gbatch
    x = torch.randn(batch, seq, dim, device="cuda").to(tdt)
    compiled = api.compile_from_bundle(bundle, (x, model, opt), {})
    step = lambda: compiled(x, model, opt)
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    if not args.no_cuda_graph:
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        step = graph.replay
    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / args.steps], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    if rank == 0:
        ms = t.item()
        print(json.dumps({"metric": "train_step_throughput", "value": batch / ms * 1e3, "unit": "samples/s",
                          "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
                          "ms_per_step": ms, "higher_is_better": True, "scaling": "strong",
                          "vs_baseline": None, "data": "synthetic",
                          "dtype": "bf16" if tdt == torch.bfloat16 else "f32",
                          "config": {"workload": f"GPT depth {depth} dim {dim} heads {heads}, batch "
                                                 f"{batch}x{seq}, auto-SPMD plan of the reference solver"
                                                 + ("" if custom else " (config 1)"),
                                     "mesh": list(mesh_shape), "cuda_graph": not args.no_cuda_graph,
                                     "bucket_comm": os.environ.get("EDB_BUCKET_COMM", "0")},
                          "parity": {"ok": parity_ok, "what": "3 steps vs vanilla fp32 PyTorch: outputs, every "
                                     "parameter, every momentum buffer (rtol 1e-4, atol 1e-5)"},
                          "localized_foreach": compiled.info.get("localized_foreach"),
                          "fused": compiled.info.get("fused"),
                          "comm_nodes": compiled.info["comm_nodes"]}), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
