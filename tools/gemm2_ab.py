"""A/B of the plain-GEMM kernels on the bench workload, all arms in one process on one card.

Arms are the values of the `gemm2` option / EDB_GEMM2: 0 = k_gemm_bf16 everywhere, 1 = k_gemm2_bf16
for the plain 128 x 256-tile launches.

  1. the GEMM launch list of one bench step (GPT-2 medium, bf16, 8 x 512 tokens, zero3), recorded
     from the compiled step and replayed from one CUDA graph per arm as bench.gemm_roofline does
     (fresh operands per launch, plain launches: the list does not record epilogues); arms alternate
     inside every round; TF/s per arm and round, and the spread of each arm over the rounds;
  2. every distinct (M, N, K, layout) of the list on its own, us and TF/s per arm;
  3. the bench step itself: `bench.py` as a subprocess per arm and round (the compiled step bakes the
     kernel choice into its CUDA graph, so an arm is a process), ms/step per arm and round.

    python tools/gemm2_ab.py [--rounds 5] [--replays 20] [--step-rounds 3] [--steps 50]
                             [--out DIR]

Needs an H100; there is no CPU fall-back.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown (nvidia-smi failed)"


def step_launch_list(torch):
    """Compile the bench step once (as bench.run_edb does) and return its recorded GEMM launches."""
    import dataclasses
    from easydist_b200 import gemm, runtime
    from easydist_b200.api import easydist_compile
    from easydist_b200.device_mesh import set_device_mesh
    from easydist_b200.workloads import GPT2, GPT2_CONFIGS, gpt2_train_step, synthetic_tokens
    rt = runtime.init(0, 1, 0, heap_bytes=12 << 30)
    set_device_mesh([0], ["dp"], rank=0)
    cfg = dataclasses.replace(GPT2_CONFIGS["gpt2-medium"], attn="sdpa")
    torch.manual_seed(0)
    model = GPT2(cfg).to(device="cuda", dtype=torch.bfloat16)
    opt = torch.optim.SGD(model.parameters(), lr=1e-3, momentum=0.9, foreach=True)
    t, y = synthetic_tokens(cfg, 8, 512, seed=0)
    step_fn = easydist_compile(gpt2_train_step, parallel_mode="zero3", tracing_mode="fake",
                               cuda_graph=False, fuse=True)
    gemm.reset_stats()
    step_fn(t.cuda(), y.cuda(), model, opt)
    torch.cuda.synchronize()
    calls = gemm.recorded_calls()[:gemm.stats()["edb_gemm"]]
    del step_fn, model, opt
    torch.cuda.empty_cache()
    return rt, gemm, calls


def graph_of(torch, rt, gemm, ops, arm):
    """One CUDA graph of gemm.mm over `ops`, captured with the option at `arm`."""
    rt.set_option("gemm2", arm)
    for a, b in ops:
        gemm.mm(a, b)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for a, b in ops:
            gemm.mm(a, b)
    g.replay()
    torch.cuda.synchronize()
    return g


def replay_ms(torch, g, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def operands(torch, call):
    M, N, K, a_k, b_k, a_stride, b_stride = call
    a = torch.empty_strided((M, K), a_stride, device="cuda", dtype=torch.bfloat16).normal_()
    b = torch.empty_strided((K, N), b_stride, device="cuda", dtype=torch.bfloat16).normal_()
    return a, b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--step-rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", default=None, help="directory for gemm2_ab.json")
    args = ap.parse_args()
    arms = [0, 1]
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("gemm2_ab: no CUDA device: this measurement only exists on the GPU")
    result = {"card": card(), "arms": arms}
    print("card (name, power limit, max SM clock):", result["card"], flush=True)

    rt, gemm, calls = step_launch_list(torch)
    flops = sum(2 * c[0] * c[1] * c[2] for c in calls)
    print(f"launch list: {len(calls)} GEMMs, {flops / 1e12:.2f} TFLOP per step", flush=True)

    # 1. the whole list
    ops = [operands(torch, c) for c in calls]
    graphs = {arm: graph_of(torch, rt, gemm, ops, arm) for arm in arms}
    tf = {arm: [] for arm in arms}
    for r in range(args.rounds):
        for arm in arms:
            tf[arm].append(flops / replay_ms(torch, graphs[arm], args.replays) / 1e9)
        print(f"list round {r}: " + "  ".join(f"arm {a}: {tf[a][-1]:.1f} TF/s" for a in arms), flush=True)
    for arm in arms:
        lo, hi = min(tf[arm]), max(tf[arm])
        print(f"list arm {arm}: min {lo:.1f} max {hi:.1f} TF/s, spread {100 * (hi - lo) / lo:.2f} %")
    result["list_tflops"] = tf
    del graphs, ops
    torch.cuda.empty_cache()

    # 2. per distinct shape: 4 operand sets, 8 launches per replay
    shapes = {}
    for c in calls:
        shapes.setdefault(c[:5] + (c[5], c[6]), 0)
        shapes[c[:5] + (c[5], c[6])] += 1
    table = []
    print("per shape: M N K a_kmajor b_kmajor count | us and TF/s per arm", flush=True)
    for c, count in sorted(shapes.items(), key=lambda kv: -kv[1] * kv[0][0] * kv[0][1] * kv[0][2]):
        sets = [operands(torch, c) for _ in range(4)]
        gs = {arm: graph_of(torch, rt, gemm, sets * 2, arm) for arm in arms}
        best = {arm: float("inf") for arm in arms}
        for _ in range(3):
            for arm in arms:
                best[arm] = min(best[arm], replay_ms(torch, gs[arm], 10) / 8)
        row = {"M": c[0], "N": c[1], "K": c[2], "a_kmajor": c[3], "b_kmajor": c[4], "count": count,
               "us": {a: 1e3 * best[a] for a in arms},
               "tflops": {a: 2 * c[0] * c[1] * c[2] / best[a] / 1e9 for a in arms}}
        table.append(row)
        print(f"{c[0]:6d} {c[1]:6d} {c[2]:6d} {int(c[3])} {int(c[4])} x{count:3d} | " +
              "  ".join(f"{row['us'][a]:8.1f} us {row['tflops'][a]:6.1f}" for a in arms), flush=True)
        del gs, sets
    result["per_shape"] = table
    rt.set_option("gemm2", 1)

    # 3. the bench step, one process per arm and round
    step_ms = {arm: [] for arm in arms}
    for r in range(args.step_rounds):
        for arm in arms:
            env = dict(os.environ, EDB_GEMM2=str(arm))
            t0 = time.time()
            p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps",
                                str(args.steps), "--warmup", "5", "--no-parity", "--no-roofline",
                                "--no-cpu-baseline"], env=env, capture_output=True, text=True)
            line = next((l for l in reversed(p.stdout.splitlines()) if l.startswith("{")), None)
            if p.returncode != 0 or line is None:
                raise SystemExit(f"bench.py failed (arm {arm}):\n{p.stdout[-2000:]}\n{p.stderr[-2000:]}")
            step_ms[arm].append(json.loads(line)["ms_per_step"])
            print(f"step round {r} arm {arm}: {step_ms[arm][-1]:.3f} ms/step "
                  f"({time.time() - t0:.0f} s of process)", flush=True)
    result["step_ms"] = step_ms
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "gemm2_ab.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
