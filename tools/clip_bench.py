"""Gradient-norm clipping on the native kernels (edb_clip.cu, edb_sgd_momentum_scaled) against the
ATen ops they replace, on one GPU.  The card's name and power limit are read in the same run.

    python tools/clip_bench.py [--iters 100] [--step-iters 10] [--no-step] [--out results/clip.json]

kernel: the llama2-7b-l4 gradient shapes in bf16 (39 tensors, about 1.07 B elements), CUDA events:
        grad_norms against the T per-tensor linalg_vector_norm + stack, and sgd_momentum_ with
        grad_scale against the T mul_ + the fused SGD.  Algorithmic bytes: sum(numel)*2 per pass over
        the gradients (norms: one pass; SGD: read p, g, m and write p, m = five passes for both, the
        ATen chain adds a read and a write of g).
step:   llama2-7b-l4 (batch 4 x 2048, bf16, SGD-momentum, CUDA graph) with clip_grad_norm_(1.0),
        compiled with EDB_NATIVE_CLIP=0 and =1, two alternating runs each; each run checks the
        compiled losses against each other (same seeds, same model).
"""
import argparse
import dataclasses
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _time_ms(fn, iters):
    for _ in range(5):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def _cfg():
    from easydist_b200.workloads import LLAMA_CONFIGS
    return dataclasses.replace(LLAMA_CONFIGS["llama2-7b"], n_layer=4)


def kernels(iters):
    from easydist_b200 import clip, optim
    from easydist_b200.workloads import Llama
    with torch.device("meta"):
        shapes = [tuple(p.shape) for p in Llama(_cfg()).parameters()]
    bf = torch.bfloat16
    grads = [torch.randn(s, device="cuda", dtype=bf) * 1e-3 for s in shapes]
    params = [torch.randn(s, device="cuda", dtype=bf) for s in shapes]
    bufs = [torch.zeros(s, device="cuda", dtype=bf) for s in shapes]
    coef = torch.tensor(0.5, device="cuda", dtype=bf)
    numel = sum(g.numel() for g in grads)
    aten = torch.ops.aten
    # the values must agree before the times mean anything: the norms within one bf16 rounding of the
    # ATen norms (another fp32 summation order), the scaled SGD bit for bit
    ours, ref = clip.grad_norms(grads), torch.stack([aten.linalg_vector_norm(g, 2.0) for g in grads])
    assert torch.allclose(ours.float(), ref.float(), rtol=2 ** -7, atol=0), (ours, ref)
    p1, m1 = [p.clone() for p in params], [m.clone() for m in bufs]
    optim.sgd_momentum_(p1, grads, m1, 0.9, 1.0, -1e-3, grad_scale=coef)
    g2 = [g.clone() for g in grads]
    for g in g2:
        g.mul_(coef)
    p2, m2 = [p.clone() for p in params], [m.clone() for m in bufs]
    optim.sgd_momentum_(p2, g2, m2, 0.9, 1.0, -1e-3)
    assert all(torch.equal(a, b) for a, b in zip(p1 + m1, p2 + m2))
    del p1, m1, p2, m2, g2

    def aten_scale_sgd():
        for g in grads:
            g.mul_(coef)
        optim.sgd_momentum_(params, grads, bufs, 0.9, 1.0, -1e-3)

    cases = [
        ("grad_norms (edb_grad_sumsq NORM)", lambda: clip.grad_norms(grads), 1),
        ("ATen linalg_vector_norm x T + stack",
         lambda: torch.stack([aten.linalg_vector_norm(g, 2.0) for g in grads]), 1),
        ("sgd_momentum_(grad_scale=c)",
         lambda: optim.sgd_momentum_(params, grads, bufs, 0.9, 1.0, -1e-3, grad_scale=coef), 5),
        ("ATen mul_ x T + sgd_momentum_", aten_scale_sgd, 7),
    ]
    rows = []
    for name, fn, passes in cases:
        ms = _time_ms(fn, iters)
        nbytes = passes * numel * 2
        tbs = nbytes / ms / 1e9
        rows.append(dict(case=name, tensors=len(grads), elements=numel, algorithmic_bytes=nbytes,
                         us=round(ms * 1e3, 1), TBps=round(tbs, 3), of_3_35=round(tbs / 3.35, 3)))
    return rows


def step_run(native, iters, warmup):
    """One compiled llama2-7b-l4 step timing in this process (EDB_NATIVE_CLIP=native)."""
    os.environ["EDB_NATIVE_CLIP"] = "1" if native else "0"
    from easydist_b200.api import easydist_compile
    from easydist_b200.workloads import Llama, synthetic_tokens
    cfg = _cfg()

    def step(tokens, targets, model, opt):
        loss = model(tokens, targets)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 1.0)
        opt.step()
        opt.zero_grad(True)
        return loss

    torch.manual_seed(0)
    model = Llama(cfg).to(device="cuda", dtype=torch.bfloat16)
    opt = torch.optim.SGD(model.parameters(), lr=1e-4, momentum=0.9, foreach=True)
    compiled = easydist_compile(step, parallel_mode="zero3", tracing_mode="fake", cuda_graph=True)
    tok, tgt = synthetic_tokens(cfg, 4, 2048, 0, device="cuda")
    losses = [float(compiled(tok, tgt, model, opt)) for _ in range(warmup)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        loss = compiled(tok, tgt, model, opt)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) / iters * 1e3
    losses.append(float(loss))
    info = compiled.compiled_func.info
    return dict(native_clip=native, ms_per_step=round(ms, 2), clip_nodes=list(info["clip_nodes"]),
                losses=losses, peak_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--step-iters", type=int, default=10)
    ap.add_argument("--no-step", action="store_true")
    ap.add_argument("--step-child", type=int, default=None, help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU")
    from easydist_b200 import runtime
    from easydist_b200.device_mesh import set_device_mesh
    runtime.init(rank=0, world=1, device=0, heap_bytes=1 << 30)
    set_device_mesh([0], ["dp"], rank=0)
    if a.step_child is not None:
        print("STEP " + json.dumps(step_run(bool(a.step_child), a.step_iters, 3)), flush=True)
        return
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    res = dict(gpu=q, kernels=kernels(a.iters))
    if not a.no_step:
        runs = []
        for native in (0, 1, 0, 1):  # alternating, one process each
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--step-child", str(native),
                                "--step-iters", str(a.step_iters)], capture_output=True, text=True,
                               cwd=ROOT)
            line = next((x for x in r.stdout.splitlines() if x.startswith("STEP ")), None)
            if line is None:
                sys.exit(f"step run failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}")
            runs.append(json.loads(line[5:]))
        # parity: the same seeds and model give the same losses up to bf16 rounding of the norms
        ref = runs[0]["losses"]
        res["step_parity_ok"] = all(
            all(abs(x - y) <= 2e-2 * abs(y) for x, y in zip(r_["losses"], ref)) for r_ in runs)
        res["step"] = runs
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
