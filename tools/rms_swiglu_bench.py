"""Per-kernel time of the RMSNorm and SwiGLU kernels (edb_rms.cu) at the Llama-2-7B shapes, from CUDA
events, as achieved GB/s over the algorithmic bytes; the peak memory of the compiled llama2-7b-l4 step
with the rewrites on and off; and what F.rms_norm traces to on CUDA tensors.

    python tools/rms_swiglu_bench.py [--tokens 8192] [--iters 50] [--out results/rms_swiglu.json]
"""
import argparse
import json
import os
import subprocess
import sys

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


def kernels(tokens, iters):
    from easydist_b200 import act, norm
    H, F = 4096, 11008
    bf = torch.bfloat16
    x = torch.randn(tokens, H, device="cuda").to(bf)
    w = torch.randn(H, device="cuda").to(bf)
    dy = torch.randn(tokens, H, device="cuda").to(bf)
    add = torch.randn(tokens, H, device="cuda").to(bf)
    gate = torch.randn(tokens, F, device="cuda").to(bf)
    up = torch.randn(tokens, F, device="cuda").to(bf)
    gdy = torch.randn(tokens, F, device="cuda").to(bf)
    _, rstd = norm.rms_norm_fwd(x, w, 1e-5, norm.RMS_CAST_THEN_SCALE)
    e = 2
    rows = []
    cases = [
        ("k_rms_fwd", f"{tokens}x{H}", 2 * tokens * H * e + tokens * 4,
         lambda: norm.rms_norm_fwd(x, w, 1e-5, norm.RMS_CAST_THEN_SCALE)),
        ("k_rms_bwd (+finish)", f"{tokens}x{H}", 3 * tokens * H * e + tokens * 4,
         lambda: norm.rms_norm_bwd(dy, x, rstd, w, norm.RMS_CAST_THEN_SCALE, [True, True])),
        ("k_rms_bwd _add (+finish)", f"{tokens}x{H}", 4 * tokens * H * e + tokens * 4,
         lambda: norm.rms_norm_bwd(dy, x, rstd, w, norm.RMS_CAST_THEN_SCALE, [True, True], _add=add)),
        ("k_swiglu_fwd", f"{tokens}x{F}", 3 * tokens * F * e, lambda: act.swiglu_fwd(gate, up)),
        ("k_swiglu_bwd", f"{tokens}x{F}", 5 * tokens * F * e, lambda: act.swiglu_bwd(gdy, gate, up)),
    ]
    for name, shape, nbytes, fn in cases:
        ms = _time_ms(fn, iters)
        gbs = nbytes / ms / 1e6
        rows.append(dict(kernel=name, shape=shape, bytes=nbytes, us=round(ms * 1e3, 2),
                         GBps=round(gbs, 1), of_3350=round(gbs / 3350, 3)))
    return rows


def rms_norm_trace():
    """Targets of the traced F.rms_norm step on CUDA tensors that mention rms / rsqrt."""
    from easydist_b200.compile import trace_train_step

    class M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.n = torch.nn.RMSNorm(256, eps=1e-5)

        def forward(self, x):
            return self.n(x).float().pow(2).mean()

    def step(x, model, opt):
        loss = model(x)
        loss.backward()
        opt.step()
        opt.zero_grad(True)
        return loss

    m = M().cuda().bfloat16()
    opt = torch.optim.SGD(m.parameters(), lr=0.1)
    gm = trace_train_step(step, (torch.randn(8, 256, device="cuda").bfloat16(), m, opt), {}, "fake")[3]
    return sorted({str(n.target) for n in gm.graph.nodes if n.op == "call_function"
                   and ("rms" in str(n.target) or "rsqrt" in str(n.target))})


def peak_memory(native):
    """max_memory_allocated of the compiled llama2-7b-l4 step (batch 4, seq 2048, ddp, 1 GPU) in a
    fresh process, with EDB_NATIVE_RMS / EDB_NATIVE_SWIGLU set to `native`."""
    code = (
        "import torch, json\n"
        "from easydist_b200 import runtime\n"
        "from easydist_b200.api import easydist_compile\n"
        "from easydist_b200.device_mesh import set_device_mesh\n"
        "from easydist_b200.workloads import LLAMA_CONFIGS, Llama, LlamaConfig, gpt2_train_step, "
        "synthetic_tokens\n"
        "import dataclasses\n"
        "runtime.init(rank=0, world=1, device=0, heap_bytes=2 << 30)\n"
        "set_device_mesh([0], ['dp'], rank=0)\n"
        "cfg = dataclasses.replace(LLAMA_CONFIGS['llama2-7b'], n_layer=4)\n"
        "torch.manual_seed(0)\n"
        "model = Llama(cfg).cuda().bfloat16()\n"
        "opt = torch.optim.SGD(model.parameters(), lr=1e-4, momentum=0.9, foreach=True)\n"
        "step = easydist_compile(gpt2_train_step, parallel_mode='ddp', tracing_mode='fake', "
        "cuda_graph=False)\n"
        "tok, tgt = synthetic_tokens(cfg, 4, 2048, 0)\n"
        "tok, tgt = tok.cuda(), tgt.cuda()\n"
        "step(tok, tgt, model, opt); torch.cuda.synchronize()\n"
        "torch.cuda.reset_peak_memory_stats()\n"
        "step(tok, tgt, model, opt); torch.cuda.synchronize()\n"
        "print(json.dumps(dict(peak_gib=torch.cuda.max_memory_allocated() / 2**30, "
        "info={k: step.compiled_func.info.get(k) for k in ('rms_norm_nodes', 'swiglu_nodes')})))\n")
    env = dict(os.environ, EDB_NATIVE_RMS=native, EDB_NATIVE_SWIGLU=native,
               PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    if r.returncode != 0:
        return {"error": r.stderr[-2000:]}
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU")
    from easydist_b200 import runtime
    from easydist_b200.device_mesh import set_device_mesh
    runtime.init(rank=0, world=1, device=0, heap_bytes=1 << 30)
    set_device_mesh([0], ["dp"], rank=0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    res = dict(gpu=q, kernels=kernels(a.tokens, a.iters), rms_norm_trace=rms_norm_trace(),
               peak_memory={"native": peak_memory("1"), "aten": peak_memory("0")})
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
