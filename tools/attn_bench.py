"""Per-call time and run-to-run repeatability of the attention kernels (edb_attn.cu) against ATen's
cuDNN attention (what SDPA traces to in the compiled H100 steps) and its flash attention
(FlashAttention-2), forward and backward, at the GPT-2 medium (B 8, H 16, T 512, hd 64) and
Llama-2-7B (B 4, H 32, T 2048, hd 128) attention shapes, causal, bf16, on the c_attn split views the
models hand them.  Every ATen backward is measured twice: as it runs by default and under
`torch.use_deterministic_algorithms(True)`, where ATen switches to its deterministic algorithms.
The card's name and power limit are read in the same run.

    python tools/attn_bench.py [--iters 50] [--out results/attn.json]

Times are kernel times: each call is captured once in a CUDA graph and the graph is replayed
`iters` times between CUDA events, so the host work of a call (dispatch checks, tensor maps,
allocations) is not in them.  `repeatable` runs the call 10 times on the same inputs and reports
whether every output was bit-identical to the first run's.

Causal FLOPs: the forward does 2 matmuls of 2·B·H·T²·hd over half the score matrix, 2·B·H·T²·hd
in all; the backward's five matmuls are 5·B·H·T²·hd (what FlashAttention reports).  The native
backward recomputes two more products for determinism; they are not counted.
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
aten = torch.ops.aten


@contextlib.contextmanager
def _deterministic(on):
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def _time_ms(fn, iters, det):
    with _deterministic(det):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(3):
                fn()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
    for _ in range(3):
        g.replay()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        g.replay()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def _results(r):
    """The results a call is judged by: (out, lse) of a forward (ATen's also return its RNG
    state, which moves between calls), every gradient of a backward."""
    return list(r[:2] if len(r) > 3 else r)


def _repeatable(fn, det):
    with _deterministic(det):
        first = [t.clone() for t in _results(fn())]
        for _ in range(9):
            got = _results(fn())
            if not all(torch.equal(a, b) for a, b in zip(first, got)):
                return False
    return True


def kernels(name, B, H, T, hd, iters):
    from easydist_b200 import attn
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(B, T, 3 * H * hd, device="cuda", generator=g).bfloat16()
    q, k, v = (t.view(B, T, H, hd).transpose(1, 2) for t in qkv.split(H * hd, dim=2))
    dout = torch.randn(B, H, T, hd, device="cuda", generator=g).bfloat16()
    r = aten._scaled_dot_product_flash_attention.default(q, k, v, 0.0, True)
    c = aten._scaled_dot_product_cudnn_attention.default(q, k, v, None, True, 0.0, True)
    out, lse = attn.attention_fwd(q, k, v, True)
    assert (out.float() - r[0].float()).abs().max() < 2e-2, "native forward disagrees with ATen"
    cudnn_bwd = lambda: aten._scaled_dot_product_cudnn_attention_backward.default(
        dout, q, k, v, c[0], c[1], c[6], c[7], None, None, None, T, T, 0.0, True)
    flash_bwd = lambda: aten._scaled_dot_product_flash_attention_backward.default(
        dout, q, k, v, r[0], r[1], r[2], r[3], r[4], r[5], 0.0, True, r[6], r[7])
    cases = [
        ("edb_attn forward", 2, lambda: attn.attention_fwd(q, k, v, True), False),
        ("ATen cuDNN forward", 2, lambda: aten._scaled_dot_product_cudnn_attention.default(
            q, k, v, None, True, 0.0, True), False),
        ("ATen flash forward", 2, lambda: aten._scaled_dot_product_flash_attention.default(
            q, k, v, 0.0, True), False),
        ("edb_attn backward", 5, lambda: attn.attention_bwd(dout, q, k, v, out, lse, True), False),
        ("ATen cuDNN backward", 5, cudnn_bwd, False),
        ("ATen cuDNN backward, deterministic", 5, cudnn_bwd, True),
        ("ATen flash backward", 5, flash_bwd, False),
        ("ATen flash backward, deterministic", 5, flash_bwd, True),
    ]
    rows = []
    for case, mults, fn, det in cases:
        ms = _time_ms(fn, iters, det)
        flops = mults * B * H * T * T * hd
        rows.append(dict(case=case, shape=f"{name}: B{B} H{H} T{T} hd{hd} bf16 causal",
                         us=round(ms * 1e3, 1), TFLOPs=round(flops / ms / 1e9, 1),
                         repeatable=_repeatable(fn, det)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("attn_bench needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    rows = kernels("GPT-2 medium", 8, 16, 512, 64, args.iters) \
        + kernels("Llama-2-7B", 4, 32, 2048, 128, args.iters)
    print(f"card: {card}")
    for r in rows:
        print(f"{r['shape']:48s} {r['case']:36s} {r['us']:9.1f} us {r['TFLOPs']:7.1f} TFLOP/s"
              f"  repeatable={r['repeatable']}")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=card, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
