"""Per-call time of the embedding kernels (edb_embed.cu) against the ATen chains they replace, from
CUDA events over --iters calls after warm-up, as achieved TB/s over the algorithmic bytes.  The card's
name, power limit and SM clock are read in the same run.

    python tools/embed_bench.py [--iters 200] [--out results/embed.json]

Shapes:
  GPT-2 medium: 8 x 512 tokens, V 50257, C 1024, bf16, wte + wpe, tied LM head;
  Llama-2-7B:   4 x 2048 tokens, V 32000, C 4096, bf16, untied.
Cases and algorithmic bytes (N tokens, C, 2-byte elements):
  forward     : read N indexed rows (+ N position rows), write N rows: 2*N*C*2 (+ N*C*2);
  dense bwd   : read dy (N*C*2), write the [V, C] gradient (V*C*2);
  tied bwd    : GPT-2 only; kernel: read dy and read + write the indexed rows of the LM-head
                gradient (N*C*2 + 2*min(N, V)*C*2); ATen: embedding_dense_backward followed by the
                V x C add into a fresh tensor (the bytes of the kernel's form are used for both).
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
aten = torch.ops.aten


def _time_ms(fn, iters):
    for _ in range(10):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def _row(case, shape, nbytes, ms):
    tbs = nbytes / ms / 1e9
    return dict(case=case, shape=shape, algorithmic_bytes=nbytes, us=round(ms * 1e3, 2),
                TBps=round(tbs, 3))


def gpt2(iters):
    from easydist_b200 import embed
    B, T, V, C = 8, 512, 50257, 1024
    N, bf = B * T, torch.bfloat16
    W = (torch.randn(V, C, device="cuda") * 0.02).to(bf)
    P = (torch.randn(1024, C, device="cuda") * 0.02).to(bf)
    idx = torch.randint(0, V, (B, T), device="cuda")
    pos = torch.arange(T, device="cuda")
    dy = torch.randn(B, T, C, device="cuda").to(bf)
    lm = torch.randn(V, C, device="cuda").to(bf)
    acc = lm.clone()
    assert torch.equal(embed.embedding_fwd(W, idx, P, pos),
                       aten.add(aten.embedding(W, idx), aten.embedding(P, pos)))
    shape = f"B{B} T{T} V{V} C{C} bf16"
    hit = int(torch.unique(idx).numel())
    fb, bb, tb = 3 * N * C * 2, N * C * 2 + V * C * 2, N * C * 2 + 2 * hit * C * 2
    return [
        _row("edb_embedding_fwd (wte + wpe)", shape, fb,
             _time_ms(lambda: embed.embedding_fwd(W, idx, P, pos), iters)),
        _row("ATen embedding x2 + add", shape, fb,
             _time_ms(lambda: aten.add(aten.embedding(W, idx), aten.embedding(P, pos)), iters)),
        _row("edb_embedding_bwd_acc_ (tied, in place)", shape, tb,
             _time_ms(lambda: embed.embedding_bwd_acc_(acc, dy, idx, -1), iters)),
        _row("ATen embedding_dense_backward + add (tied)", shape, tb,
             _time_ms(lambda: aten.add(lm, aten.embedding_dense_backward(dy, idx, V, -1, False)),
                      iters)),
        _row("edb_embedding_bwd (dense)", shape, bb,
             _time_ms(lambda: embed.embedding_bwd(dy, idx, V, -1), iters)),
        _row("ATen embedding_dense_backward", shape, bb,
             _time_ms(lambda: aten.embedding_dense_backward(dy, idx, V, -1, False), iters)),
    ]


def llama(iters):
    from easydist_b200 import embed
    B, T, V, C = 4, 2048, 32000, 4096
    N, bf = B * T, torch.bfloat16
    W = (torch.randn(V, C, device="cuda") * 0.02).to(bf)
    idx = torch.randint(0, V, (B, T), device="cuda")
    dy = torch.randn(B, T, C, device="cuda").to(bf)
    shape = f"B{B} T{T} V{V} C{C} bf16"
    fb, bb = 2 * N * C * 2, N * C * 2 + V * C * 2
    return [
        _row("edb_embedding_fwd", shape, fb, _time_ms(lambda: embed.embedding_fwd(W, idx), iters)),
        _row("ATen embedding", shape, fb, _time_ms(lambda: aten.embedding(W, idx), iters)),
        _row("edb_embedding_bwd (dense)", shape, bb,
             _time_ms(lambda: embed.embedding_bwd(dy, idx, V, -1), iters)),
        _row("ATen embedding_dense_backward", shape, bb,
             _time_ms(lambda: aten.embedding_dense_backward(dy, idx, V, -1, False), iters)),
    ]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = dict(gpu=q, gpt2_medium=gpt2(a.iters), llama2_7b=llama(a.iters))
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
