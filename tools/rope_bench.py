"""Per-call time of the RoPE kernel (edb_rope.cu) against the ATen chains it replaces, at the
Llama-2-7B attention shapes (B 4, T 2048, H 32, hd 128, bf16), from CUDA events, as achieved TB/s
over the algorithmic bytes and as a share of 3.35 TB/s.  The card's name and power limit are read
in the same run.

    python tools/rope_bench.py [--iters 100] [--out results/rope.json]

forward : the input is the transposed view of the [B, T, H*hd] projection output, as in the model;
          the output is the contiguous [B, H, T, hd] tensor attention reads.
backward: the input is the contiguous [B, H, T, hd] attention gradient; the output is the
          [B, T, H, hd] tensor the projection GEMMs read (kernel: written directly; ATen: the chain
          followed by transpose(1, 2) + clone).
Algorithmic bytes: one read of x and one write of y, 2*n*sizeof(bf16) per direction (the
[T, hd/2] tables stay in L2).
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


def _rotate_half_fwd(x, cos, sin):
    h = x.shape[-1] // 2
    c, s = torch.cat((cos, cos), -1), torch.cat((sin, sin), -1)
    return x * c + torch.cat((-x[..., h:], x[..., :h]), -1) * s


def kernels(B, T, H, hd, iters):
    from easydist_b200 import rope, workloads
    bf = torch.bfloat16
    x = torch.randn(B, T, H * hd, device="cuda").to(bf).view(B, T, H, hd).transpose(1, 2)
    dy = torch.randn(B, H, T, hd, device="cuda").to(bf)
    inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2, device="cuda").float() / hd))
    ang = torch.arange(T, device="cuda").float()[:, None] * inv[None, :]
    cos, sin = ang.cos().to(bf), ang.sin().to(bf)
    # the kernel must give the chains' bits at this shape before its time means anything
    assert torch.equal(rope.rope(x, cos, sin), workloads._rope(x, cos, sin))
    assert torch.equal(rope.rope(dy, cos, sin, True, transposed=True),
                       rope._chain(dy, cos, sin, True).transpose(1, 2).contiguous())
    nbytes = 2 * x.numel() * x.element_size()
    cases = [
        ("edb_rope forward", lambda: rope.rope(x, cos, sin)),
        ("ATen half-split forward", lambda: workloads._rope(x, cos, sin)),
        ("ATen rotate_half forward", lambda: _rotate_half_fwd(x, cos, sin)),
        ("edb_rope backward (to [B,T,H,hd])", lambda: rope.rope(dy, cos, sin, True, transposed=True)),
        ("ATen half-split backward + transpose/clone",
         lambda: rope._chain(dy, cos, sin, True).transpose(1, 2).contiguous()),
    ]
    rows = []
    for name, fn in cases:
        ms = _time_ms(fn, iters)
        tbs = nbytes / ms / 1e9
        rows.append(dict(case=name, shape=f"B{B} H{H} T{T} hd{hd} bf16", algorithmic_bytes=nbytes,
                         us=round(ms * 1e3, 2), TBps=round(tbs, 3), of_3_35=round(tbs / 3.35, 3)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
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
    res = dict(gpu=q, kernels=kernels(4, 2048, 32, 128, a.iters))
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
