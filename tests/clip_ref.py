"""Float64 reference and per-tensor error bound for the sum of squares of edb_grad_sumsq (edb_clip.cu).

The kernel splits every tensor into chunks of CE = 256 threads x 4 vectors x EPV elements (EPV = 8 for
bf16, 4 for fp32).  A thread adds its squares in sequence with fmaf (k <= 4*EPV + 1 terms: its vector
elements, plus one tail element in the last chunk); a CTA combines 256 thread sums in a 5-level
shuffle tree and then adds its 8 warp sums in order (7 additions).  The finish kernel does the same
with the P = ceil(numel / CE) chunk partials: ceil(P / 256) in sequence per thread, then 5 + 7.  So a
term passes through at most
    d = (4*EPV + 1) + 12 + ceil(P / 256) + 12
roundings of fp32 (unit e = 2^-24); x^2 itself is exact inside fmaf.  Every term is non-negative,
so the sum of their magnitudes is the exact sum S and
    |s - S| <= ((1 + e)^d - 1) * S <= (d + 1) * e * S."""
import math

import torch

F32_E = 2.0 ** -24
THREADS, UNROLL = 256, 4


def epv(dtype):
    return 8 if dtype == torch.bfloat16 else 4


def chunk_elems(dtype):
    return THREADS * UNROLL * epv(dtype)


def depth(numel, dtype):
    chunks = math.ceil(numel / chunk_elems(dtype))
    return (UNROLL * epv(dtype) + 1) + 12 + math.ceil(chunks / THREADS) + 12


def exact(t):
    """Sum of squares in float64."""
    x = t.detach().double()
    return float((x * x).sum())


def bound(t):
    return (depth(t.numel(), t.dtype) + 1) * F32_E * exact(t)


def worst(got, grads):
    """Largest |got_i - S_i| / bound_i over the list (<= 1 passes).  An all-zero tensor must give 0."""
    w = 0.0
    for s, g in zip(got.tolist(), grads):
        ref, b = exact(g), bound(g)
        err = abs(s - ref)
        w = max(w, err / b if b > 0 else (0.0 if err == 0 else math.inf))
    return w
