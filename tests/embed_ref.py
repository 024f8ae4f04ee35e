"""Float64 reference, per-element error bound and an fp32 emulation of the embedding backward
(edb_embed.cu).

The kernel gives g[v] = T(s[v]), s[v] the fp32 sum of the k = k[v] rows dy[r] with idx[r] == v,
added one by one in increasing r onto 0.  Every term passes through at most k fp32 additions, so
|s - S| <= gamma(k) * sum|terms| with S the exact sum, and the final rounding to T adds u*|s|:
    |g - S| <= u*|S| + (1 + u) * gamma(k) * sum|terms|      (u = 2^-8 bf16, 2^-24 fp32).
The in-place mode returns T(fl32(acc + g)) for an acc of T: one more fp32 addition (e relative)
and one more rounding to T (u relative) of the value acc + g, hence
    |out - (acc + S)| <= (u + e) * |acc + S| + (1 + u) * (1 + e) * (bound of g),
terms of second order covered by a factor 1 + 2^-10."""
import torch

from tests.reduce_ref import F32_E, SECOND_ORDER, gamma, unit


def bwd_ref(dy, idx, V):
    """-> (S [V, C] float64 sums, A [V, C] sums of |terms|, k [V] number of terms); ids outside
    [0, V) contribute nothing."""
    C = dy.shape[-1]
    d64, ix = dy.double().reshape(-1, C), idx.reshape(-1).long()
    keep = (ix >= 0) & (ix < V)
    d64, ix = d64[keep], ix[keep]
    S = torch.zeros(V, C, dtype=torch.float64, device=dy.device).index_add_(0, ix, d64)
    A = torch.zeros(V, C, dtype=torch.float64, device=dy.device).index_add_(0, ix, d64.abs())
    k = torch.zeros(V, dtype=torch.float64, device=dy.device).index_add_(
        0, ix, torch.ones_like(ix, dtype=torch.float64))
    return S, A, k


def bwd_bound(S, A, k, dtype):
    u = unit(dtype)
    g = (k * F32_E / (1.0 - k * F32_E))[:, None]
    return u * S.abs() + (1 + u) * SECOND_ORDER * g * A + 1e-300


def acc_bound(acc, S, A, k, dtype):
    """Bound of the in-place mode against acc + S (acc: the tensor before the call)."""
    u, e = unit(dtype), F32_E
    tot = acc.double() + S
    return SECOND_ORDER * ((u + e) * tot.abs() + (1 + u) * (1 + e) * bwd_bound(S, A, k, dtype))


def worst(got, ref, bound, rows=None):
    """max |got - ref| / bound over the rows `rows` (default all): <= 1 passes."""
    r = ((got.double() - ref).abs() / bound)
    return float((r if rows is None else r[rows]).max())


def emulate(dy, idx, V, padding_idx=-1, dtype=None, acc=None, fault=None):
    """The kernel's arithmetic in fp32 on the host: per id, the rows in increasing r added onto 0,
    the sum rounded to dtype; acc given: T(acc + T(sum)) on the indexed rows.  `fault` seeds one
    error: "drop" (a term left out), "double" (a term added twice), "bf16_acc" (the running sum
    rounded to bf16 after every addition), "off_by_one" (one term sent to the next id) or "pad"
    (the padding row not zeroed)."""
    dtype = dtype or dy.dtype
    C = dy.shape[-1]
    d, ix = dy.float().reshape(-1, C), idx.reshape(-1).tolist()
    s = torch.zeros(V, C, dtype=torch.float32)
    hit = [False] * V
    victim = next(r for r, v in enumerate(ix) if 0 <= v < V and v != padding_idx)
    for r, v in enumerate(ix):
        if fault == "off_by_one" and r == victim:
            v = (v + 1) % V
        if not 0 <= v < V:
            continue
        if fault == "drop" and r == victim:
            continue
        s[v] += d[r]
        if fault == "double" and r == victim:
            s[v] += d[r]
        if fault == "bf16_acc":
            s[v] = s[v].bfloat16().float()
        hit[v] = True
    if 0 <= padding_idx < V and fault != "pad":
        s[padding_idx] = 0.0
        hit[padding_idx] = False
    g = s.to(dtype)
    if acc is None:
        return g
    out = acc.clone()
    rows = torch.tensor(hit)
    out[rows] = (acc[rows].float() + g[rows].float()).to(dtype)
    return out
