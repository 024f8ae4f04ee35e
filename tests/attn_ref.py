"""Float64 reference and error bounds for scaled-dot-product attention (edb_attn.cu), forward and
backward, and a float32 emulation of the kernels' arithmetic in their order.

The bounds follow the kernels' rounding points: S = q·kᵀ accumulated in fp32, P rounded to bf16
before P·V (forward), before dO (dV) and before dS; dS rounded to bf16; D = rowsum(dO∘O) from the
bf16 O; fp32 accumulation over the keys or queries; outputs rounded to bf16.  Each term is the
worst case of its rounding, summed with absolute values, and the total is doubled."""
import math

import torch

U = 2.0 ** -8    # bf16 relative rounding (one ulp, twice the half-ulp of round-to-nearest)
E = 2.0 ** -23   # fp32 relative rounding, with the same margin


def reference(q, k, v, dout, causal, scale=None):
    """Float64 (out, lse, dq, dk, dv) and the intermediates the bounds need."""
    q, k, v = (t.detach().double() for t in (q, k, v))
    T, hd = q.shape[-2], q.shape[-1]
    scale = hd ** -0.5 if scale is None else scale
    s = scale * (q @ k.transpose(-1, -2))
    if causal:
        s = s.masked_fill(torch.ones(T, T, dtype=torch.bool, device=q.device).triu(1), float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    out = p @ v
    d = None if dout is None else dout.double()
    r = dict(out=out, lse=lse, p=p, scale=scale, q=q, k=k, v=v)
    if d is not None:
        dp = d @ v.transpose(-1, -2)
        D = (d * out).sum(-1)
        ds = p * (dp - D[..., None])
        r.update(dout=d, dp=dp, D=D, ds=ds, dq=scale * ds @ k, dk=scale * ds.transpose(-1, -2) @ q,
                 dv=p.transpose(-1, -2) @ d)
    return r


def _dp_err(r):
    """Bound on |ΔP| from the fp32 S and the fp32 logsumexp."""
    hd, T = r["q"].shape[-1], r["q"].shape[-2]
    es = (hd + 4) * E * r["scale"] * (r["q"].abs() @ r["k"].abs().transpose(-1, -2))
    return r["p"] * (2 * es + (T + 8) * E)


def fwd_bound(r):
    T = r["q"].shape[-2]
    p, av = r["p"], r["v"].abs()
    return 2 * (((U + T * E) * p + _dp_err(r)) @ av + U * r["out"].abs()) + 1e-30


def bwd_bound(r):
    """(dq, dk, dv) bounds."""
    T, hd = r["q"].shape[-2], r["q"].shape[-1]
    p, dpe = r["p"], _dp_err(r)
    ad, aq, ak, av = r["dout"].abs(), r["q"].abs(), r["k"].abs(), r["v"].abs()
    e_p = (U + T * E) * p + dpe
    dv = e_p.transpose(-1, -2) @ ad + U * r["dv"].abs()
    e_D = (U + hd * E) * (ad * r["out"].abs()).sum(-1) + hd * E * ad.sum(-1) * av.max()
    e_dp = (hd + 2) * E * (ad @ av.transpose(-1, -2))
    ads = e_p * (r["dp"] - r["D"][..., None]).abs() + p * (e_D[..., None] + e_dp) + U * r["ds"].abs()
    acc = T * E * r["scale"]
    dq = r["scale"] * ads @ ak + acc * r["ds"].abs() @ ak + U * r["dq"].abs()
    dk = r["scale"] * ads.transpose(-1, -2) @ aq + acc * r["ds"].abs().transpose(-1, -2) @ aq \
        + U * r["dk"].abs()
    return 2 * dq + 1e-30, 2 * dk + 1e-30, 2 * dv + 1e-30


def _bf(x):
    return x.to(torch.bfloat16).float()


def emulate(q, k, v, dout, causal, scale=None, fault=None, block=128):
    """The kernels' arithmetic in fp32, in their order, on bf16-valued inputs: the online softmax over
    key blocks of `block` (128, the forward kernel's; exp2 of scale·log2e-scaled scores), P rounded to bf16 before P·V, O
    rounded to bf16, lse in natural log; the backward from that O and lse with P and dS rounded to
    bf16.  `fault` seeds one defect: "mask" (causal mask off by one), "scale" (1/hd instead of
    1/sqrt(hd)), "lse" (logsumexp off by 0.05), "no_D" (dS without the D term), "tail" (the
    partial last key block dropped).  Returns (out, lse, dq, dk, dv) as float64."""
    q, k, v, d = (t.float() for t in (q, k, v, dout))
    T, hd = q.shape[-2], q.shape[-1]
    scale = hd ** -0.5 if scale is None else scale
    if fault == "scale":
        scale = 1.0 / hd
    sl2 = scale * math.log2(math.e)
    shift = 1 if fault == "mask" else 0
    cols = torch.arange(T)
    n_keys = T - T % block if fault == "tail" and T % block else T
    m = torch.full(q.shape[:-1], float("-inf"))
    l = torch.zeros(q.shape[:-1])
    o = torch.zeros(q.shape)
    for n0 in range(0, n_keys, block):
        n1 = min(n0 + block, n_keys)
        s = q @ k[..., n0:n1, :].transpose(-1, -2)
        if causal:
            s = s.masked_fill(cols[n0:n1][None, :] > cols[:, None] + shift, float("-inf"))
        mx = torch.maximum(m, s.amax(-1))
        base = torch.where(mx == float("-inf"), torch.zeros_like(mx), mx * sl2)
        alpha = torch.exp2(m * sl2 - base)
        p = torch.exp2(s * sl2 - base[..., None])
        l = l * alpha + p.sum(-1)
        o = o * alpha[..., None] + _bf(p) @ v[..., n0:n1, :]
        m = mx
    out = _bf(o / l[..., None])
    lse = (m * sl2 + torch.log2(l)) * math.log(2)
    if fault == "lse":
        lse = lse + 5e-2
    s = q @ k.transpose(-1, -2)
    if causal:
        s = s.masked_fill(cols[None, :] > cols[:, None] + shift, float("-inf"))
    if fault == "tail" and n_keys < T:
        s[..., n_keys:] = float("-inf")
    p = _bf(torch.exp2(s * sl2 - (lse * math.log2(math.e))[..., None]))
    D = (d * out).sum(-1)
    dp = d @ v.transpose(-1, -2)
    ds = _bf(p * (dp - (0 if fault == "no_D" else D[..., None])))
    dq = _bf(scale * (ds @ k))
    dk = _bf(scale * (ds.transpose(-1, -2) @ q))
    dv = _bf(p.transpose(-1, -2) @ d)
    return tuple(t.double() for t in (out, lse, dq, dk, dv))


def inputs(B, H, T, hd, seed, layout="contiguous", device="cpu"):
    """bf16 q, k, v, dout [B, H, T, hd] in one of the layouts a traced graph hands the kernels:
    "contiguous", "split" (the c_attn split views of a [B, T, 3 H hd] projection), "transposed"
    (views of [B, T, H, hd] buffers), "offset" (a storage offset of 8 elements)."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, generator=g)
    if layout == "split":
        qkv = rnd(B, T, 3 * H * hd).to(torch.bfloat16).to(device)
        q, k, v = (t.view(B, T, H, hd).transpose(1, 2) for t in qkv.split(H * hd, dim=2))
    elif layout == "transposed":
        q, k, v = (rnd(B, T, H, hd).to(torch.bfloat16).to(device).transpose(1, 2) for _ in range(3))
    elif layout == "offset":
        q, k, v = (rnd(B * H * T * hd + 8).to(torch.bfloat16).to(device)[8:].view(B, H, T, hd)
                   for _ in range(3))
    else:
        q, k, v = (rnd(B, H, T, hd).to(torch.bfloat16).to(device) for _ in range(3))
    dout = rnd(B, H, T, hd).to(torch.bfloat16).to(device)
    return q, k, v, dout
