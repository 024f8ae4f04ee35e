"""Float64 reference and per-element error bounds for the RMSNorm kernels (edb_rms.cu).

The reference evaluates the kernel's formula in float64 and applies the mode's rounding points to T
in the same places: n^ = T(x*rstd) in RMS_CAST_THEN_SCALE, g = T(dy*w) likewise (exact in fp32 for
bf16 operands, so kernel and reference round the same value).  u = 2^-8 (bf16) or 2^-24 (f32) is the
unit roundoff of T, e = 2^-24 that of the fp32 arithmetic.

rstd.  The kernel sums x^2 in fp32: every thread adds its k = NV*EPV squares in sequence, a warp
combines 32 partials in a 5-level shuffle tree and WPR warps are added in order, so a term passes
through at most d = k + 5 + WPR additions (+1 for its own square).  For non-negative terms the
relative error of that sum is <= d*e; the division by H and the add of eps add e each, rsqrt halves
the relative error of its argument and rsqrtf adds at most 2 ulp (<= 2^-22 relative):
    |rstd - r64| <= eps_r * r64,   eps_r = (d + 3)/2 * e + 2^-22.

y.  y = T(n^ * w) (CAST) or T(x*rstd*w) (FUSED): the final rounding <= u*|y64|, the fp32 products and
the rstd error <= (2e + eps_r)*|x*r64*w|.  In CAST mode n^ itself may round the other way where
x*r64 lies within eps_r of a rounding boundary of T: there (and only there, `flip`) add one ulp of
n^ times |w|.

dx = T(add + rstd*(g - n*s)), s = mean(g*n), one rounding: u*|dx64| plus the fp32 evaluation.  s is a
sum with the depth d above: <= (d + 2)*e*A/H with A = sum|g*n|; n carries eps_r (so n*s carries
3*eps_r: rstd enters n, s and the factor), rstd*g carries eps_r; the last four fp32 operations add
4e of the magnitude M = rstd*(|g| + |n|*A/H) + |add|:
    |dx - dx64| <= u*|dx64| + ((d + 2)*e + 3*eps_r + 4*e) * M + e*|add|.

dw = T(sum_rows dy*n^): u*|dw64| plus an fp32 sum of `rows` terms whose depth is at most
D = (rows per CTA partial) + 4 + (partials per finish slice) + 8 <= rows + 12 + G/8, bounded here by
rows + 16 + 8*132/8 (at most 8 CTAs per SM on 132 SMs), times sum|dy*n^|; n^ carries eps_r (FUSED)
or flips by one ulp where `flip` (CAST):
    |dw - dw64| <= u*|dw64| + (D*e + eps_r) * sum|dy*n^| + sum_flip |dy| * ulp(n^).
"""
import torch

BF16_U, F32_E = 2.0 ** -8, 2.0 ** -24
CAST, FUSED = 0, 1


def unit(dtype):
    return BF16_U if dtype == torch.bfloat16 else F32_E


def kernel_config(H, dtype):
    """(WPR, NV) as edb_rms.cu's rms_config picks them."""
    nvec = H // (8 if dtype == torch.bfloat16 else 4)
    if nvec <= 32:
        return 1, 1
    if nvec <= 64:
        return 1, 2
    if nvec <= 128:
        return 1, 4
    for w in (2, 4, 8, 16):
        if nvec <= w * 32 * 4:
            return w, 4
    return 16, 8


def eps_rstd(H, dtype):
    wpr, nv = kernel_config(H, dtype)
    d = nv * (8 if dtype == torch.bfloat16 else 4) + 5 + wpr + 1
    return (d + 3) / 2 * F32_E + 2.0 ** -22, d


def ulp(v, dtype):
    """Spacing of T at |v| (bf16: 8 significant bits, f32: 24)."""
    bits = 8 if dtype == torch.bfloat16 else 24
    m = v.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(m)) - (bits - 1))


def rnd(v, dtype):
    return v.to(dtype).double()


def forward_ref(x, w, eps, mode):
    """-> (y64, r64, nhat64, flip) in float64 from T-valued x, w."""
    x64, w64 = x.double(), w.double()
    r64 = 1.0 / torch.sqrt((x64 * x64).mean(-1, keepdim=True) + eps)
    n64 = x64 * r64
    er, _ = eps_rstd(x.shape[-1], x.dtype)
    if mode == CAST:
        nhat = rnd(n64, x.dtype)
        flip = rnd(n64 * (1 - er), x.dtype) != rnd(n64 * (1 + er), x.dtype)
    else:
        nhat = n64
        flip = torch.zeros_like(n64, dtype=torch.bool)
    return nhat * w64, r64, nhat, flip


def forward_bound(x, w, y64, nhat, flip, mode):
    u = unit(x.dtype)
    er, _ = eps_rstd(x.shape[-1], x.dtype)
    w64 = w.double()
    b = u * y64.abs() + (2 * F32_E + er) * (nhat * w64).abs()
    if mode == CAST:
        b = b + flip * ulp(nhat, x.dtype) * w64.abs() * (1 + u)
    return b + 1e-300


def rstd_bound(x, r64):
    er, _ = eps_rstd(x.shape[-1], x.dtype)
    return er * r64


def backward_ref(dy, x, w, r64, mode, add=None):
    """-> (dx64, dw64, M, S) with M the dx magnitude term and S = sum_rows |dy*n^| per column."""
    H = x.shape[-1]
    x64, dy64, w64 = x.double(), dy.double(), w.double()
    n64 = x64 * r64
    g = dy64 * w64
    if mode == CAST:
        g = rnd(g, x.dtype)
        nhat = rnd(n64, x.dtype)
    else:
        nhat = n64
    s = (g * n64).sum(-1, keepdim=True) / H
    dx = r64 * (g - n64 * s)
    a = (g * n64).abs().sum(-1, keepdim=True)
    M = r64 * (g.abs() + n64.abs() * a / H)
    if add is not None:
        dx = dx + add.double()
        M = M + add.double().abs()
    red = tuple(range(x.dim() - 1))
    dw = (dy64 * nhat).sum(red)
    S = (dy64 * nhat).abs().sum(red)
    return dx, dw, M, S


def dx_bound(x, dx64, M, add=None):
    u = unit(x.dtype)
    er, d = eps_rstd(x.shape[-1], x.dtype)
    b = u * dx64.abs() + ((d + 2) * F32_E + 3 * er + 4 * F32_E) * M
    if add is not None:
        b = b + F32_E * add.double().abs()
    return b + 1e-300


def dw_bound(dy, x, dw64, S, flip, nhat, mode):
    u = unit(x.dtype)
    er, _ = eps_rstd(x.shape[-1], x.dtype)
    rows = dy.numel() // dy.shape[-1]
    D = rows + 16 + 8 * 132 // 8
    b = u * dw64.abs() + (D * F32_E + (er if mode == FUSED else 0.0)) * S
    if mode == CAST:
        red = tuple(range(x.dim() - 1))
        b = b + (flip * dy.double().abs() * ulp(nhat, x.dtype)).sum(red) * (1 + u)
    return b + 1e-300


def worst(got, ref, bound):
    """max |got - ref| / bound (<= 1 passes)."""
    return float(((got.double() - ref).abs() / bound).max())

