"""Float64 references and per-element error bounds for the reductions that end a GPT-2 step:
column sums (edb_colsum, every bias gradient), LayerNorm dw / db (k_ln_bwd partials +
k_ln_bwd_finish) and cross-entropy (edb_loss.cu).

Notation: T is the I/O dtype, u its unit roundoff (2^-8 bf16, 2^-24 fp32), e = 2^-24 that of the
fp32 arithmetic.  A value that passes through D fp32 roundings carries a relative error of at most
(1 + e)^D - 1 <= gamma(D) = D*e / (1 - D*e); a sum whose terms each pass through at most D additions
is off by at most gamma(D) * sum|terms|.  The final rounding of an fp32 value s to T adds u*|s|, and
|s| <= |s64| + |s - s64|, hence the common form
    |out - s64| <= u*|s64| + (1 + u) * (error of the fp32 value).

Column sums.  edb_colsum splits the rows into `splits` slices of `rps` rows (host rule copied in
`colsum_config`).  In a slice, each of 8 warps adds every 8th row in sequence (ceil(rps/8) additions
per lane), the 8 warp partials are added in order (8), the finish kernel adds every 8th slice partial
in sequence (ceil(splits/8)) and then its 8 slices in order (8):
    D = ceil(rps/8) + 8 + ceil(splits/8) + 8,
    |out - s64| <= u*|s64| + (1 + u) * gamma(D) * sum|x|.

LayerNorm dw / db.  The backward grid is persistent, grid = min(2*sms, ceil(rows/4)) CTAs of 4 warps;
warp w of CTA b takes rows b*4 + w + k*4*grid, so a lane adds at most ceil(rows/(4*grid)) rows in
sequence; the CTA adds its 4 warps (4), the finish kernel adds every 8th CTA partial
(ceil(grid/8)) and then 8 slices (8):
    D = ceil(rows/(4*grid)) + 4 + ceil(grid/8) + 8.
db is a plain sum of dy.  dw sums dy * xh with xh = (x - mean) * rstd evaluated in fp32 from the fp32
mean / rstd the kernel is given: two roundings for xh, one for the product, so every term of dw has
depth D + 3 relative to xh_in = (x - mean) * rstd in float64.  mean / rstd themselves are fp32
approximations of the exact statistics; the error that xh carries through them is exactly
xh_in - xh64 and enters dw as sum|dy| * |xh_in - xh64|:
    |db - db64| <= u*|db64| + (1 + u) * gamma(D) * sum|dy|,
    |dw - dw64| <= u*|dw64| + (1 + u) * (gamma(D + 3) * sum|dy*xh_in| + sum|dy|*|xh_in - xh64|).

Cross-entropy.  k_ce_fwd keeps per thread a running pair (m, s), m = fl(max(x) * L) in the log2
domain (L = fp32(log2 e)) and s = sum 2^fl(x*L - m) by ex2.approx.ftz.f32; when m grows, s is
rescaled by ex2(fl(m_old - m_new)).  A thread sees k elements in at most r vectors (16-byte path:
k = EPV*ceil(nvec/256) + [tail], r = ceil(nvec/256) + [tail]; scalar path: k = r = ceil(V/256)),
then 5 xor-shuffle merges and 7 sequential warp merges, each merge
s_a*ex2(m_a - m) + s_b*ex2(m_b - m).  The PTX ISA gives ex2.approx.f32 a maximum error of 2 ulp over
the full range, a relative error <= 2^-22 = 4e; results below 2^-126 flush to zero (.ftz).

  s.  Relative to S = sum_j 2^(x_j*L - M) in exact arithmetic (M the final m), a term gets 4e from
  its own ex2, at most k additions (e each), r in-thread rescales (ex2 + multiply: 5e) and 12 merges
  (ex2, multiply, add: 6e).  The exponent of a term is off by the rounding of fl(x*L - m) and of every
  fl(m_old - m_new) after it: <= e*(|x*L - m| + (M - m)) <= 3e*(x_max - x_j)*log2 e (+ e*|x_max|
  because fl(x*L) may exceed m by half an ulp), i.e. a relative error of 3e*(x_max - x_j) + 2e*|x_max|
  of the term.  Weighted by the terms, with E = sum_j p_j*(x_max - x_j) (p = softmax(x)):
      eps_s = e*(76 + k + 5r + 3E + 2|x_max|) + V*2^-125.
  lse.  l = fl(M*c + logf(s)), c = fp32(1/L).  The rounding of M cancels between M*c and S except
  through c - ln2 (<= 2e*ln2 relative): 2e*|x_max|.  L differs from log2 e by e relative, which
  scales x: e*|sum p_j x_j| <= e*(|x_max| + E).  logf is within 1 ulp (CUDA Programming Guide):
  2e*|ln s|.  The product M*c and the final add: e*|x_max| + e*|l|.  With ln s - ln S <=
  eps_s / (1 - eps_s):
      |l - lse64| <= eps_s/(1 - eps_s) + e*(4|x_max| + E + 2|lse64 - x_max| + |lse64|).
  loss.  row_loss = fl(l - x_t) adds e*|row_loss|.  k_ce_finish adds the row losses of every
  1024th row in sequence and then in a 10-level tree: depth ceil(rows/1024) + 10; the division by
  the (exact) count of non-ignored rows adds e*|loss|.
  dx.  p = ex2(fl(fma(x, L, nl))), nl = fl(-l*L).  Relative to p64 = exp(x - lse64) the argument is
  off by (log2 e times) the error of l, e*|l| from rounding nl, e*|x - l| from L and from the fma.
  The e*|l| term (6e-5 at a +1000 logit shift) is the price of an fp32 lse: forming x - l first, as
  ATen does, rounds the same fp32 l and errs by the same order (3e-5).  So
      p_rel = B_lse + e*|lse64| + 2e*|x - lse64| + 4e (ex2).
  Then v = p*c or fma(p, c, -c) and c = fl(grad_out / count) under mean: 2e*|dx64|; flushed p and
  subnormal T values: an absolute 2^-125*|c| + 2^-132.
      |dx - dx64| <= u*|dx64| + (1 + u) * (|c|*p64*p_rel + 2e*|dx64|) + 2^-125*|c| + 2^-132.
Terms of second order in e (products of two first-order terms, below 2^-10 of them for every input
used here) are covered by multiplying the fp32 error terms by 1 + 2^-10.
"""
import math

import torch

BF16_U, F32_E = 2.0 ** -8, 2.0 ** -24
SECOND_ORDER = 1.0 + 2.0 ** -10
CE_THREADS = 256
LOG2E_F32 = float(torch.tensor(math.log2(math.e), dtype=torch.float32))
H100_SMS = 132


def unit(dtype):
    return BF16_U if dtype == torch.bfloat16 else F32_E


def epv(dtype):
    """Elements per 16-byte vector."""
    return 8 if dtype == torch.bfloat16 else 4


def gamma(depth):
    return depth * F32_E / (1.0 - depth * F32_E)


def worst(got, ref, bound):
    """max |got - ref| / bound (<= 1 passes)."""
    return float(((got.double() - ref).abs() / bound).max())


# ---- column sums --------------------------------------------------------------------------------

def colsum_config(rows, cols, dtype, sms):
    """(splits, rows per split) as edb_colsum's host code picks them."""
    stripes = -(-cols // (32 * epv(dtype)))
    splits = min(-(-4 * sms // stripes), 128)
    if splits > rows // 64:
        splits = rows // 64 if rows // 64 > 0 else 1
    splits = max(splits, 1)
    rps = -(-rows // splits)
    return -(-rows // rps), rps


def colsum_depth(rows, cols, dtype, sms):
    splits, rps = colsum_config(rows, cols, dtype, sms)
    return -(-rps // 8) + 8 + -(-splits // 8) + 8


def colsum_ref(x):
    """-> (s64, sum|x|) per column of a [rows, cols] tensor."""
    x64 = x.double()
    return x64.sum(0), x64.abs().sum(0)


def colsum_bound(s64, A, depth, dtype):
    u = unit(dtype)
    return u * s64.abs() + (1 + u) * SECOND_ORDER * gamma(depth) * A + 1e-300


# ---- LayerNorm dw / db --------------------------------------------------------------------------

def ln_grid(rows, sms):
    return min(2 * sms, -(-rows // 4))


def ln_depth(rows, sms):
    grid = ln_grid(rows, sms)
    return -(-rows // (4 * grid)) + 4 + -(-grid // 8) + 8


def ln_dwdb_ref(dy, x, mean, rstd, eps):
    """-> (dw64, db64, Sw, Sb, Dx): dw64 / db64 from the exact statistics of x, Sw = sum|dy*xh_in|
    and Sb = sum|dy| per column, Dx = sum|dy|*|xh_in - xh64| (xh_in from the fp32 mean / rstd)."""
    H = x.shape[-1]
    x64, dy64 = x.double().reshape(-1, H), dy.double().reshape(-1, H)
    mu = x64.mean(-1, keepdim=True)
    r64 = ((x64 - mu) ** 2).mean(-1, keepdim=True).add(eps).rsqrt()
    xh64 = (x64 - mu) * r64
    xh_in = (x64 - mean.double().reshape(-1, 1)) * rstd.double().reshape(-1, 1)
    return ((dy64 * xh64).sum(0), dy64.sum(0), (dy64 * xh_in).abs().sum(0), dy64.abs().sum(0),
            (dy64.abs() * (xh_in - xh64).abs()).sum(0))


def ln_dw_bound(dw64, Sw, Dx, depth, dtype):
    u = unit(dtype)
    return u * dw64.abs() + (1 + u) * (SECOND_ORDER * gamma(depth + 3) * Sw + Dx) + 1e-300


def ln_db_bound(db64, Sb, depth, dtype):
    return colsum_bound(db64, Sb, depth, dtype)


# ---- cross-entropy ------------------------------------------------------------------------------

def ce_vec_fwd(x):
    """True when k_ce_fwd takes its 16-byte path for this logits view."""
    return x.stride(0) % epv(x.dtype) == 0 and x.data_ptr() % 16 == 0


def ce_thread_counts(vocab, dtype, vec):
    """(k elements, r vectors) one thread of k_ce_fwd reads at most."""
    if not vec:
        k = -(-vocab // CE_THREADS)
        return k, k
    n = epv(dtype)
    steps = -(-(vocab // n) // CE_THREADS)
    tail = 1 if vocab % n else 0
    return n * steps + tail, steps + tail


def ce_ref(x, target, ignore_index, reduction, grad_out):
    """Float64 cross-entropy of T-valued logits x [rows, vocab]: a dict with the per-row lse64,
    row_loss64 and bound inputs (x_max, E), the reduced loss64, the count of counted rows, the
    per-row gradient scale c64 and dx64 = c64 * (softmax - onehot)."""
    x64 = x.double()
    rows, vocab = x64.shape
    xmax = x64.max(1).values
    lse = torch.logsumexp(x64, 1)
    p = torch.exp(x64 - lse[:, None])
    gap = torch.where(p > 0, xmax[:, None] - x64, torch.zeros_like(x64))
    E = (p * gap).sum(1)
    keep = target != ignore_index
    tc = target.clamp(0, vocab - 1)
    xt = x64.gather(1, tc[:, None])[:, 0]
    rl = torch.where(keep, lse - xt, torch.zeros_like(lse))
    count = int(keep.sum())
    loss = rl.sum() / count if reduction == 1 else rl.sum()
    c = grad_out / max(count, 1) if reduction == 1 else grad_out  # no row is counted: all c are 0
    c = torch.where(keep, torch.full_like(lse, c), torch.zeros_like(lse))
    onehot = torch.zeros_like(x64)
    onehot.scatter_(1, tc[:, None], 1.0)
    dx = c[:, None] * (p - onehot * keep[:, None])
    return dict(lse=lse, xmax=xmax, E=E, row_loss=rl, loss=loss, count=count, c=c, p=p, dx=dx,
                vocab=vocab, rows=rows, keep=keep)


def ce_lse_bound(ref, dtype, vec):
    k, r = ce_thread_counts(ref["vocab"], dtype, vec)
    e, xm, E, lse = F32_E, ref["xmax"].abs(), ref["E"], ref["lse"]
    eps_s = e * (76 + k + 5 * r + 3 * E + 2 * xm) + ref["vocab"] * 2.0 ** -125
    b = eps_s / (1 - eps_s) + e * (4 * xm + E + 2 * (lse - ref["xmax"]).abs() + lse.abs())
    return SECOND_ORDER * b


def ce_row_loss_bound(ref, dtype, vec):
    b = ce_lse_bound(ref, dtype, vec) * (1 + F32_E) + F32_E * ref["row_loss"].abs()
    return torch.where(ref["keep"], SECOND_ORDER * b, torch.zeros_like(b)) + 1e-300


def ce_loss_bound(ref, dtype, vec, reduction):
    brl = ce_row_loss_bound(ref, dtype, vec)
    depth = -(-ref["rows"] // 1024) + 10
    b = brl.sum() + gamma(depth) * (ref["row_loss"].abs() + brl).sum()
    if reduction == 1:
        b = b / ref["count"] + F32_E * abs(float(ref["loss"]))
    return SECOND_ORDER * float(b) + 1e-300


def ce_dx_bound(ref, dtype, vec):
    u, e = unit(dtype), F32_E
    lse = ref["lse"][:, None]
    p_rel = ce_lse_bound(ref, dtype, vec)[:, None] + e * lse.abs() + 4 * e
    c = ref["c"].abs()[:, None]
    x_lse = (torch.log(ref["p"])).abs()  # |x - lse64|, inf where p == 0 (multiplied by p = 0 below)
    err = c * ref["p"] * (p_rel + 2 * e * torch.where(ref["p"] > 0, x_lse, torch.zeros_like(x_lse)))
    err = SECOND_ORDER * (err + 2 * e * ref["dx"].abs())
    return u * ref["dx"].abs() + (1 + u) * err + 2.0 ** -125 * c + 2.0 ** -132
