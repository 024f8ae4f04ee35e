"""Float64 references and error bounds for the bf16 GEMM kernels (fp32 tensor-core accumulation,
one round-to-nearest to bf16 in the epilogue).

For a plain, bias or residual-add output the kernel returns c = bf16(acc), where acc is the fp32
accumulation of the exact bf16 products (plus bias and aux, added in fp32).  With r the exact result
and s the sum of the magnitudes of every term that entered it (s = |A| @ |B| + |bias| + |aux|):

    |c - r| <= 2^-8 * |r| + 2^-16 * s

  * 2^-8 |r| is one round-to-nearest to bf16 (8 significant bits: half an ulp is at most 2^-8 of
    the value).  Round-toward-zero can be off by a whole ulp, up to 2^-7 |r|, so it fails this term.
  * 2^-16 s covers the fp32 accumulation.  Each of the K/16 additions into the accumulator errs by
    at most 2^-23 of the running magnitude (<= s; tensor cores may truncate), so K <= 2048 is covered
    outright; beyond that the errors of random-sign data grow like a random walk (sqrt of the count)
    and stay far inside.  Dropping a 16-wide k-step, a partial k-block, a split-K slice or the bias
    changes c by O(sqrt(16) * rms(a*b)), i.e. O(1) against a bound of O(2^-8 sqrt(K) + 2^-16 K).

For a correct kernel the largest err / bound sits close to (but below) 1: the rounding term is tight
by construction, an element just above a power of two can round by almost exactly half an ulp.  The
margin the accumulation error needs shows in `excess`, the part of the error beyond the rounding
term as a share of the accumulation term, which stays far below 1.
"""
import math

import torch

U_BF16 = 2.0 ** -8     # unit roundoff of bf16, round-to-nearest
U_ACC = 2.0 ** -16     # fp32 accumulation (and fp32 epilogue adds), relative to s
EPS_GELU = 2.0 ** -20  # absolute error of the kernel's fp32 gelu'(x) (ex2.approx / rcp.approx)

_BETA = math.sqrt(2.0 / math.pi)
_KAPPA = 0.044715


def gelu_tanh_grad64(x):
    """d/dx of the tanh-approximated GeLU, in float64 (ATen's formula)."""
    x = x.double()
    t = torch.tanh(_BETA * (x + _KAPPA * x ** 3))
    return 0.5 * (1 + t) + 0.5 * x * (1 - t * t) * _BETA * (1 + 3 * _KAPPA * x * x)


def reference(A, B, bias=None, add=None, gelu_pre=None):
    """(r, bound) in float64 on A's device for the bf16 GEMM A[M,K] @ B[K,N] (any strides):

      plain / bias / add:  r = A @ B (+ bias) (+ add), bound = 2^-8 |r| + 2^-16 s  (module docstring)
      gelu_bwd:            r = (A @ B) * g with g = gelu'(gelu_pre) exact.  The kernel computes
                           c = bf16(fp32(bf16(p~) * g~)), p~ the fp32 accumulation (|p~ - p| <= e,
                           e = 2^-16 s) and g~ its fp32 gelu' (|g~ - g| <= EPS_GELU, absolute: g lies
                           in [-0.17, 1.13] and near its zero only an absolute bound holds).  With
                           P = |p| + e >= |p~| and G = |g| + EPS_GELU >= |g~|:
                             |bf16(p~) g~ - p g| <= |bf16(p~) - p| G + |p| |g~ - g|
                                                 <= (2^-8 P + e) G + EPS_GELU |p|            =: D
                           and the final rounding (fp32 product 2^-24, bf16 2^-8) adds
                           2^-8 (1 + 2^-16) (|r| + D), so
                             |c - r| <= 2^-8 |r| + (1 + 2^-7) D.
    """
    A64, B64 = A.double(), B.double()
    p = A64 @ B64
    s = A64.abs() @ B64.abs()
    if gelu_pre is not None:
        assert bias is None and add is None
        g = gelu_tanh_grad64(gelu_pre)
        r = p * g
        e = U_ACC * s
        D = (U_BF16 * (p.abs() + e) + e) * (g.abs() + EPS_GELU) + EPS_GELU * p.abs()
        return r, U_BF16 * r.abs() + (1 + 2.0 ** -7) * D
    r = p
    if bias is not None:
        r = r + bias.double()
        s = s + bias.double().abs()
    if add is not None:
        r = r + add.double()
        s = s + add.double().abs()
    return r, U_BF16 * r.abs() + U_ACC * s


def ratio(c, r, bound):
    """Largest |c - r| / bound (inf where the bound is 0 but c differs; NaN in c counts as inf)."""
    err = (c.double() - r).abs()
    q = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    q = torch.nan_to_num(q, nan=math.inf)
    return float(q.max())


def excess(c, r, A, B):
    """Largest share of the accumulation term 2^-16 |A| @ |B| that the error of a plain output needs
    beyond the rounding term 2^-8 |r| (<= 0 where the rounding term alone covers the error)."""
    s = A.double().abs() @ B.double().abs()
    err = (c.double() - r).abs()
    return float(((err - U_BF16 * r.abs()) / (U_ACC * s).clamp_min(1e-300)).max())
