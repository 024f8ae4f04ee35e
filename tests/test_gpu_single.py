"""Single-GPU parity tests (H100): every call goes through the C-ABI (ctypes -> libedb.so).
  * local reshard ops and n=1 collectives vs the oracle (bit-exact)
  * wgmma GEMM vs a plain PyTorch fp32 reference (floating point: tolerance stated below)
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rt():
    from easydist_b200 import runtime
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    r = runtime.init(rank=0, world=1, device=0, heap_bytes=2 << 30) \
        if not runtime.is_initialized() else runtime.get_runtime()
    return r


def _np(t):
    return t.float().cpu().numpy() if t.dtype in (torch.bfloat16, torch.float16) else t.cpu().numpy()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.int64, torch.uint8])
def test_scatter_matches_oracle(rt, dtype):
    from easydist_b200 import reshard
    from oracle import reshard_oracle as O
    rng = np.random.RandomState(0)
    for shape, dim, n in [((8, 6, 10), 0, 2), ((8, 6, 10), 1, 3), ((8, 6, 10), 2, 4), ((7,), 0, 3),
                          ((5, 4096), 1, 8), ((4, 128, 1024), 2, 4), ((9, 2), 0, 4), ((0, 4), 0, 2)]:
        x = rng.randint(0, 100, size=shape).astype(np.float32)
        xt = torch.from_numpy(x).cuda().to(dtype)
        pieces = O.chunk(x, n, dim)
        for i in range(len(pieces)):
            got = reshard.scatter_wrapper(xt, n, dim, i)
            assert np.array_equal(_np(got), O.scatter(x, n, dim, i)), (shape, dim, n, i)
        if len(pieces) < n:
            with pytest.raises(IndexError):
                reshard.scatter_wrapper(xt, n, dim, n - 1)


def test_copy_wrapper(rt):
    from easydist_b200 import reshard
    for n in (1, 17, 4096, 1000003):
        a = torch.zeros(n, device="cuda")
        b = torch.randn(n, device="cuda")
        assert reshard.copy_wrapper(a, b) is a
        assert torch.equal(a, b)
    a = torch.zeros(4, 4, device="cuda", dtype=torch.float32)
    b = torch.ones(4, device="cuda", dtype=torch.bfloat16)
    reshard.copy_wrapper(a, b)  # broadcasting + cast goes through aten.copy_
    assert torch.equal(a, torch.ones(4, 4, device="cuda"))


def test_collectives_world1_are_identities(rt):
    from easydist_b200 import reshard
    g = [0]
    for dtype in (torch.float32, torch.bfloat16, torch.int64):
        x = torch.randint(-8, 9, (4, 6, 8), device="cuda").to(dtype)
        for d in range(3):
            assert torch.equal(reshard.all_gather_start(x, d, g), x)
            assert torch.equal(reshard.reduce_scatter_start(x, "sum", d, g), x)
        assert torch.equal(reshard.all_reduce_start(x, "sum", g), x)
        assert torch.equal(reshard.all_reduce_start(x, "max", g), x)
        assert torch.equal(reshard.all_to_all_start(x, 0, 2, 1, 0, g), x)
    xb = torch.randint(-8, 9, (16, 64), device="cuda").bfloat16()
    y = reshard.reduce_scatter_start(xb, "sum", 1, g, _scale=0.25, _out_dtype=torch.float32)
    assert torch.equal(y, xb.float() * 0.25)


def test_box_copy_general_strides(rt):
    """Strided N-D boxes (Partition boxes, sharding.py:427-446) vs numpy slicing."""
    from easydist_b200._lib import check, i64_array
    rng = np.random.RandomState(1)
    src = rng.randint(0, 1000, size=(6, 10, 14)).astype(np.int32)
    s = torch.from_numpy(src).cuda()
    for (lo, ext) in [((1, 2, 3), (4, 5, 6)), ((0, 0, 0), (6, 10, 14)), ((5, 9, 13), (1, 1, 1)),
                      ((0, 3, 0), (6, 2, 14)), ((2, 0, 1), (3, 10, 9))]:
        d = torch.zeros(ext, dtype=torch.int32, device="cuda")
        sstr = [st * 4 for st in s.stride()]
        dstr = [st * 4 for st in d.stride()]
        off = sum(l * st for l, st in zip(lo, sstr))
        check(rt.lib.edb_box_copy_local(d.data_ptr(), i64_array(dstr), s.data_ptr() + off,
                                        i64_array(sstr), i64_array(ext), 3, 4, rt.stream()))
        want = src[lo[0]:lo[0] + ext[0], lo[1]:lo[1] + ext[1], lo[2]:lo[2] + ext[2]]
        assert np.array_equal(d.cpu().numpy(), want), (lo, ext)


# GEMM accuracy across layouts, tile widths and shapes: tests/test_gpu_kernel_sweep.py (fp64 bound)


def test_gemm_exact_on_integer_inputs(rt):
    """Size-independent property: small-integer operands make every product and partial sum
    exactly representable, so the result must equal the fp32 reference bit for bit."""
    from easydist_b200 import gemm
    torch.manual_seed(1)
    for (M, N, K) in [(4096, 1024, 1024), (256, 4096, 512), (1024, 1024, 2048)]:  # last: split-K
        A = torch.randint(-1, 2, (M, K), device="cuda").bfloat16()
        B = torch.randint(-1, 2, (K, N), device="cuda").bfloat16()
        c = gemm.mm(A, B.t().contiguous().t())
        ref = (A.float() @ B.float())
        assert float(ref.abs().max()) < 256  # representable in bf16
        assert torch.equal(c.float(), ref)


def test_gemm_unaligned_extents_run_natively(rt):
    """Leading dimensions that break TMA's 16-byte stride rule (vocab 50257 of the GPT-2 LM head)
    are handled by padded staging, not by falling back to cuBLAS: forward (N unaligned), dgrad
    (K unaligned, A row stride unaligned) and wgrad (M unaligned, A column-major)."""
    from easydist_b200 import gemm
    torch.manual_seed(2)
    V, H, T = 50257, 256, 384
    x = torch.randn(T, H, device="cuda", dtype=torch.bfloat16)
    W = (torch.randn(V, H, device="cuda") * 0.05).bfloat16()
    dl = (torch.randn(T, V, device="cuda") * 0.05).bfloat16()

    def close(c, ref):
        err = (c.float() - ref).abs()
        return bool((err <= ref.abs() * 2 ** -7 + 2e-2).all())

    gemm.reset_stats()
    logits = gemm.mm(x, W.t())                     # [T,V] = x @ W^T
    assert logits.shape == (T, V) and close(logits, x.float() @ W.float().t())
    dx = gemm.mm(dl, W)                            # [T,H] = dl @ W      (K = 50257)
    assert close(dx, dl.float() @ W.float())
    dW = gemm.mm(dl.t(), x)                        # [V,H] = dl^T @ x    (M = 50257, A col-major)
    assert close(dW, dl.float().t() @ x.float())
    st = gemm.stats()
    assert st["edb_gemm"] == 3 and st["aten_mm"] == 0 and st["padded_operands"] >= 2, st
    # small odd sizes
    A = torch.randn(64, 50, device="cuda", dtype=torch.bfloat16)
    B = torch.randn(50, 24, device="cuda", dtype=torch.bfloat16)
    assert close(gemm.mm(A, B), A.float() @ B.float())


def test_addmm_bias_fused_in_epilogue(rt):
    from easydist_b200 import gemm
    torch.manual_seed(3)
    for (M, N, K) in [(256, 512, 128), (4096, 3072, 1024), (100, 72, 40), (512, 1024, 4096)]:
        a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
        w = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
        bias = torch.randn(N, device="cuda", dtype=torch.bfloat16)
        gemm.reset_stats()
        c = gemm.addmm(bias, a, w.t())
        assert gemm.stats()["edb_gemm"] == 1
        ref = a.float() @ w.float().t() + bias.float()
        err = (c.float() - ref).abs()
        assert bool((err <= ref.abs() * 2 ** -7 + 2e-2).all()), (M, N, K, float(err.max()))


def test_non_bf16_goes_to_aten(rt):
    from easydist_b200 import gemm
    A = torch.randn(64, 48, device="cuda")
    B = torch.randn(48, 24, device="cuda")
    gemm.reset_stats()
    c = gemm.mm(A, B)
    assert gemm.stats()["aten_mm"] == 1 and gemm.stats()["edb_gemm"] == 0
    assert torch.allclose(c, A @ B, atol=1e-4, rtol=1e-4)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_layer_norm_kernels_match_aten(rt, dtype):
    """edb_layer_norm_fwd/bwd vs aten.native_layer_norm(_backward) in fp32 on the same inputs.
    fp32: rtol 1e-5 (the north star's fp tolerance); bf16 I/O: one bf16 ulp on the outputs."""
    from easydist_b200 import norm
    aten = torch.ops.aten
    torch.manual_seed(4)
    for rows, H in [(4096, 1024), (37, 256), (1000, 768), (5, 2048 if dtype == torch.bfloat16 else 1024)]:
        x = torch.randn(rows, H, device="cuda", dtype=dtype)
        w = (torch.randn(H, device="cuda") * 0.5 + 1).to(dtype)
        b = torch.randn(H, device="cuda").to(dtype)
        dy = torch.randn(rows, H, device="cuda", dtype=dtype)
        norm.reset_stats()
        y, mean, rstd = norm.native_layer_norm(x.view(1, rows, H), [H], w, b, 1e-5)
        dx, dw, db = norm.native_layer_norm_backward(dy.view(1, rows, H), x.view(1, rows, H), [H],
                                                     mean, rstd, w, b, [True, True, True])
        assert norm.stats()["edb_ln_fwd"] == 1 and norm.stats()["edb_ln_bwd"] == 1, norm.stats()
        xf, wf, bf, dyf = x.float(), w.float(), b.float(), dy.float()
        ry, rmean, rrstd = aten.native_layer_norm.default(xf.view(1, rows, H), [H], wf, bf, 1e-5)
        rdx, rdw, rdb = aten.native_layer_norm_backward.default(
            dyf.view(1, rows, H), xf.view(1, rows, H), [H], rmean, rrstd, wf, bf, [True, True, True])
        assert mean.shape == rmean.shape and rstd.shape == rrstd.shape
        assert torch.allclose(mean, rmean, rtol=1e-5, atol=1e-6)
        assert torch.allclose(rstd, rrstd, rtol=1e-5, atol=1e-6)
        if dtype == torch.float32:
            tol = dict(rtol=1e-5, atol=1e-5)
            red_tol = dict(rtol=1e-4, atol=1e-4 * rows ** 0.5)
        else:
            tol = dict(rtol=2 ** -7, atol=2e-2)
            red_tol = dict(rtol=2 ** -6, atol=0.05 * rows ** 0.5)
        assert torch.allclose(y.float(), ry, **tol), (rows, H, float((y.float() - ry).abs().max()))
        assert torch.allclose(dx.float(), rdx, **tol), (rows, H, float((dx.float() - rdx).abs().max()))
        assert torch.allclose(dw.float(), rdw, **red_tol), (rows, H, float((dw.float() - rdw).abs().max()))
        assert torch.allclose(db.float(), rdb, **red_tol), (rows, H, float((db.float() - rdb).abs().max()))
    # unsupported width goes to ATen
    x = torch.randn(8, 100, device="cuda", dtype=dtype)
    norm.reset_stats()
    norm.native_layer_norm(x, [100], torch.ones(100, device="cuda", dtype=dtype), None, 1e-5)
    assert norm.stats()["aten_ln"] == 1


def test_colsum_matches_fp32_reference(rt):
    """edb_colsum (bias gradients) vs an fp32 column sum; fp32 accumulation in both, so only the
    final rounding to the I/O dtype differs: 1 ulp of bf16 / 1e-5 relative for fp32."""
    from easydist_b200 import norm
    torch.manual_seed(5)
    for dtype in (torch.bfloat16, torch.float32):
        for rows, cols in [(4096, 1024), (4096, 3072), (4096, 4096), (100, 256), (777, 1032)]:
            x = torch.randn(rows, cols, device="cuda", dtype=dtype)
            norm.reset_stats()
            got = norm.sum_dim_intlist(x, [0], True)
            assert norm.stats()["edb_colsum"] == 1 and got.shape == (1, cols)
            want = x.double().sum(0, keepdim=True)
            if dtype == torch.float32:
                assert torch.allclose(got.double(), want, rtol=1e-5, atol=1e-4)
            else:
                assert torch.allclose(got.double(), want, rtol=2 ** -7, atol=0.05 * rows ** 0.5)
    x = torch.randn(8, 5, 16, device="cuda")
    norm.reset_stats()
    norm.sum_dim_intlist(x, [0, 1], False)
    assert norm.stats()["aten_sum"] == 1


def _ce_reference(logits, target, ignore_index, reduction):
    x = logits.detach().float().requires_grad_(True)
    red = "mean" if reduction == 1 else "sum"
    l = torch.nn.functional.cross_entropy(x, target, ignore_index=ignore_index, reduction=red)
    l.backward()
    return l.detach(), x.grad


def test_cross_entropy_matches_fp32_reference(rt):
    """edb_cross_entropy_fwd/bwd vs F.cross_entropy on the fp32 copy of the same logits (the chain
    the traced step contains).  Loss: fp32 online logsumexp, rtol 1e-5.  Gradient: computed in fp32
    and rounded once to the logits dtype like ATen's chain, but with ex2.approx and x - lse instead of
    the stored log-softmax: within 1 ulp of the I/O dtype (bf16: 2^-7 relative) plus 1e-7 absolute."""
    from easydist_b200 import loss
    torch.manual_seed(11)
    cases = [(64, 512, torch.bfloat16, "contig"), (37, 50257, torch.bfloat16, "padded"),
             (37, 50257, torch.bfloat16, "contig"), (129, 1000, torch.float32, "contig"),
             (16, 1003, torch.float32, "padded"), (4096, 50257, torch.bfloat16, "padded")]
    for rows, vocab, dtype, layout in cases:
        for reduction in (1, 2):
            if layout == "padded":
                ld = (vocab + 7) // 8 * 8
                buf = torch.full((rows, ld), 1e4, device="cuda", dtype=dtype)  # poison the padding
                logits = buf[:, :vocab]
                logits.copy_(torch.randn(rows, vocab, device="cuda") * 3)
            else:
                logits = (torch.randn(rows, vocab, device="cuda") * 3).to(dtype)
            target = torch.randint(0, vocab, (rows,), device="cuda")
            target[::7] = -100
            target[1] = vocab - 1
            target[2] = 0
            loss.reset_stats()
            l, tw, lse = loss.cross_entropy_fwd(logits, target, -100, reduction)
            g = torch.full((), 0.5, device="cuda")
            dx = loss.cross_entropy_bwd(g, logits, target, lse, tw, -100, reduction)
            st = loss.stats()
            assert st["edb_ce_fwd"] == 1 and st["edb_ce_bwd"] == 1 and st["aten_ce"] == 0
            want_l, want_dx = _ce_reference(logits, target, -100, reduction)
            assert torch.allclose(l, want_l, rtol=1e-5, atol=1e-5), (rows, vocab, dtype, l, want_l)
            assert float(tw) == float((target != -100).sum())
            assert torch.allclose(lse, torch.logsumexp(logits.float(), 1), rtol=1e-6, atol=1e-5)
            assert dx.dtype == dtype and dx.shape == (rows, vocab) and dx.stride(0) % 8 == 0
            ulp = 2.0 ** -7 if dtype == torch.bfloat16 else 1e-5
            err = (dx.float() - 0.5 * want_dx).abs()
            bound = ulp * (0.5 * want_dx).abs() + 1e-7
            assert bool((err <= bound).all()), (rows, vocab, dtype, float((err - bound).max()))
            assert bool((dx[target == -100] == 0).all())  # ignored rows carry no gradient
            # padding columns of the output buffer are zero (TMA reads them as part of a box)
            if dx.stride(0) != vocab:
                pad = dx.as_strided((rows, dx.stride(0) - vocab), (dx.stride(0), 1), vocab)
                assert bool((pad == 0).all())
    # determinism: same bits on a second run
    l2, _, _ = loss.cross_entropy_fwd(logits, target, -100, 1)
    l3, _, _ = loss.cross_entropy_fwd(logits, target, -100, 1)
    assert l2.item() == l3.item()
    # 3-D logits are not this kernel's case
    loss.reset_stats()
    loss.cross_entropy_fwd(torch.randn(4, 10, device="cuda", dtype=torch.float64),
                           torch.randint(0, 10, (4,), device="cuda"), -100, 1)
    assert loss.stats()["aten_ce"] == 1


def test_sgd_momentum_is_bit_identical_to_the_foreach_ops(rt):
    """edb_sgd_momentum vs the three ATen foreach ops it replaces (integer-exactness is not enough
    here: the claim is identical rounding, so torch.equal on random data, bf16 and fp32)."""
    from easydist_b200 import optim
    torch.manual_seed(13)
    shapes = [(50257, 64), (1024,), (3, 5), (7,), (1,), (4096, 1024), (8,), (1000, 33)] + \
        [(16 + i,) for i in range(330)]  # > 320 tensors: more than one launch
    for dtype in (torch.bfloat16, torch.float32):
        for mu, ga, nlr in [(0.9, 1, -1e-3), (0.8, 0.9, -0.05)]:
            p = [torch.randn(s, device="cuda").to(dtype) for s in shapes]
            g = [(torch.randn(s, device="cuda") * 0.1).to(dtype) for s in shapes]
            m = [(torch.randn(s, device="cuda") * 0.1).to(dtype) for s in shapes]
            p2, m2 = [t.clone() for t in p], [t.clone() for t in m]
            torch.ops.aten._foreach_mul_.Scalar(m2, mu)
            torch.ops.aten._foreach_add_.List(m2, g, alpha=ga)
            torch.ops.aten._foreach_add_.List(p2, m2, alpha=nlr)
            optim.reset_stats()
            optim.sgd_momentum_(p, g, m, mu, ga, nlr)
            assert optim.stats() == {"edb_sgd": 1, "aten_sgd": 0}
            for i, s in enumerate(shapes):
                assert torch.equal(m[i], m2[i]), (dtype, s, "momentum buffer")
                assert torch.equal(p[i], p2[i]), (dtype, s, "parameter")
    # views that are not 16-byte aligned take the ATen ops
    base = torch.randn(64, device="cuda")
    optim.reset_stats()
    optim.sgd_momentum_([base[1:9]], [torch.randn(8, device="cuda")], [torch.zeros(8, device="cuda")],
                        0.9, 1, -0.1)
    assert optim.stats()["aten_sgd"] == 1


def test_gemm_split_k_agrees_with_unsplit(rt):
    """Split-K only reorders the fp32 accumulation: on small-integer operands the split and the
    unsplit kernel must agree bit for bit, on random data within one bf16 ulp; the option turns it
    off; and the workspace is reused across calls (results of consecutive GEMMs do not mix)."""
    from easydist_b200 import gemm
    torch.manual_seed(17)
    M, N, K = 1024, 1024, 4096
    Ai = torch.randint(-1, 2, (M, K), device="cuda").bfloat16()
    Bi = torch.randint(-1, 2, (K, N), device="cuda").bfloat16()
    Ar = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    Br = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
    launches0 = rt.lib.edb_launch_count()
    ci, cr = gemm.mm(Ai.t().contiguous().t(), Bi), gemm.mm(Ar.t().contiguous().t(), Br)  # wgrad layout
    assert rt.lib.edb_launch_count() - launches0 == 4  # GEMM + reduce, twice
    rt.set_option("gemm_splitk", 0)
    try:
        launches0 = rt.lib.edb_launch_count()
        ci0, cr0 = gemm.mm(Ai.t().contiguous().t(), Bi), gemm.mm(Ar.t().contiguous().t(), Br)
        assert rt.lib.edb_launch_count() - launches0 == 2
    finally:
        rt.set_option("gemm_splitk", 1)
    assert torch.equal(ci, ci0)
    err = (cr.float() - cr0.float()).abs()
    assert bool((err <= cr0.float().abs() * 2 ** -7 + 1e-2).all())


@pytest.mark.parametrize("with_bias", [False, True])
def test_gemm_epilogue_residual_add(rt, with_bias):
    """edb_gemm_epi_bf16 (add): res + (a @ b + bias) in one kernel vs a plain fp32 PyTorch
    computation (one bf16 rounding of the exact sum: <= 1 bf16 ulp of the result's magnitude) and vs
    the unfused GEMM-then-add (which rounds twice: <= 2 ulp apart)."""
    from easydist_b200 import gemm
    torch.manual_seed(3)
    for (M, N, K) in [(4096, 1024, 1024), (512, 1024, 4096), (384, 264, 320)]:
        a = torch.randn(M, K, device="cuda").bfloat16()
        b = (torch.randn(K, N, device="cuda") * 0.05).bfloat16()
        res = torch.randn(M, N, device="cuda").bfloat16()
        bias = torch.randn(N, device="cuda").bfloat16() if with_bias else None
        gemm.reset_stats()
        out = gemm.mm_add(a, b, res, bias)
        assert gemm.stats()["edb_gemm_epi"] == 1, gemm.stats()
        prod = a.float() @ b.float()
        ref = prod + res.float() + (bias.float() if with_bias else 0.0)
        # spacing of bf16 at the larger of |result| and |product|: where the residual cancels the
        # product, the tensor cores' fp32 accumulation error (relative to the product) shows
        mag = torch.maximum(ref.abs(), prod.abs()).clamp_min(1e-30)
        ulp = torch.exp2(torch.floor(torch.log2(mag)) - 7)
        # <= 1 ulp for the single rounding, + the accumulator's own error (relative to the product)
        assert float(((out.float() - ref).abs() / ulp).max()) <= 1.5, (M, N, K)
        unfused = (gemm.addmm(bias, a, b) if with_bias else gemm.mm(a, b)) + res
        # the unfused path rounds (product + bias) to bf16 before the add: its error scales with that
        # intermediate's magnitude, not with the (possibly cancelled) result's
        pb = prod + (bias.float() if with_bias else 0.0)
        ulp2 = torch.exp2(torch.floor(torch.log2(torch.maximum(mag, pb.abs()))) - 7)
        assert float(((out.float() - unfused.float()).abs() / ulp2).max()) <= 2.0


def test_gemm_epilogue_gelu_backward(rt):
    """edb_gemm_epi_bf16 (gelu_bwd): aten.gelu_backward(a @ b, pre, approximate='tanh') in the GEMM
    epilogue vs the same formula in fp32 PyTorch on the fp32 product (tolerance: the bf16 rounding of
    the GEMM result that ATen's operand order implies plus the final rounding = 2 bf16 ulp) and vs
    ATen's kernel applied to this library's GEMM output (<= 1 ulp: same rounding points)."""
    from easydist_b200 import gemm
    torch.manual_seed(4)
    for (M, N, K) in [(4096, 4096, 1024), (256, 512, 384)]:
        a = torch.randn(M, K, device="cuda").bfloat16()
        b = (torch.randn(K, N, device="cuda") * 0.05).bfloat16()
        pre = (torch.randn(M, N, device="cuda") * 2).bfloat16()
        gemm.reset_stats()
        out = gemm.mm_gelu_bwd(a, b, pre)
        assert gemm.stats()["edb_gemm_epi"] == 1, gemm.stats()
        prod = a.float() @ b.float()
        ref = torch.ops.aten.gelu_backward(prod, pre.float(), approximate="tanh")
        # bf16 spacing at max(|result|, |product| * 2^-4): gelu' ranges over [-0.13, 1.13], elements
        # where it is ~0 carry the absolute error of the rounded product times the slope error
        # ... and the tensor cores' fp32 accumulation error is absolute (relative to the typical
        # product, not to a product that happens to cancel to ~0): floor at rms(product) / 16
        floor = float(prod.pow(2).mean().sqrt()) * 0.0625
        mag = torch.maximum(ref.abs(), prod.abs() * 0.0625).clamp_min(floor)
        scale = torch.exp2(torch.floor(torch.log2(mag)) - 7)
        assert float(((out.float() - ref).abs() / scale).max()) <= 2.5, (M, N, K)
        aten = torch.ops.aten.gelu_backward(gemm.mm(a, b), pre, approximate="tanh")
        # vs ATen's kernel on this library's GEMM output: same rounding points (ex2/rcp.approx vs tanhf)
        assert float(((out.float() - aten.float()).abs() / scale).max()) <= 1.0, (M, N, K)
        # saturated units (|pre| > 5): the gradient must vanish like ATen's, not like 1 - t*t of an
        # approximate tanh
        sat = pre.float().abs() > 5
        if bool(sat.any()):
            assert float((out.float() - aten.float()).abs()[sat].max()) <= 1e-3


def test_layer_norm_backward_with_fused_accumulation(rt):
    """edb_layer_norm_bwd_add: dx = bf16(bf16(dx_ln) + add) — bit-identical to the LayerNorm
    backward kernel followed by aten.add (the same two roundings)."""
    from easydist_b200 import norm
    torch.manual_seed(5)
    rows, H = 4096, 1024
    x = torch.randn(rows, H, device="cuda").bfloat16()
    dy = torch.randn(rows, H, device="cuda").bfloat16()
    w = torch.randn(H, device="cuda").bfloat16()
    b = torch.randn(H, device="cuda").bfloat16()
    add = torch.randn(rows, H, device="cuda").bfloat16()
    _, mean, rstd = norm.native_layer_norm(x, [H], w, b, 1e-5)
    dx0, dw0, db0 = norm.native_layer_norm_backward(dy, x, [H], mean, rstd, w, b, [True, True, True])
    dx1, dw1, db1 = norm.native_layer_norm_backward(dy, x, [H], mean, rstd, w, b, [True, True, True],
                                                    _add=add)
    assert torch.equal(dx1, dx0 + add)
    assert torch.equal(dw1, dw0) and torch.equal(db1, db0)
