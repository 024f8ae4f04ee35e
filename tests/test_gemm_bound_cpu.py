"""The GEMM error bound of tests/gemm_ref.py is strict enough to catch a subtly wrong kernel: an
emulation of the correct kernel (fp32 accumulation over 16-wide k-steps, one bf16 round-to-nearest)
passes it, and the same emulation with one seeded fault fails it."""
import pytest
import torch

from tests import gemm_ref

M, N, K = 64, 128, 1000  # K = 15 full 64-deep k-blocks + a partial one of 40


def _emulate(A, B, bias=None, drop_step=None, drop_tail=False, rtz=False, swap_cols=False,
             split_twice=False):
    """fp32 accumulation over 16-wide k-steps (each step's 16 products summed exactly), then bias in
    fp32 and one rounding to bf16 — the kernel's arithmetic — with optional faults."""
    A64, B64 = A.double(), B.double()
    steps = [(k, min(k + 16, K)) for k in range(0, K, 16)]
    if drop_step is not None:
        del steps[drop_step]
    if drop_tail:
        steps = [st for st in steps if st[0] < (K // 64) * 64]
    acc = torch.zeros(M, N, dtype=torch.float32)
    for k0, k1 in steps:
        acc = (acc.double() + A64[:, k0:k1] @ B64[k0:k1]).float()
    if split_twice:
        # split-K in 4 slices of 4 k-blocks: slice 1 (k-blocks 4..7) is summed in twice
        part = torch.zeros(M, N, dtype=torch.float32)
        for k0 in range(256, 512, 16):
            part = (part.double() + A64[:, k0:k0 + 16] @ B64[k0:k0 + 16]).float()
        acc = acc + part
    if bias is not None:
        acc = acc + bias.float()
    if rtz:
        bits = acc.view(torch.int32) & ~0xFFFF  # truncate the fp32 mantissa: round toward zero
        c = bits.view(torch.float32).bfloat16()
        assert torch.equal(c.float(), bits.view(torch.float32))
    else:
        c = acc.bfloat16()
    if swap_cols:
        c = c.clone()
        c[:, 8:16], c[:, 16:24] = c[:, 16:24].clone(), c[:, 8:16].clone()  # within chunk [0, 64)
    return c


@pytest.fixture(scope="module")
def operands():
    g = torch.Generator().manual_seed(0)
    A = torch.randn(M, K, generator=g).bfloat16()
    B = torch.randn(K, N, generator=g).bfloat16()
    bias = torch.randn(N, generator=g).bfloat16()
    return A, B, bias


def test_correct_emulation_meets_the_bound(operands):
    A, B, bias = operands
    for bi in (None, bias):
        r, bound = gemm_ref.reference(A, B, bias=bi)
        assert gemm_ref.ratio(_emulate(A, B, bias=bi), r, bound) <= 1.0
    r, _ = gemm_ref.reference(A, B)
    assert gemm_ref.excess(_emulate(A, B), r, A, B) < 0.1


@pytest.mark.parametrize("fault", [dict(drop_step=17), dict(drop_tail=True), dict(rtz=True),
                                   dict(swap_cols=True), dict(split_twice=True), "no_bias"],
                         ids=["dropped_k_step", "dropped_partial_k_block", "round_toward_zero",
                              "swapped_column_groups", "split_slice_twice", "bias_omitted"])
def test_seeded_fault_breaks_the_bound(operands, fault):
    A, B, bias = operands
    r, bound = gemm_ref.reference(A, B, bias=bias)
    c = _emulate(A, B, bias=None) if fault == "no_bias" else _emulate(A, B, bias=bias, **fault)
    assert gemm_ref.ratio(c, r, bound) > 1.0


def test_gelu_bound_holds_for_the_kernel_arithmetic(operands):
    """gelu_bwd: bf16(fp32(bf16(p~) * g~)) meets its bound; a flipped sign or gelu' evaluated at a
    pre-activation 1 % off does not."""
    A, B, _ = operands
    B = (B.float() * 0.05).bfloat16()
    pre = (torch.randn(M, N, generator=torch.Generator().manual_seed(1)) * 2).bfloat16()
    r, bound = gemm_ref.reference(A, B, gelu_pre=pre)
    acc = _emulate(A, B).float()  # bf16(p~)
    g = gemm_ref.gelu_tanh_grad64(pre).float()
    assert gemm_ref.ratio((acc * g).bfloat16(), r, bound) <= 1.0
    assert gemm_ref.ratio((acc * (-g)).bfloat16(), r, bound) > 1.0
    assert gemm_ref.ratio((acc * gemm_ref.gelu_tanh_grad64(pre * 1.01).float()).bfloat16(), r,
                          bound) > 1.0
