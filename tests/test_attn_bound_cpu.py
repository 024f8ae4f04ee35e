"""The float64 error bounds of tests/attn_ref.py: an fp32 emulation of the attention kernels'
arithmetic, in their order, stays inside them, and each seeded defect breaks them.  The kernels
themselves are checked against the same bounds by tests/test_gpu_attention.py."""
import pytest
import torch

from tests import attn_ref as R

CASES = [(1, 2, 1, 64), (2, 2, 17, 64), (1, 3, 129, 128), (1, 2, 200, 64)]


def _worst(r, got):
    out, lse, dq, dk, dv = got
    refs = (r["out"], r["dq"], r["dk"], r["dv"])
    bounds = (R.fwd_bound(r), *R.bwd_bound(r))
    return max(float(((g - w).abs() / b).max()) for g, w, b in zip((out, dq, dk, dv), refs, bounds))


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("B,H,T,hd", CASES)
def test_emulation_is_inside_the_bound(B, H, T, hd, causal):
    q, k, v, d = R.inputs(B, H, T, hd, seed=T + hd)
    r = R.reference(q, k, v, d, causal)
    got = R.emulate(q, k, v, d, causal)
    assert _worst(r, got) <= 1.0
    assert torch.allclose(got[1], r["lse"], rtol=0, atol=1e-4)


@pytest.mark.parametrize("fault,causal", [("mask", True), ("scale", False), ("lse", True),
                                          ("no_D", False), ("tail", False), ("tail", True)])
def test_each_seeded_fault_breaks_the_bound(fault, causal):
    q, k, v, d = R.inputs(1, 2, 200, 64, seed=3)
    r = R.reference(q, k, v, d, causal)
    assert _worst(r, R.emulate(q, k, v, d, causal)) <= 1.0
    assert _worst(r, R.emulate(q, k, v, d, causal, fault=fault)) > 1.0, fault
