"""The embedding-backward bound of tests/embed_ref.py: an fp32 emulation of edb_embed.cu's summation
order stays within it, and each seeded fault (a dropped term, a doubled term, a sum accumulated in
bf16, a term sent to the wrong id, a padding row that is not zeroed) pushes it above 1."""
import pytest
import torch

from tests import embed_ref as E

FAULTS = ["drop", "double", "bf16_acc", "off_by_one", "pad"]


def _inputs(dtype, seed):
    """512 rows over 40 ids: one id takes half the rows, one id is the padding row, a few ids are
    never indexed; dy has a few large entries so that a single lost term stands out."""
    g = torch.Generator().manual_seed(seed)
    V, C, N = 40, 64, 512
    idx = torch.randint(0, V - 4, (N,), generator=g)
    idx[::2] = 7
    idx[5] = 3  # padding row
    dy = torch.randn(N, C, generator=g)
    dy[torch.rand(N, C, generator=g) < 0.02] *= 64
    acc = (torch.randn(V, C, generator=g) * 4).to(dtype)
    return dy.to(dtype), idx, V, 3, acc


def _ratio(got, dy, idx, V, pad, dtype, acc=None):
    S, A, k = E.bwd_ref(dy, idx, V)
    S[pad], A[pad], k[pad] = 0.0, 0.0, 0.0
    if acc is None:
        return E.worst(got, S, E.bwd_bound(S, A, k, dtype))
    return E.worst(got, acc.double() + S, E.acc_bound(acc, S, A, k, dtype))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("mode", ["dense", "acc"])
def test_kernel_order_is_within_the_bound(dtype, mode):
    for seed in range(3):
        dy, idx, V, pad, acc = _inputs(dtype, seed)
        a = acc if mode == "acc" else None
        got = E.emulate(dy, idx, V, pad, dtype, acc=a)
        assert _ratio(got, dy, idx, V, pad, dtype, a) <= 1.0, seed


@pytest.mark.parametrize("fault", FAULTS)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("mode", ["dense", "acc"])
def test_seeded_faults_break_the_bound(dtype, mode, fault):
    dy, idx, V, pad, acc = _inputs(dtype, 0)
    a = acc if mode == "acc" else None
    if fault == "pad" and mode == "acc":
        # the in-place mode leaves the padding row alone: the fault is adding into it
        a[pad] = 0
    got = E.emulate(dy, idx, V, pad, dtype, acc=a, fault=fault)
    assert _ratio(got, dy, idx, V, pad, dtype, a) > 1.0
