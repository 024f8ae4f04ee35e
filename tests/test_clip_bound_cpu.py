"""The sum-of-squares bound of tests/clip_ref.py accepts an fp32 evaluation in the kernel's chunk
structure and rejects seeded faults: a dropped chunk, a chunk counted twice and a sum accumulated in
bf16."""
import pytest
import torch

from tests import clip_ref as R


def _emulate(g, fault=None):
    """Per-chunk fp32 partials (torch's own order inside a chunk), added in index order."""
    ce = R.chunk_elems(g.dtype)
    x = g.detach().float().flatten()
    parts = [float((c * c).sum()) for c in x.split(ce)]
    if fault == "drop":
        parts = parts[:1] + parts[2:]
    elif fault == "twice":
        parts = parts + parts[1:2]
    if fault == "bf16":
        acc = torch.zeros((), dtype=torch.bfloat16)
        for p in parts:
            acc = acc + torch.tensor(p).bfloat16()
        return float(acc)
    acc = torch.zeros((), dtype=torch.float32)
    for p in parts:
        acc = acc + torch.tensor(p, dtype=torch.float32)
    return float(acc)


def _grads(dtype):
    g = torch.Generator().manual_seed(0)
    return [(torch.randn(n, generator=g) * s).to(dtype)
            for n, s in ((1, 1.0), (7, 3.0), (4095, 0.01), (3 * 8192 + 5, 1.0), (40 * 8192, 0.1))]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_correct_emulation_passes_and_faults_fail(dtype):
    grads = _grads(dtype)
    ok = R.worst(torch.tensor([_emulate(g) for g in grads], dtype=torch.float64), grads)
    assert ok <= 1.0, ok
    multi = [g for g in grads if g.numel() > 2 * R.chunk_elems(dtype)]
    for fault in ("drop", "twice", "bf16"):
        bad = R.worst(torch.tensor([_emulate(g, fault) for g in multi], dtype=torch.float64), multi)
        assert bad > 1.0, (fault, bad)
