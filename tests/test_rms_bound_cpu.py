"""The RMSNorm bounds of tests/rms_ref.py accept a correct fp32 evaluation of the kernel's formula
and reject seeded faults: a wrong eps, a dropped mean(g*n) term, and dw summed in bf16."""
import pytest
import torch

from tests import rms_ref as R


def _emulate(x, w, dy, eps, mode, fault=None):
    """The kernel's arithmetic in fp32 on CPU (torch's own summation order), outputs rounded to T."""
    T = x.dtype
    x32, w32, dy32 = x.float(), w.float(), dy.float()
    e = eps * 10 if fault == "eps" else eps
    rs = torch.rsqrt((x32 * x32).sum(-1, keepdim=True) / x.shape[-1] + e)
    n = x32 * rs
    nhat = n.to(T).float() if mode == R.CAST else n
    y = (nhat * w32).to(T)
    g = dy32 * w32
    if mode == R.CAST:
        g = g.to(T).float()
    s = (g * n).sum(-1, keepdim=True) / x.shape[-1]
    dx = (rs * g if fault == "drop_mean" else rs * (g - n * s)).to(T)
    if fault == "dw_bf16":
        acc = torch.zeros(x.shape[-1], dtype=torch.bfloat16)
        for r in range(x.shape[0]):
            acc = acc + (dy32[r] * nhat[r]).to(torch.bfloat16)
        dw = acc.to(T)
    else:
        dw = (dy32 * nhat).sum(0).to(T)
    return y, rs, dx, dw


def _worst(x, w, dy, eps, mode, out):
    y, rs, dx, dw = out
    y64, r64, nhat, flip = R.forward_ref(x, w, eps, mode)
    dx64, dw64, M, S = R.backward_ref(dy, x, w, r64, mode)
    return dict(rstd=R.worst(rs, r64, R.rstd_bound(x, r64)),
                y=R.worst(y, y64, R.forward_bound(x, w, y64, nhat, flip, mode)),
                dx=R.worst(dx, dx64, R.dx_bound(x, dx64, M)),
                dw=R.worst(dw, dw64, R.dw_bound(dy, x, dw64, S, flip, nhat, mode)))


def _inputs(dtype, rows=2048, H=256):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(rows, H, generator=g).to(dtype)
    w = (torch.randn(H, generator=g) * 0.5 + 1).to(dtype)
    dy = torch.randn(rows, H, generator=g).to(dtype)
    return x, w, dy


@pytest.mark.parametrize("mode", [R.CAST, R.FUSED])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_correct_emulation_passes_and_faults_fail(dtype, mode):
    x, w, dy = _inputs(dtype)
    eps = 1e-5
    ok = _worst(x, w, dy, eps, mode, _emulate(x, w, dy, eps, mode))
    assert max(ok.values()) <= 1.0, ok
    bad_eps = _worst(x, w, dy, eps, mode, _emulate(x, w, dy, eps, mode, "eps"))
    assert bad_eps["rstd"] > 1.0, bad_eps
    bad_mean = _worst(x, w, dy, eps, mode, _emulate(x, w, dy, eps, mode, "drop_mean"))
    assert bad_mean["dx"] > 1.0, bad_mean


def test_dw_summed_in_bf16_fails():
    x, w, dy = _inputs(torch.bfloat16)
    bad = _worst(x, w, dy, 1e-5, R.CAST, _emulate(x, w, dy, 1e-5, R.CAST, "dw_bf16"))
    assert bad["dw"] > 1.0, bad
