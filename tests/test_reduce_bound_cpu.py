"""The bounds of tests/reduce_ref.py accept an fp32 CPU emulation of each kernel's arithmetic, in the
kernel's own summation order, and reject seeded faults.

Column sums and LayerNorm dw / db: the last row of a split dropped, a row counted twice, the lane
partials accumulated in bf16, the column tail lost (cols = 1032).  Cross-entropy: the target column
off by one, the vocabulary tail of the 16-byte path dropped, the mean division applied under
reduction = sum, ignored rows counted in total_weight, the sum of exponentials accumulated in bf16.
ex2.approx is emulated by a correctly rounded exp2 (with the flush to zero below 2^-126)."""
import math

import pytest
import torch

from tests import reduce_ref as R

SMS = R.H100_SMS
L2E = R.LOG2E_F32
C_INV = float(torch.tensor(1.0, dtype=torch.float32) / torch.tensor(L2E, dtype=torch.float32))
ACC = {None: torch.float32, "bf16": torch.bfloat16}


def _add(a, b, fault):
    """a + b rounded to the accumulator type (fp32, or bf16 for the fault)."""
    return (a + b).to(ACC.get(fault, torch.float32)).float()


def _finish(part):
    """k_colsum_finish / k_ln_bwd_finish: slice ky adds partials ky, ky + 8, ... in sequence, then the
    8 slices are added in order."""
    sl = torch.zeros(8, part.shape[-1])
    for k in range(part.shape[0]):
        sl[k % 8] += part[k]
    t = torch.zeros(part.shape[-1])
    for ky in range(8):
        t += sl[ky]
    return t


def _lanes(terms, n_part, warps, steps, fault):
    """Per-lane sequential sums of `terms` [n_part * steps * warps rows (zero-padded), cols] laid out
    as [n_part][steps][warps] for colsum or [steps][n_part][warps] for LayerNorm, then the warps of
    each partial added in order -> [n_part, cols]."""
    acc = torch.zeros(n_part, warps, terms.shape[-1])
    for s in range(steps):
        acc = _add(acc, terms[:, s], fault)
    part = torch.zeros(n_part, terms.shape[-1])
    for w in range(warps):
        part += acc[:, w]
    return part


def _seed(x, fault, last_row):
    x = x.clone()
    if fault == "drop":
        x[last_row] = 0
    elif fault == "twice":
        x[0] *= 2
    return x


def _colsum(x, fault=None):
    rows, cols = x.shape
    splits, rps = R.colsum_config(rows, cols, x.dtype, SMS)
    steps = -(-rps // 8)
    x32 = _seed(x.float(), fault, rps - 1)  # the last row of the first split
    pad = torch.zeros(splits, steps * 8, cols)
    for k in range(splits):
        blk = x32[k * rps:(k + 1) * rps]
        pad[k, :blk.shape[0]] = blk
    out = _finish(_lanes(pad.view(splits, steps, 8, cols), splits, 8, steps, fault)).to(x.dtype)
    if fault == "tail":
        out[1024:] = 0
    return out


def _ln_dwdb(dy, x, mean, rstd, fault=None):
    rows, H = x.shape
    grid = R.ln_grid(rows, SMS)
    steps = -(-rows // (4 * grid))
    xh = (x.float() - mean[:, None]) * rstd[:, None]
    outs = []
    for terms in (dy.float() * xh, dy.float()):
        # row r = step * 4*grid + cta * 4 + warp; the last row of the grid's last pass is dropped
        terms = _seed(terms, fault, rows - 1)
        pad = torch.zeros(steps * 4 * grid, H)
        pad[:rows] = terms
        lanes = pad.view(steps, grid, 4, H).transpose(0, 1)
        out = _finish(_lanes(lanes, grid, 4, steps, fault)).to(x.dtype)
        if fault == "tail":
            out[1024:] = 0
        outs.append(out)
    return outs


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_colsum_bound(dtype):
    g = torch.Generator().manual_seed(0)
    for rows, cols, scale in [(4096, 1024, 0.01), (8193, R.epv(dtype), 1.0), (777, 1032, 1.0)]:
        x = (torch.randn(rows, cols, generator=g) * scale).to(dtype)
        s64, A = R.colsum_ref(x)
        bound = R.colsum_bound(s64, A, R.colsum_depth(rows, cols, dtype, SMS), dtype)
        ok = R.worst(_colsum(x), s64, bound)
        assert ok <= 1.0, (rows, cols, ok)
        faults = ("drop", "twice", "bf16") + (("tail",) if cols == 1032 else ())
        for fault in faults:
            bad = R.worst(_colsum(x, fault), s64, bound)
            assert bad > 1.0, (rows, cols, fault, bad)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_layer_norm_dw_db_bound(dtype):
    g = torch.Generator().manual_seed(1)
    eps = 1e-5
    for rows, H in [(2048, 256), (8 * SMS + 1, 1032), (100, 512)]:
        x = torch.randn(rows, H, generator=g).to(dtype)
        dy = (torch.randn(rows, H, generator=g) * 1e-2).to(dtype)
        x32 = x.float()
        mean = x32.mean(-1)
        rstd = torch.rsqrt(((x32 - mean[:, None]) ** 2).mean(-1) + eps)
        dw64, db64, Sw, Sb, Dx = R.ln_dwdb_ref(dy, x, mean, rstd, eps)
        depth = R.ln_depth(rows, SMS)
        bw = R.ln_dw_bound(dw64, Sw, Dx, depth, dtype)
        bb = R.ln_db_bound(db64, Sb, depth, dtype)
        dw, db = _ln_dwdb(dy, x, mean, rstd)
        ok = (R.worst(dw, dw64, bw), R.worst(db, db64, bb))
        assert max(ok) <= 1.0, (rows, H, ok)
        # 100 rows: a shrunk grid, one row per lane, so a bf16 lane accumulator only adds to zero
        faults = ("drop", "twice") + (("bf16",) if rows > 8 * SMS else ()) + \
            (("tail",) if H == 1032 else ())
        for fault in faults:
            dw, db = _ln_dwdb(dy, x, mean, rstd, fault)
            bad = (R.worst(dw, dw64, bw), R.worst(db, db64, bb))
            assert min(bad) > 1.0, (rows, H, fault, bad)


# ---- cross-entropy ------------------------------------------------------------------------------

def _ex2(a):
    y = torch.exp2(a.double()).float()
    return torch.where(y < 2.0 ** -126, torch.zeros_like(y), y)


def _fma(a, b, c):
    return (a.double() * b + c.double()).float()


def _merge(am, as_, bm, bs):
    om = torch.maximum(am, bm)
    fin = om != -math.inf
    z = torch.zeros_like(om)
    s = as_ * _ex2(torch.where(fin, am - om, z)) + bs * _ex2(torch.where(fin, bm - om, z))
    return om, torch.where(fin, s, z)


def _ce_lse(x, vec, fault=None):
    """k_ce_fwd's logsumexp: per-thread online (max, sum) over its vectors, xor-shuffle merges, the 8
    warps merged in order."""
    rows, V = x.shape
    x32 = x.float()
    n = R.epv(x.dtype) if vec else 1
    nbody = V // n * n
    blocks = []
    for part, width in ((x32[:, :nbody], n), (x32[:, nbody:], 1)):
        if part.shape[1] == 0 or (fault == "tail" and width == 1 and vec):
            continue
        steps = -(-part.shape[1] // (R.CE_THREADS * width))
        pad = torch.full((rows, steps * R.CE_THREADS * width), -math.inf)
        pad[:, :part.shape[1]] = part
        blocks.append(pad.view(rows, steps, R.CE_THREADS, width))
    m = torch.full((rows, R.CE_THREADS), -math.inf)
    s = torch.zeros(rows, R.CE_THREADS)
    for X in blocks:
        for st in range(X.shape[1]):
            f = X[:, st]
            vm = (f.max(-1).values.double() * L2E).float()
            up = vm > m
            s = torch.where(up, s * _ex2(m - vm), s)
            m = torch.where(up, vm, m)
            live = m != -math.inf
            for e in range(f.shape[-1]):
                t = _ex2(_fma(f[..., e], L2E, torch.where(live, -m, torch.zeros_like(m))))
                s = _add(s, torch.where(live, t, torch.zeros_like(t)), fault)
    m, s = m.view(rows, 8, 32), s.view(rows, 8, 32)
    for o in (16, 8, 4, 2, 1):
        idx = torch.arange(32) ^ o
        m, s = _merge(m, s, m[..., idx], s[..., idx])
    tm, ts = m[:, 0, 0], s[:, 0, 0]
    for w in range(1, 8):
        tm, ts = _merge(tm, ts, m[:, w, 0], s[:, w, 0])
    return (tm * C_INV).float() + torch.log(ts.double()).float()


def _ce(x, target, ign, red, g, vec, fault=None):
    """-> (lse, row_loss, loss, dx) as k_ce_fwd + k_ce_finish + k_ce_bwd compute them."""
    rows, V = x.shape
    l = _ce_lse(x, vec, fault)
    keep = target != ign
    tc = target.clamp(0, V - 1)
    tcol = (tc + 1).clamp(max=V - 1) if fault == "target" else tc
    x32 = x.float()
    rl = torch.where(keep, l - x32.gather(1, tcol[:, None])[:, 0], torch.zeros_like(l))
    cnt = float(rows if fault == "count" else keep.sum())
    acc = torch.zeros(1024)
    for r in range(rows):
        acc[r % 1024] += rl[r]
    o = 512
    while o:
        acc[:o] += acc[o:2 * o]
        o //= 2
    mean = red == 1 or fault == "mean"
    loss = acc[0] / cnt if mean else acc[0]
    c = torch.tensor(g, dtype=torch.float32) / cnt if mean else torch.tensor(g, dtype=torch.float32)
    c = torch.where(keep, c, torch.zeros_like(l))[:, None]
    nl = (-l.double() * L2E).float()
    p = _ex2(_fma(x32, L2E, nl[:, None]))
    v = p * c
    cols = torch.arange(V)[None, :] == tcol[:, None]
    v = torch.where(cols, (p.double() * c - c).float(), v)
    dx = v.to(x.dtype)
    if fault == "tail" and vec:
        dx[:, V // R.epv(x.dtype) * R.epv(x.dtype):] = 0
    return l, rl, loss, dx


def _ce_ratios(x, target, ign, red, g, vec, fault=None):
    ref = R.ce_ref(x, target, ign, red, g)
    l, rl, loss, dx = _ce(x, target, ign, red, g, vec, fault)
    return dict(lse=R.worst(l, ref["lse"], R.ce_lse_bound(ref, x.dtype, vec)),
                row_loss=R.worst(rl, ref["row_loss"], R.ce_row_loss_bound(ref, x.dtype, vec)),
                loss=abs(float(loss) - float(ref["loss"])) / R.ce_loss_bound(ref, x.dtype, vec, red),
                dx=R.worst(dx, ref["dx"], R.ce_dx_bound(ref, x.dtype, vec)))


# which output each seeded fault must push above its bound
CE_FAULTS = [("target", 1, "loss"), ("target", 2, "dx"), ("tail", 1, "lse"), ("mean", 2, "loss"),
             ("count", 1, "loss"), ("bf16", 1, "lse")]


@pytest.mark.parametrize("vec", [True, False], ids=["vec16", "scalar"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_cross_entropy_bound(dtype, vec):
    g = torch.Generator().manual_seed(2)
    rows, V = 48, 2049  # 2049: one element past the 16-byte body in both dtypes
    for scale, shift in ((3.0, 0.0), (1.0, 1000.0)):
        x = (torch.randn(rows, V, generator=g) * scale + shift).to(dtype)
        target = torch.randint(0, V - 1, (rows,), generator=g)
        target[::5] = -100
        target[1] = V - 2
        for red, go in ((1, 0.5), (2, -3.0)):
            ok = _ce_ratios(x, target, -100, red, go, vec)
            assert max(ok.values()) <= 1.0, (scale, shift, red, ok)
        if shift:
            continue
        for fault, red, what in CE_FAULTS:
            if fault == "tail" and not vec:
                continue
            bad = _ce_ratios(x, target, -100, red, 0.5, vec, fault)
            assert bad[what] > 1.0, (fault, red, bad)
