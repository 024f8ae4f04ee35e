"""The native entry points on the tensor layouts a traced graph hands them (H100): transposes, slices
of wider buffers, contiguous views at a misaligned storage offset, expanded (stride-0) operands and,
for the GEMM, MN-major operands, leading dimensions that are not a multiple of 8 and overlapping rows.
The padding of every wider buffer holds NaN, so a kernel that reads it shows in the result.

Every case checks that the call raises nothing, which path it took (the module's stats), its values
and that its inputs are untouched (every byte of their storage, padding included).  Values: where the
native path runs the kernel variant the dense case runs, the result must carry the bits of the same
entry point called on dense, aligned clones; where the layout picks another variant (GEMM operand
major, cross-entropy's 16-byte or scalar loads) the float64 bounds of tests/gemm_ref.py and
tests/reduce_ref.py apply.  Two tiny compiled bf16 steps cover the graph side: a bias-free head whose
narrowed GEMM output is flattened, and a loss that sum-pools a Linear output over its rows (its
backward hands the GEMMs an expanded gradient)."""
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from tests import gemm_ref as G
from tests import reduce_ref as R

pytestmark = pytest.mark.gpu
aten = torch.ops.aten
BF = torch.bfloat16


@pytest.fixture(scope="module")
def rt():
    from easydist_b200 import runtime
    from easydist_b200.device_mesh import set_device_mesh
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    r = runtime.init(rank=0, world=1, device=0, heap_bytes=2 << 30) \
        if not runtime.is_initialized() else runtime.get_runtime()
    set_device_mesh([0], ["dp"], rank=0)
    return r


# ---- layouts ----------------------------------------------------------------------------------

def _same_bits(a, b):
    it = {2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    return a.dtype == b.dtype and a.shape == b.shape and \
        torch.equal(a.contiguous().view(it), b.contiguous().view(it))


def _nan(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _layout(d, kind):
    """A tensor with d's values (for "expanded", d's first row broadcast along dim 0) laid out as
    `kind`; whatever else its buffer holds is NaN."""
    if kind == "dense":
        return d.clone()
    if kind.startswith("offset"):                 # contiguous, k elements past an aligned start
        k = int(kind[6:])
        buf = _nan((d.numel() + k + 16,), d.dtype)
        v = buf[k:k + d.numel()].view(d.shape)
        v.copy_(d)
        return v
    if kind == "expanded":                        # the buffer is d's size: a dense read stays inside it
        buf = _nan(d.shape, d.dtype)
        buf[:1] = d[:1]
        return buf[:1].expand(d.shape)
    if d.dim() == 1:
        assert kind == "strided", kind             # every second element of a longer buffer
        buf = _nan((2 * d.numel(),), d.dtype)
        buf[::2] = d
        return buf[::2]
    R_, C = d.shape
    if kind == "transposed":                      # column-major storage of the same matrix
        buf = _nan((C, R_), d.dtype)
        buf.copy_(d.t())
        return buf.t()
    if kind in ("sliced", "sliced_odd"):          # rows of a wider buffer (ld % 8 == 0 or == 3)
        buf = _nan((R_, C + (24 if kind == "sliced" else 3)), d.dtype)
        buf[:, :C] = d
        return buf[:, :C]
    if kind == "overlapping":                     # rows 64 elements apart, each C > 64 long
        assert C > 64
        buf = torch.empty(R_ * 64 + C, dtype=d.dtype, device="cuda")
        buf.copy_(torch.arange(buf.numel(), device="cuda").remainder(61).sub(30).div(16))
        return buf.as_strided((R_, C), (64, 1))
    raise ValueError(kind)


def _clone(t):
    """A dense, aligned copy in a fresh allocation."""
    return t.clone(memory_format=torch.contiguous_format)


def _storage(t):
    return torch.empty(0, dtype=torch.uint8, device=t.device).set_(t.untyped_storage()).clone()


class _Untouched:
    """Every byte of the given tensors' storages is the same on exit as on entry."""

    def __init__(self, *ts):
        self.ts = [t for t in ts if isinstance(t, torch.Tensor)]

    def __enter__(self):
        self.before = [_storage(t) for t in self.ts]

    def __exit__(self, *exc):
        if exc[0] is None:
            torch.cuda.synchronize()
            for i, (t, b) in enumerate(zip(self.ts, self.before)):
                assert torch.equal(_storage(t), b), f"input {i} was written"
        return False


def _randn(g, *shape, dtype=BF, scale=1.0, shift=0.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale + shift).to(dtype)


# ---- LayerNorm --------------------------------------------------------------------------------

_ACT = ["transposed", "sliced", "offset1", "offset2", "offset3", "expanded"]
_VEC = ["strided", "offset1", "offset2", "offset3", "expanded"]
_NORM_CASES = [(op, k) for op in ("x", "dy", "add") for k in _ACT] + \
              [(op, k) for op in ("weight", "bias") for k in _VEC]


@pytest.mark.parametrize("dtype", [BF, torch.float32])
@pytest.mark.parametrize("operand,layout", _NORM_CASES)
def test_layer_norm_layouts_give_the_dense_bits(rt, dtype, operand, layout):
    """Every layout runs natively and gives the bits of the dense call: the kernel reads dense,
    aligned copies of whatever is not (a strided weight used to be read as if it were dense)."""
    from easydist_b200 import norm
    H, rows = (768, 96) if dtype == BF else (512, 96)
    g = torch.Generator(device="cuda").manual_seed(len(operand) * 31 + len(layout))
    ops = {"x": _randn(g, rows, H, dtype=dtype, scale=2, shift=0.1), "dy": _randn(g, rows, H, dtype=dtype),
           "add": _randn(g, rows, H, dtype=dtype), "weight": _randn(g, H, dtype=dtype, scale=0.5, shift=1),
           "bias": _randn(g, H, dtype=dtype)}
    ops[operand] = _layout(ops[operand], layout)
    dense = {k: _clone(v) for k, v in ops.items()}

    def run(o):
        y, mean, rstd = norm.native_layer_norm(o["x"], [H], o["weight"], o["bias"], 1e-5)
        grads = norm.native_layer_norm_backward(o["dy"], o["x"], [H], mean, rstd, o["weight"], o["bias"],
                                                [True, True, True])
        dxa = norm.native_layer_norm_backward(o["dy"], o["x"], [H], mean, rstd, o["weight"], o["bias"],
                                              [True, False, False], _add=o["add"])[0]
        return [y, mean, rstd, *grads, dxa]

    norm.reset_stats()
    with _Untouched(*ops.values()):
        got = run(ops)
    st = norm.stats()
    assert st["aten_ln"] == 0 and st["edb_ln_fwd"] == 1 and st["edb_ln_bwd"] == 2, st
    want = run(dense)
    for i, (a, b) in enumerate(zip(got, want)):
        assert _same_bits(a, b), ("y mean rstd dx dw db dx+add".split()[i], operand, layout)


# ---- RMSNorm ----------------------------------------------------------------------------------

_RMS_CASES = [(op, k) for op in ("x", "dy", "add") for k in _ACT] + [("w", k) for k in _VEC]


@pytest.mark.parametrize("dtype", [BF, torch.float32])
@pytest.mark.parametrize("operand,layout", _RMS_CASES)
def test_rms_norm_layouts_give_the_dense_bits(rt, dtype, operand, layout):
    from easydist_b200 import norm
    H, rows = (1024, 80) if dtype == BF else (512, 80)
    g = torch.Generator(device="cuda").manual_seed(len(operand) * 37 + len(layout))
    ops = {"x": _randn(g, rows, H, dtype=dtype, scale=2, shift=0.1), "dy": _randn(g, rows, H, dtype=dtype),
           "add": _randn(g, rows, H, dtype=dtype), "w": _randn(g, H, dtype=dtype, scale=0.5, shift=1)}
    ops[operand] = _layout(ops[operand], layout)
    dense = {k: _clone(v) for k, v in ops.items()}

    def run(o):
        outs = []
        for mode in (norm.RMS_CAST_THEN_SCALE, norm.RMS_FUSED):
            y, rstd = norm.rms_norm_fwd(o["x"], o["w"], 1e-5, mode)
            outs += [y, rstd, *norm.rms_norm_bwd(o["dy"], o["x"], rstd, o["w"], mode, [True, True])]
            outs.append(norm.rms_norm_bwd(o["dy"], o["x"], rstd, o["w"], mode, [True, False],
                                          _add=o["add"])[0])
        return outs

    norm.reset_stats()
    with _Untouched(*ops.values()):
        got = run(ops)
    st = norm.stats()
    assert st["aten_rms"] == 0 and st["edb_rms_fwd"] == 2 and st["edb_rms_bwd"] == 4, st
    for i, (a, b) in enumerate(zip(got, run(dense))):
        assert _same_bits(a, b), (i, operand, layout)


# ---- GEMM -------------------------------------------------------------------------------------

M, K, N = 192, 320, 256
# layout -> (runs natively, operands staged into a padded buffer, same kernel variant as dense)
_GEMM_PATH = {"dense": (True, 0, True), "sliced": (True, 0, True), "sliced_odd": (True, 1, True),
              "offset1": (True, 1, True), "offset2": (True, 1, True), "offset3": (True, 1, True),
              "transposed": (True, 0, False), "expanded": (False, 0, None),
              "overlapping": (False, 0, None)}
_GEMM_OPS = ["mm", "addmm", "mm_add", "mm_gelu_bwd"]


def _gemm_inputs(seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return {"a": _randn(g, M, K), "b": _randn(g, K, N), "bias": _randn(g, N),
            "aux": _randn(g, M, N, scale=2)}


def _gemm_call(op, o):
    from easydist_b200 import gemm
    if op == "mm":
        return gemm.mm(o["a"], o["b"])
    if op == "addmm":
        return gemm.addmm(o["bias"], o["a"], o["b"])
    if op == "mm_add":
        return gemm.mm_add(o["a"], o["b"], o["aux"], o["bias"])
    return gemm.mm_gelu_bwd(o["a"], o["b"], o["aux"])


def _gemm_ref(op, o):
    if op == "mm":
        return G.reference(o["a"], o["b"])
    if op == "addmm":
        return G.reference(o["a"], o["b"], bias=o["bias"])
    if op == "mm_add":
        return G.reference(o["a"], o["b"], bias=o["bias"], add=o["aux"])
    return G.reference(o["a"], o["b"], gelu_pre=o["aux"])


@pytest.mark.parametrize("op", _GEMM_OPS)
@pytest.mark.parametrize("operand", ["a", "b"])
@pytest.mark.parametrize("layout", list(_GEMM_PATH))
def test_gemm_operand_layouts(rt, op, operand, layout):
    """A and B in every layout.  Overlapping rows (an expanded operand has ld 0) are no matrix TMA
    can describe: they go to ATen, counted."""
    from easydist_b200 import gemm
    native, padded, same = _GEMM_PATH[layout]
    o = _gemm_inputs(seed=sum(map(ord, op + operand + layout)))
    o[operand] = _layout(o[operand], layout)
    dense = {k: _clone(v) for k, v in o.items()}
    gemm.reset_stats()
    with _Untouched(*o.values()):
        c = _gemm_call(op, o)
    st = gemm.stats()
    fused = op in ("mm_add", "mm_gelu_bwd")
    if native:
        assert st["aten_mm"] == 0 and st["edb_gemm"] == 1 and st["padded_operands"] == padded, st
        assert st["edb_gemm_epi"] == int(fused), st
    else:
        assert st["aten_mm"] == 1 and st["edb_gemm"] == 0 and st["edb_gemm_epi"] == 0, st
    assert c.shape == (M, N) and c.dtype == BF
    if same:
        gemm.reset_stats()
        assert _same_bits(c, _gemm_call(op, dense)), (op, operand, layout)
    elif native:
        r, bound = _gemm_ref(op, dense)
        assert G.ratio(c, r, bound) <= 1.0, (op, operand, layout, G.ratio(c, r, bound))
    else:
        # ATen's mm on the same operands, followed by the op's elementwise ATen step
        p = aten.mm.default(o["a"], o["b"])
        want = {"mm": lambda: p, "addmm": lambda: aten.addmm.default(o["bias"], o["a"], o["b"]),
                "mm_add": lambda: aten.add.Tensor(o["aux"], aten.addmm.default(o["bias"], o["a"], o["b"])),
                "mm_gelu_bwd": lambda: aten.gelu_backward.default(p, o["aux"], approximate="tanh")}[op]()
        assert _same_bits(c, want), (op, operand, layout)


# epilogue operand layout -> fused into the GEMM epilogue (else: plain GEMM, then ATen)
_AUX_PATH = {"dense": True, "sliced": True, "transposed": False, "sliced_odd": False, "offset1": False,
             "offset2": False, "offset3": False, "expanded": False}


@pytest.mark.parametrize("op", ["mm_add", "mm_gelu_bwd"])
@pytest.mark.parametrize("layout", list(_AUX_PATH))
def test_gemm_epilogue_operand_layouts(rt, op, layout):
    """The residual / pre-activation the epilogue reads with a row stride: rows of a wider buffer
    are read in place, everything else (stride(0) < N included) takes the unfused path."""
    from easydist_b200 import gemm
    o = _gemm_inputs(seed=len(layout) + 7 * len(op))
    o["aux"] = _layout(o["aux"], layout)
    dense = {k: _clone(v) for k, v in o.items()}
    gemm.reset_stats()
    with _Untouched(*o.values()):
        c = _gemm_call(op, o)
    st = gemm.stats()
    fused = _AUX_PATH[layout]
    assert st["aten_mm"] == 0 and st["edb_gemm"] == 1 and st["edb_gemm_epi"] == int(fused), st
    if fused:
        want = _gemm_call(op, dense)
    elif op == "mm_add":
        want = aten.add.Tensor(dense["aux"], gemm.addmm(dense["bias"], dense["a"], dense["b"]))
    else:
        want = aten.gelu_backward.default(gemm.mm(dense["a"], dense["b"]), dense["aux"], approximate="tanh")
    assert _same_bits(c, want), (op, layout)


@pytest.mark.parametrize("layout", ["strided", "offset1", "offset2", "offset3", "expanded"])
def test_gemm_bias_layouts(rt, layout):
    """A bias the epilogue cannot read (not dense or not 16-byte aligned) is added by ATen behind the
    plain GEMM, for addmm and for mm_add."""
    from easydist_b200 import gemm
    o = _gemm_inputs(seed=len(layout))
    o["bias"] = _layout(o["bias"], layout)
    dense = {k: _clone(v) for k, v in o.items()}
    gemm.reset_stats()
    with _Untouched(*o.values()):
        c = gemm.addmm(o["bias"], o["a"], o["b"])
        c2 = gemm.mm_add(o["a"], o["b"], o["aux"], o["bias"])
    st = gemm.stats()
    assert st["aten_mm"] == 0 and st["edb_gemm"] == 2 and st["edb_gemm_epi"] == 0, st
    plain = gemm.mm(dense["a"], dense["b"])
    assert _same_bits(c, aten.add.Tensor(plain, dense["bias"])), layout
    assert _same_bits(c2, aten.add.Tensor(dense["aux"], aten.add.Tensor(plain, dense["bias"]))), layout


@pytest.mark.parametrize("n_out", [3, 250])
def test_gemm_narrowed_output_feeds_the_next_gemm(rt, n_out):
    """An output with N % 8 != 0 is a narrowed view of a padded buffer: as the next GEMM's A it is
    read in place, as the other operand of a wgrad (transposed) too."""
    from easydist_b200 import gemm
    g = torch.Generator(device="cuda").manual_seed(n_out)
    x, w, w2 = _randn(g, M, K), _randn(g, n_out, K, scale=0.1).t(), _randn(g, n_out, 64)  # w: a Linear's
    gemm.reset_stats()
    h = gemm.mm(x, w)
    assert h.stride() == (n_out + (-n_out) % 8, 1)
    with _Untouched(h, w2, x):
        y = gemm.mm(h, w2)                   # A with a padded row stride
        dw = gemm.mm(h.t(), x)               # A MN-major, from the same buffer
    st = gemm.stats()
    assert st["edb_gemm"] == 3 and st["aten_mm"] == 0 and st["padded_operands"] == 0, st
    hd = _clone(h)
    assert _same_bits(y, gemm.mm(hd, w2))
    r, bound = G.reference(hd.t(), x)
    assert G.ratio(dw, r, bound) <= 1.0


# ---- SwiGLU and RoPE --------------------------------------------------------------------------

def _swiglu_chain(gate, up, dy):
    out = aten.mul.Tensor(aten.silu.default(gate), up)
    dup = aten.mul.Tensor(dy, aten.silu.default(gate))
    dgate = aten.silu_backward.default(aten.mul.Tensor(dy, up), gate)
    return out, dgate, dup


@pytest.mark.parametrize("dtype", [BF, torch.float32])
@pytest.mark.parametrize("layout", ["chunks", "chunks_offset1", "transposed", "expanded"])
def test_swiglu_layouts_equal_the_aten_chains(rt, dtype, layout):
    """gate / up as the two chunk(2, -1) halves of one [rows, 2F] buffer (also at a misaligned
    start), as transposes, and dy expanded along rows: the bits of the ATen chains."""
    from easydist_b200 import act
    rows, Fd = 96, 344
    g = torch.Generator(device="cuda").manual_seed(len(layout))
    both = _randn(g, rows, 2 * Fd, dtype=dtype, scale=3)
    dy = _randn(g, rows, Fd, dtype=dtype)
    if layout.startswith("chunks"):
        if layout.endswith("offset1"):
            both = _layout(both, "offset1")
        gate, up = both.chunk(2, -1)
    elif layout == "transposed":
        gate, up = _layout(both[:, :Fd], "transposed"), _layout(both[:, Fd:], "transposed")
        dy = _layout(dy, "transposed")
    else:
        gate, up = both.chunk(2, -1)
        dy = _layout(dy, "expanded")
    act.reset_stats()
    with _Untouched(gate, up, dy):
        out = act.swiglu_fwd(gate, up)
        dgate, dup = act.swiglu_bwd(dy, gate, up)
    st = act.stats()
    assert st["aten_swiglu"] == 0 and st["edb_swiglu_fwd"] == 1 and st["edb_swiglu_bwd"] == 1, st
    for got, want in zip((out, dgate, dup), _swiglu_chain(gate, up, dy)):
        assert _same_bits(got, want), layout


@pytest.mark.parametrize("dtype", [BF, torch.float32])
@pytest.mark.parametrize("source", ["transposed", "qkv", "qkv_offset1"])
def test_rope_layouts_equal_the_formula(rt, dtype, source):
    """x as the transpose(1, 2) of [B, T, H, hd], or sliced out of a fused qkv projection (whose
    rows hold q, k and v); cos / sin as the first T rows of a longer table."""
    from easydist_b200 import rope
    B, T, H, hd, Tmax = 2, 40, 4, 64, 128
    g = torch.Generator(device="cuda").manual_seed(len(source))
    if source == "transposed":
        x = _randn(g, B, T, H, hd, dtype=dtype).transpose(1, 2)
    else:
        qkv = _randn(g, B * T, 3 * H * hd, dtype=dtype)
        if source.endswith("offset1"):
            qkv = _layout(qkv, "offset1")
        x = qkv.view(B, T, 3, H, hd)[:, :, 1].transpose(1, 2)     # k
    ang = torch.arange(Tmax, device="cuda")[:, None] * torch.rand(hd // 2, device="cuda", generator=g)
    cos_t, sin_t = torch.cos(ang).to(dtype), torch.sin(ang).to(dtype)
    cos, sin = cos_t[:T], sin_t[:T]
    rope.reset_stats()
    with _Untouched(x, cos_t, sin_t):
        y = rope.rope(x, cos, sin)
        dx = rope.rope(x, cos, sin, True)
        dxt = rope.rope(x, cos, sin, True, transposed=True)
    st = rope.stats()
    assert st["aten_rope"] == 0 and st["edb_rope_fwd"] == 1 and st["edb_rope_bwd"] == 2, st
    assert _same_bits(y, rope.formula(x, cos, sin))
    want = rope.formula(x, cos, sin, inverse=True)
    assert _same_bits(dx, want) and _same_bits(dxt, want.transpose(1, 2).contiguous())


# ---- cross-entropy ----------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [BF, torch.float32])
@pytest.mark.parametrize("layout", ["lm_head", "offset1", "offset3", "strided_target"])
def test_cross_entropy_layouts(rt, dtype, layout):
    """Logits as the narrowed LM-head output (row stride 50264, 16-byte loads), at a misaligned
    start (scalar loads): float64 bounds of the load path taken.  A non-contiguous target is not the
    kernel's case: the ATen ops, counted, with the bits they give on dense operands."""
    from easydist_b200 import loss
    rows, vocab = 48, 50257
    g = torch.Generator(device="cuda").manual_seed(len(layout))
    x = _randn(g, rows, vocab, dtype=dtype, scale=3)
    target = torch.randint(0, vocab, (rows,), device="cuda", generator=g)
    target[5] = target[17] = -100
    if layout == "lm_head":
        buf = _nan((rows, 50264), dtype)
        buf[:, :vocab] = x
        x = buf[:, :vocab]
    elif layout.startswith("offset"):
        x = _layout(x, layout)
    else:
        tbuf = torch.full((2 * rows,), 7, dtype=torch.int64, device="cuda")
        tbuf[::2] = target
        target = tbuf[::2]
    go = torch.tensor(1.0, device="cuda")
    loss.reset_stats()
    with _Untouched(x, target):
        l, tw, lse = loss.cross_entropy_fwd(x, target, -100, 1)
        dx = loss.cross_entropy_bwd(go, x, target, lse, tw, -100, 1)
    st = loss.stats()
    if layout == "strided_target":
        assert st["aten_ce"] == 2 and st["edb_ce_fwd"] == 0 and st["edb_ce_bwd"] == 0, st
        xd, td = _clone(x), _clone(target)
        want = loss._aten_fwd(xd, td, -100, 1)
        for a, b in zip((l, tw, lse), want):
            assert _same_bits(a, b), layout
        ls = xd.float() - want[2].unsqueeze(1)
        wdx = aten._log_softmax_backward_data.default(
            aten.nll_loss_backward.default(go, ls, td, None, 1, -100, want[1]), ls, 1, torch.float32)
        assert _same_bits(dx, wdx.to(dtype)), layout
        return
    assert st["aten_ce"] == 0 and st["edb_ce_fwd"] == 1 and st["edb_ce_bwd"] == 1, st
    vec = R.ce_vec_fwd(x)
    assert vec == (layout == "lm_head")
    ref = R.ce_ref(x, target, -100, 1, 1.0)
    assert float(tw) == ref["count"]
    assert abs(float(l) - float(ref["loss"])) <= R.ce_loss_bound(ref, dtype, vec, 1), layout
    assert R.worst(lse, ref["lse"], R.ce_lse_bound(ref, dtype, vec)) <= 1.0, layout
    assert dx.shape == x.shape and dx.dtype == dtype
    assert R.worst(dx, ref["dx"], R.ce_dx_bound(ref, dtype, vec)) <= 1.0, layout
    assert bool((dx[~ref["keep"]] == 0).all()), layout


# ---- SGD --------------------------------------------------------------------------------------

def test_sgd_list_mixing_dense_narrowed_and_transposed_gradients(rt):
    """Dense gradients take the kernel and give the bits of the kernel on dense clones; a narrowed
    or transposed gradient (not dense) takes the counted ATen group, within two fp32 roundings of
    float64."""
    from easydist_b200 import optim
    g = torch.Generator(device="cuda").manual_seed(3)
    shapes = [(64, 40), (96, 24), (40, 64), (128,)]
    params = [_randn(g, *s, dtype=torch.float32) for s in shapes]
    bufs = [_randn(g, *s, dtype=torch.float32, scale=0.1) for s in shapes]
    grads = [_randn(g, *s, dtype=torch.float32) for s in shapes]
    grads[1] = _layout(grads[1], "sliced")            # rows of the padded output of a GEMM
    grads[2] = _layout(grads[2], "transposed")        # the t() of a wgrad
    p0, m0, g0 = [_clone(t) for t in params], [_clone(t) for t in bufs], [_clone(t) for t in grads]
    optim.reset_stats()
    with _Untouched(*grads):
        optim.sgd_momentum_(params, grads, bufs, 0.9, 1, -0.1)
    assert optim.stats() == {"edb_sgd": 1, "aten_sgd": 1}, optim.stats()
    p1, m1 = [_clone(t) for t in p0], [_clone(t) for t in m0]
    optim.sgd_momentum_(p1, g0, m1, 0.9, 1, -0.1)
    for i in (0, 3):
        assert _same_bits(params[i], p1[i]) and _same_bits(bufs[i], m1[i]), i
    for i in (1, 2):
        m64 = 0.9 * m0[i].double() + g0[i].double()
        p64 = p0[i].double() - 0.1 * m64
        for got, want in ((bufs[i], m64), (params[i], p64)):
            err = (got.double() - want).abs()
            assert bool((err <= 2 * 2.0 ** -24 * (want.abs() + m64.abs() + g0[i].double().abs())).all()), i


# ---- compiled steps ---------------------------------------------------------------------------

class _HeadModel(nn.Module):
    """A bias-free Linear(d, 3) head whose [B, T, 3] output is flattened for an MSE loss."""

    def __init__(self, d=64):
        super().__init__()
        self.fc = nn.Linear(d, d)
        self.head = nn.Linear(d, 3, bias=False)

    def forward(self, x, y):
        return F.mse_loss(self.head(torch.relu(self.fc(x))).reshape(-1), y)


class _PoolModel(nn.Module):
    """A loss on the column sums of a 2-D Linear output: the backward of sum(dim=0) is an expanded
    gradient, strides (0, 1), for the data- and weight-gradient GEMMs of `out`."""

    def __init__(self, d=64, n=64):
        super().__init__()
        self.fc = nn.Linear(d, d)
        self.out = nn.Linear(d, n)

    def forward(self, x, y):
        return F.mse_loss(self.out(torch.relu(self.fc(x))).sum(0) / x.shape[0], y)


def _batches(kind, steps):
    g = torch.Generator().manual_seed(11)
    if kind == "head":
        return [(torch.randn(4, 16, 64, generator=g), torch.randn(4 * 16 * 3, generator=g))
                for _ in range(steps)]
    return [(torch.randn(128, 64, generator=g), torch.randn(64, generator=g)) for _ in range(steps)]


def _eager(make, state, batches, dtype):
    model = make().to(device="cuda", dtype=dtype)
    model.load_state_dict({k: v.to(dtype) for k, v in state.items()})
    opt = torch.optim.SGD(model.parameters(), lr=1e-2, momentum=0.9, foreach=True)
    losses = []
    for x, y in batches:
        l = model(x.cuda().to(dtype), y.cuda().to(dtype))
        l.backward()
        opt.step()
        opt.zero_grad(True)
        losses.append(float(l.detach()))
    params = {k: v.detach().float() for k, v in model.named_parameters()}
    states = {k: {"momentum_buffer": opt.state[p]["momentum_buffer"].float()}
              for k, p in model.named_parameters()}
    return losses, params, states


@pytest.mark.parametrize("kind", ["head", "pool"])
def test_compiled_bf16_steps_on_gemm_output_layouts(rt, kind):
    """(head) gemm.mm's narrowed [*, 3] output flattened by a traced `view`; (pool) GEMMs handed
    an expanded gradient.  Losses, parameters and momentum buffers against eager PyTorch, at the
    tolerances of test_gpu_train.py."""
    from easydist_b200 import gemm
    from easydist_b200.api import easydist_compile
    from easydist_b200.workloads import gpt2_train_step
    from tools import parity as P
    make = _HeadModel if kind == "head" else _PoolModel
    torch.manual_seed(0)
    model = make().to(device="cuda", dtype=BF)
    state = {k: v.detach().float().clone() for k, v in model.state_dict().items()}
    opt = torch.optim.SGD(model.parameters(), lr=1e-2, momentum=0.9, foreach=True)
    step = easydist_compile(gpt2_train_step, parallel_mode="ddp", tracing_mode="fake", cuda_graph=False)
    batches = _batches(kind, 3)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        gemm.reset_stats()
        losses = [float(step(x.cuda().to(BF), y.cuda().to(BF), model, opt)) for x, y in batches]
        st = gemm.stats()
        ref_l, ref_p, ref_s = _eager(make, state, batches, torch.float32)
        _, van_p, van_s = _eager(make, state, batches, BF)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    assert st["edb_gemm"] > 0, st
    if kind == "pool":   # the expanded gradient's GEMMs: counted ATen
        assert st["aten_mm"] > 0, st
    for got, want in zip(losses, ref_l):
        assert math.isfinite(got) and abs(got - want) <= 3e-2 * abs(want), (losses, ref_l)
    got_p, got_s = P.compiled_state(step.compiled_func, ref_p, ref_s, 1)
    van = P.compare({k: v.bfloat16() for k, v in van_p.items()},
                    {k: {kk: vv.bfloat16() for kk, vv in s.items()} for k, s in van_s.items()},
                    ref_p, ref_s, low_precision=True)
    res = P.compare(got_p, got_s, ref_p, ref_s, low_precision=True)
    assert res["state_rel_l2"] <= max(2e-2, 2.0 * van["state_rel_l2"]), (res, van)
    assert res["param_max_ulp"] <= max(2.0, 2.0 * van["param_max_ulp"]), (res, van)


@pytest.mark.parametrize("name", ["gpt2-tiny", "gpt2-tiny-256", "llama-tiny"])
def test_tiny_model_steps_copy_nothing_for_the_norm_kernels(rt, monkeypatch, name):
    """The activations, gradients and parameters a compiled bf16 step hands LayerNorm and RMSNorm
    are dense and aligned already: the layout copy is never made, and every norm (but gpt2-tiny's
    LayerNorm: width 128 is no bf16 kernel width), activation, RoPE, loss and GEMM node runs
    natively.  gpt2-tiny-256 is gpt2-tiny at width 256, where LayerNorm runs natively."""
    import dataclasses
    from easydist_b200 import act, gemm, loss, norm, rope
    from easydist_b200.api import easydist_compile
    from easydist_b200.workloads import (GPT2, GPT2_CONFIGS, LLAMA_CONFIGS, Llama, gpt2_train_step,
                                         synthetic_tokens)
    copies = []
    dense = norm._dense

    def counting(t):
        out = dense(t)
        if out is not t:
            copies.append((tuple(t.shape), t.stride(), t.data_ptr() % 16))
        return out

    monkeypatch.setattr(norm, "_dense", counting)
    cfg = LLAMA_CONFIGS[name] if name.startswith("llama") else GPT2_CONFIGS["gpt2-tiny"]
    if name == "gpt2-tiny-256":
        cfg = dataclasses.replace(cfg, n_embd=256)
    torch.manual_seed(0)
    model = (GPT2 if name.startswith("gpt2") else Llama)(cfg).to(device="cuda", dtype=BF)
    opt = torch.optim.SGD(model.parameters(), lr=1e-3, momentum=0.9, foreach=True)
    step = easydist_compile(gpt2_train_step, parallel_mode="ddp", tracing_mode="fake", cuda_graph=False)
    for m in (act, gemm, loss, norm, rope):
        m.reset_stats()
    for b in range(2):
        tok, tgt = synthetic_tokens(cfg, 4, 64, seed=b, device="cuda")
        assert math.isfinite(float(step(tok, tgt, model, opt)))
    assert copies == [], copies
    nst, ast, rst, lst, gst = norm.stats(), act.stats(), rope.stats(), loss.stats(), gemm.stats()
    assert nst["aten_ln"] == (20 if name == "gpt2-tiny" else 0) and nst["aten_rms"] == 0, nst
    if name == "gpt2-tiny-256":
        assert nst["edb_ln_fwd"] > 0 and nst["edb_ln_bwd"] > 0, nst
    if name.startswith("llama"):
        assert nst["edb_rms_fwd"] > 0 and ast["edb_swiglu_fwd"] > 0 and rst["edb_rope_fwd"] > 0
    assert ast["aten_swiglu"] == 0 and rst["aten_rope"] == 0 and lst["aten_ce"] == 0, (ast, rst, lst)
    assert lst["edb_ce_fwd"] == 2 and gst["edb_gemm"] > 0 and gst["aten_mm"] == 0, (lst, gst)
    print(name, {"norm": nst, "act": ast, "rope": rst, "loss": lst,
                 "gemm": {k: v for k, v in gst.items() if k != "unsupported"}})
