"""First-contact probe on an H100: runtime bring-up, local reshard ops, GEMM layouts + timing.
Run on the GPU machine; prints one line per check. Not a test (tests/ holds the parity tests)."""
import sys, traceback
import torch
sys.path.insert(0, ".")
from easydist_b200 import runtime, reshard, gemm

def section(name):
    print(f"\n=== {name}", flush=True)

def run(name, fn):
    try:
        r = fn()
        print(f"[ok]   {name} {r if r is not None else ''}", flush=True)
    except Exception as e:
        print(f"[FAIL] {name}: {type(e).__name__}: {e}", flush=True)
        traceback.print_exc()

section("runtime")
rt = runtime.init(rank=0, world=1, device=0, heap_bytes=2 << 30)
print("heap", hex(rt.heap_base), rt.heap_bytes, "sm", rt.get_option("sm_count"))
def cai():
    buf = rt.alloc(1 << 20)
    t = buf.tensor(torch.float32, (256, 1024))
    t.fill_(3.0)
    torch.cuda.synchronize()
    assert float(rt.slab[buf.offset:buf.offset+4].view(torch.float32)[0]) == 3.0
run("slab tensor view", cai)

section("local reshard ops")
def t_scatter():
    for shape, dim, n in [((8, 6, 10), 0, 2), ((8, 6, 10), 1, 3), ((8, 6, 10), 2, 4), ((7,), 0, 3), ((5, 4096), 1, 8), ((4, 128, 1024), 2, 4)]:
        for dt in (torch.float32, torch.bfloat16, torch.int64, torch.uint8):
            x = (torch.arange(int(torch.tensor(shape).prod()), device="cuda") % 251).to(dt).view(shape)
            chunks = torch.chunk(x, n, dim)
            for i in range(len(chunks)):
                y = reshard.scatter_wrapper(x, n, dim, i)
                assert torch.equal(y, chunks[i].contiguous()), (shape, dim, n, i, dt)
run("scatter_wrapper == torch.chunk", t_scatter)
def t_copy():
    a = torch.zeros(1000003, device="cuda"); b = torch.randn(1000003, device="cuda")
    reshard.copy_wrapper(a, b); assert torch.equal(a, b)
run("copy_wrapper", t_copy)
def t_n1():
    g = [0]
    x = torch.randn(4, 6, 8, device="cuda")
    for d in range(3):
        assert torch.equal(reshard.all_gather_start(x, d, g), x)
        assert torch.equal(reshard.reduce_scatter_start(x, "sum", d, g), x)
    assert torch.equal(reshard.all_reduce_start(x, "sum", g), x)
    assert torch.allclose(reshard.all_reduce_start(x, "avg", g), x)
    assert torch.equal(reshard.all_to_all_start(x, 0, 2, 1, 0, g), x)
    xb = x.bfloat16()
    assert torch.equal(reshard.reduce_scatter_start(xb, "sum", 1, g, _out_dtype=torch.float32), xb.float())
run("collectives at n=1 are identities", t_n1)
def t_bw():
    x = torch.empty(1 << 28, dtype=torch.uint8, device="cuda").random_(0, 255)  # 256 MiB
    y = torch.empty_like(x)
    for _ in range(3): reshard.copy_wrapper(y, x)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(10): reshard.copy_wrapper(y, x)
    ev[1].record(); torch.cuda.synchronize()
    ms = ev[0].elapsed_time(ev[1]) / 10
    ev[0].record()
    for _ in range(10): y.copy_(x)
    ev[1].record(); torch.cuda.synchronize()
    ms_t = ev[0].elapsed_time(ev[1]) / 10
    return f"edb_copy {2*x.numel()/ms/1e6:.0f} GB/s  torch copy_ {2*x.numel()/ms_t/1e6:.0f} GB/s"
run("copy bandwidth 256MiB", t_bw)

section("gemm")
def ref_mm(a, b):
    return (a.float() @ b.float())
def t_gemm(M, N, K, a_k, b_k):
    torch.manual_seed(0)
    A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    B = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
    a = A if a_k else A.t().contiguous().t()
    b = B.t().contiguous().t() if b_k else B
    gemm.reset_stats()
    c = gemm.mm(a, b)
    torch.cuda.synchronize()
    assert gemm.stats()["edb_gemm"] == 1, gemm.stats()
    r = ref_mm(A, B)
    err = (c.float() - r).abs().max().item()
    tol = 0.02 * r.abs().max().item() + 1e-2
    assert err <= tol, f"max err {err} tol {tol}"
    return f"err {err:.3g} (tol {tol:.3g})"
for (M, N, K) in [(128, 128, 64), (128, 256, 128), (256, 512, 256), (4096, 1024, 1024), (384, 200, 136), (4096, 4096, 1024)]:
    for a_k in (True, False):
        for b_k in (True, False):
            run(f"gemm M{M} N{N} K{K} a_k={a_k} b_k={b_k}", lambda: t_gemm(M, N, K, a_k, b_k))

def bench(M, N, K, a_k=True, b_k=True):
    A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    B = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
    a = A if a_k else A.t().contiguous().t()
    b = B.t().contiguous().t() if b_k else B
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    def timeit(f, iters=20):
        for _ in range(3): f()
        ts = []
        for _ in range(iters):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); f(); e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        return ts[len(ts)//2]
    t_edb = timeit(lambda: gemm.mm(a, b))
    t_ref = timeit(lambda: torch.mm(a, b))
    fl = 2 * M * N * K
    return f"edb {t_edb*1e3:.1f}us {fl/t_edb/1e9:.0f} TF/s | cublas {t_ref*1e3:.1f}us {fl/t_ref/1e9:.0f} TF/s"
for shp in [(4096, 1024, 1024), (4096, 4096, 1024), (4096, 1024, 4096), (4096, 3072, 1024), (8192, 8192, 8192)]:
    for lay in [(True, True), (True, False), (False, False)]:
        run(f"bench {shp} a_k={lay[0]} b_k={lay[1]}", lambda: bench(*shp, *lay))
print("launches", rt.launch_count())
