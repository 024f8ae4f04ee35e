"""Tile-width sweep of the wgmma GEMM vs cuBLAS (tuning aid)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from easydist_b200 import runtime, gemm
rt = runtime.init(0, 1, 0, heap_bytes=1 << 30)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
def timeit(f, iters=15, do_flush=True):
    for _ in range(3): f()
    ts = []
    for _ in range(iters):
        if do_flush: flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); f(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort(); return ts[len(ts)//2]
shapes = [(4096,1024,1024),(4096,4096,1024),(4096,1024,4096),(4096,3072,1024),(8192,8192,8192),(4096,50257,1024),(16384,4096,4096)]
for (M,N,K) in shapes:
    a = torch.randn(M,K,device="cuda",dtype=torch.bfloat16); w = torch.randn(N,K,device="cuda",dtype=torch.bfloat16)
    fl = 2*M*N*K
    t_ref = timeit(lambda: torch.mm(a, w.t()))
    t_ref_warm = timeit(lambda: torch.mm(a, w.t()), do_flush=False)
    row = [f"cublas {t_ref*1e3:7.1f}us {fl/t_ref/1e9:5.0f}TF (warm {t_ref_warm*1e3:.1f}us)"]
    for bn in (128,256):
        rt.set_option("gemm_force_bn", bn)
        t = timeit(lambda: gemm.mm(a, w.t()))
        tw = timeit(lambda: gemm.mm(a, w.t()), do_flush=False)
        row.append(f"bn{bn} {t*1e3:7.1f}us {fl/t/1e9:5.0f}TF (warm {tw*1e3:.1f})")
    print(f"{(M,N,K)}: " + " | ".join(row), flush=True)
