"""Micro-benchmark of the TMA-fed wgmma GEMM (csrc/gemm_tma.cu) on the stage-1 GPT shapes against the tap kernel and cuBLAS TF32."""
import os, sys, torch, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from easevoice_trainer_b200 import lib, ops
L = lib.init()
dev = torch.device("cuda", 0)
def bench(fn, n=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n
for M, N, K in ((20480, 1536, 512), (20480, 512, 512), (20480, 2048, 512), (20480, 512, 2048), (16384, 1028, 512)):
    a = torch.randn(M, K, device=dev); b = torch.randn(N, K, device=dev); bias = torch.zeros(N, device=dev)
    out = torch.empty(M, N, device=dev)
    fl = 2.0 * M * N * K
    for tma in (1, 0):
        L.evk_set_backend_tma(tma)
        w = ops.pack_weight(b)
        with torch.no_grad():
            ms = bench(lambda: ops.linear(a.unsqueeze(0), w, bias))
        print(f"M{M} N{N} K{K} tma={tma}: {ms:.3f} ms  {fl/ms/1e9:.1f} TF/s", flush=True)
    ms = bench(lambda: ops.gemm_tf32(a, b, out=out))
    print(f"   direct gemm_tf32: {ms:.3f} ms {fl/ms/1e9:.1f} TF/s")
    torch.backends.cuda.matmul.allow_tf32 = True
    ms = bench(lambda: torch.matmul(a, b.t()))
    print(f"   cuBLAS tf32: {ms:.3f} ms {fl/ms/1e9:.1f} TF/s", flush=True)
# wgrad shape: dW[N][C] = dY^T X : A = dY^T [N][rows], B = X^T [C][rows]
for N, C, R in ((2048, 512, 20480), (512, 512, 20480), (1536, 512, 20480)):
    a = torch.randn(N, R, device=dev); b = torch.randn(C, R, device=dev); out = torch.zeros(N, C, device=dev)
    fl = 2.0 * N * C * R
    for sp in (1, 4, 8, 16):
        ms = bench(lambda: ops.gemm_tf32(a, b, out=out, splits=sp))
        print(f"wgrad N{N} C{C} R{R} splits={sp}: {ms:.3f} ms {fl/ms/1e9:.1f} TF/s", flush=True)
