"""GPU check of the wgmma 3xTF32 GEMM against float64."""
import os, sys, time
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from evotorch_b200 import ops

torch.manual_seed(0)
dev = "cuda"
ok = True
for (M, N, K) in [(128, 256, 32), (128, 256, 64), (128, 256, 1024), (256, 512, 96), (4096, 1024, 1024), (1024, 1024, 4096), (100, 70, 36), (129, 257, 40), (12, 6, 6)]:
    A = torch.randn(M, K, device=dev)
    B = torch.randn(N, K, device=dev)
    ref = (A.double() @ B.double().T)
    C = ops.gemm_nt(A, B)
    torch.cuda.synchronize()
    err = float((C.double() - ref).abs().max() / ref.abs().max())
    t32 = float(((A @ B.T).double() - ref).abs().max() / ref.abs().max())
    good = err < 3e-6
    ok &= good
    print(f"M={M} N={N} K={K}: max rel err {err:.2e} (torch fp32 matmul {t32:.2e}) {'OK' if good else 'FAIL'}", flush=True)
# fused second output
M, N, K = 4096, 1024, 1024
A = torch.randn(M, K, device=dev); B = torch.randn(N, K, device=dev)
alpha = torch.tensor(0.37, device=dev); bias = torch.randn(N, device=dev)
C2 = torch.empty(M, N, device=dev)
C = ops.gemm_nt(A, B, out2=C2, alpha=alpha, bias=bias)
ref = A.double() @ B.double().T
e2 = float((C2.double() - (0.37 * ref + bias.double())).abs().max() / ref.abs().max())
print("fused epilogue rel err", e2); ok &= e2 < 3e-6
# transpose_scale
Y = torch.randn(300, 70, device=dev); w = torch.randn(300, device=dev)
T = ops.transpose_scale(Y, w)
print("transpose ok", bool(torch.equal(T, (Y * w[:, None]).T.contiguous()))); ok &= bool(torch.equal(T, (Y * w[:, None]).T.contiguous()))
# timing
def timeit(fn, reps=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / reps
for (M, N, K) in [(4096, 1024, 1024), (1024, 1024, 4096), (8192, 8192, 8192)]:
    A = torch.randn(M, K, device=dev); B = torch.randn(N, K, device=dev); out = torch.empty(M, N, device=dev)
    t = timeit(lambda: ops.gemm_nt(A, B, out))
    tt = timeit(lambda: torch.matmul(A, B.T, out=out))
    print(f"M={M} N={N} K={K}: evok 3xTF32 {t:.3f} ms ({2*M*N*K/t/1e9:.1f} TFLOP/s fp32-equivalent, {6*M*N*K/t/1e9:.1f} TF32 tensor TFLOP/s) | torch fp32 {tt:.3f} ms ({2*M*N*K/tt/1e9:.1f} TFLOP/s)")
print("GEMM_CHECK", "PASS" if ok else "FAIL")
