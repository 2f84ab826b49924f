"""K6 throughput: ops.gemm_nt at CMA-ES and square sizes (3xTF32 on wgmma), torch fp32 matmul (no TF32) beside it."""
import json
import sys

import torch

sys.path.insert(0, ".")
from evotorch_b200 import ops

torch.backends.cuda.matmul.allow_tf32 = False
dev = "cuda"


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


for (M, N, K) in [(2048, 1000, 1000), (1000, 1000, 2048), (4096, 4096, 4096), (8192, 8192, 8192)]:
    A = torch.randn(M, K, device=dev)
    B = torch.randn(N, K, device=dev)
    ms = timed(lambda: ops.gemm_nt(A, B), 20)
    ms_t = timed(lambda: A @ B.T, 20)
    print(json.dumps({"M": M, "N": N, "K": K, "evok_ms": ms, "evok_tflops_fp32_equiv": 2.0 * M * N * K / ms / 1e9, "torch_fp32_ms": ms_t,
                      "torch_tflops": 2.0 * M * N * K / ms_t / 1e9}))
