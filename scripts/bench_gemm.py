"""dev: TFLOP/s of the dense wgmma GEMM on the prefill shapes (CUDA events, 20 iterations after 5 warm-ups)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from controlar_b200 import engine
for (M, N, K) in [(1920, 3584, 1280), (1920, 1280, 3584), (1920, 3840, 1280), (16384, 1280, 1280), (8192, 8192, 8192)]:
    x = torch.randn(M, K, device="cuda").to(torch.bfloat16); w = torch.randn(N, K, device="cuda").to(torch.bfloat16)
    for _ in range(5): engine.op_dense_linear(x, w)
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(20): engine.op_dense_linear(x, w)
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / 20 * 1e3
    t0, t1 = torch.cuda.Event(True), torch.cuda.Event(True)
    for _ in range(5): x @ w.t()
    torch.cuda.synchronize(); t0.record()
    for _ in range(20): x @ w.t()
    t1.record(); torch.cuda.synchronize()
    us_t = t0.elapsed_time(t1) / 20 * 1e3
    print(f"M {M} N {N} K {K}: ours {us:.1f} us = {2*M*N*K/us/1e6:.0f} TFLOP/s | cuBLAS {us_t:.1f} us = {2*M*N*K/us_t/1e6:.0f} TFLOP/s", flush=True)
