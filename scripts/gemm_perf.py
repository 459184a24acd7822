"""Rates of the wgmma 3xTF32 GEMMs (gemm_tf32x3.cu) on the current GPU.

The TN kernel (C = A^T B, contraction over the long dimension: dW_self = H^T dS, the basis dV = Agg^T G) is timed
at the block layer's shape (K = V = 5 M, M = N = 512) and at the basis shape (K = 14 541, M = d*B = 2500, N = 500),
each next to the NT kernel at the same flop count (the self-loop product H @ W_self, the basis Agg @ V).  The
first block compares both kernels with cuBLAS fp32 at a few smaller shapes.  Rates count 2*M*N*K flop.
"""
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from relationprediction_b200 import ops  # noqa: E402


def t(f, n=10):
    f()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        f()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return "%s, %s" % (torch.cuda.get_device_name(), q)


print("card:", card())
for M, N, K in [(14541, 500, 500), (200000, 512, 512), (1000000, 512, 512)]:
    A = torch.randn(M, K, device="cuda"); B = torch.randn(K, N, device="cuda")
    t_ours = t(lambda: ops.gemm_tf32x3(A, B))
    t_torch = t(lambda: A @ B)
    fl = 2.0 * M * N * K
    print("M=%d N=%d K=%d  wgmma 3xTF32: %.3f ms (%.1f TFLOP/s fp32-equivalent)   cuBLAS fp32: %.3f ms (%.1f TFLOP/s)"
          % (M, N, K, t_ours, fl / t_ours / 1e9, t_torch, fl / t_torch / 1e9))
for K, M, N in [(14541, 500, 500), (200000, 512, 512)]:
    A = torch.randn(K, M, device="cuda"); B = torch.randn(K, N, device="cuda")
    t_ours = t(lambda: ops.gemm_tn_tf32x3(A, B))
    t_torch = t(lambda: A.T @ B)
    fl = 2.0 * M * N * K
    print("TN K=%d M=%d N=%d  wgmma 3xTF32: %.3f ms (%.1f TFLOP/s fp32-equivalent)   cuBLAS fp32: %.3f ms (%.1f TFLOP/s)"
          % (K, M, N, t_ours, fl / t_ours / 1e9, t_torch, fl / t_torch / 1e9))
del A, B

# TN against NT at the same flop count: (name, TN K, M, N, NT rows, NT inner dimension, NT columns)
for name, K, M, N, nt_m, nt_k, nt_n in [("block layer, dW_self = H^T dS", 5_000_000, 512, 512, 5_000_000, 512, 512),
                                        ("basis layer, dV = Agg^T G", 14541, 2500, 500, 14541, 2500, 500)]:
    fl = 2.0 * M * N * K
    A = torch.randn(K, M, device="cuda"); B = torch.randn(K, N, device="cuda")
    C = torch.empty(M, N, device="cuda")
    t_tn = t(lambda: ops.gemm_tn_tf32x3(A, B, out=C))
    del A, B, C
    X = torch.randn(nt_m, nt_k, device="cuda"); W = torch.randn(nt_k, nt_n, device="cuda")
    Y = torch.empty(nt_m, nt_n, device="cuda")
    t_nt = t(lambda: ops.gemm_tf32x3(X, W, out=Y))
    del X, W, Y
    print("%s: TN K=%d M=%d N=%d %.3f ms (%.1f TFLOP/s) | NT M=%d K=%d N=%d %.3f ms (%.1f TFLOP/s) | TN/NT %.2f"
          % (name, K, M, N, t_tn, fl / t_tn / 1e9, nt_m, nt_k, nt_n, t_nt, fl / t_nt / 1e9, t_tn / t_nt))
