"""GPU: the split-K schedule and the staged producer of the TN GEMM (k_gemm_tn_tf32x3, C (+)= A^T B with the
contraction over the long dimension) against float64 at the 1e-5 relative bar of test_gpu_gemm.py.

Covered: split and k-block boundaries (K not a multiple of 32, many splits), fewer k-blocks than SMs, more tiles
than one wave of CTAs holds, ragged M / N, the strided A of the basis backward (lda = 2 M), K = 0, and the block
layer's own shape K = V = 5 M, M = N = 512."""
import ctypes

import pytest
import torch

from relationprediction_b200 import _lib

pytestmark = pytest.mark.gpu


def rel(a, b):
    return float((a.double() - b).abs().max() / b.abs().max())


def gemm_tn(A, lda, B, C, M, N, K, accumulate):
    """C (+)= A^T B through the C-ABI; A may be a column slice of a wider row-major matrix (leading dimension lda)."""
    lib = _lib.load()
    rc = lib.rgcn_gemm_tn_tf32x3(ctypes.c_void_p(A.data_ptr()), lda, ctypes.c_void_p(B.data_ptr()), B.stride(0),
                                 ctypes.c_void_p(C.data_ptr()), C.stride(0), M, N, K, int(accumulate),
                                 ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    _lib.check(rc, "rgcn_gemm_tn_tf32x3")
    return C


def check(A, lda, B, M, N, K, ref, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = torch.full((M, N), float("nan"), device="cuda")    # accumulate=False must overwrite every element
    gemm_tn(A, lda, B, C, M, N, K, False)
    assert torch.isfinite(C).all()
    assert rel(C, ref) < 1e-5, rel(C, ref)
    C0 = torch.randn(M, N, device="cuda", generator=g)
    C1 = gemm_tn(A, lda, B, C0.clone(), M, N, K, True)
    assert rel(C1, ref + C0.double()) < 1e-5, rel(C1, ref + C0.double())


@pytest.mark.parametrize("K,M,N", [
    # K % 32 != 0, split boundaries inside the tile's k range (1 tile: one wave of many splits)
    (100_003, 128, 128), (50_001, 512, 512), (77_777, 384, 256),
    # fewer k-blocks than SMs: 2 and 4 k-blocks for 16 tiles
    (33, 512, 512), (100, 512, 512), (1, 512, 512),
    # more tiles than SMs would give one split each (80 tiles): the basis shape and a short K
    (14541, 2500, 500), (3000, 2500, 500), (40, 2500, 500),
    # ragged tiles
    (4097, 132, 36), (100_000, 132, 36), (31, 4, 4),
])
def test_gemm_tn_schedule_matches_float64(K, M, N):
    g = torch.Generator(device="cuda").manual_seed(K * 3 + M)
    A = torch.randn(K, M, device="cuda", generator=g)
    B = torch.randn(K, N, device="cuda", generator=g)
    check(A, M, B, M, N, K, A.double().T @ B.double(), K + N)


@pytest.mark.parametrize("K,M,N", [(14541, 2500, 500), (5000, 500, 200)])
def test_gemm_tn_strided_a_basis_layout(K, M, N):
    """A = saved[:, M:] of a [K, 2M] matrix with lda = 2M, as rgcn_basis_backward passes `saved + dB`."""
    g = torch.Generator(device="cuda").manual_seed(K + 1)
    saved = torch.randn(K, 2 * M, device="cuda", generator=g)
    B = torch.randn(K, N, device="cuda", generator=g)
    A = saved[:, M:]
    check(A, 2 * M, B, M, N, K, A.double().T @ B.double(), K)
    A0 = saved[:, :M]
    check(A0, 2 * M, B, M, N, K, A0.double().T @ B.double(), K + 2)


def test_gemm_tn_empty_contraction():
    A = torch.zeros(1, 512, device="cuda")   # never read: a valid pointer for the C-ABI
    B = torch.zeros(1, 512, device="cuda")
    C = torch.full((512, 512), 7.0, device="cuda")
    gemm_tn(A, 512, B, C, 512, 512, 0, True)
    assert bool((C == 7.0).all())
    gemm_tn(A, 512, B, C, 512, 512, 0, False)
    assert bool((C == 0.0).all())


def test_gemm_tn_block_layer_shape():
    """dW_self = H^T dS at V = 5 M, d = 512: the float64 reference is summed in k-chunks on the device."""
    K, M, N = 5_000_000, 512, 512
    g = torch.Generator(device="cuda").manual_seed(5)
    A = torch.randn(K, M, device="cuda", generator=g)
    B = torch.randn(K, N, device="cuda", generator=g)
    ref = torch.zeros(M, N, dtype=torch.float64, device="cuda")
    for k0 in range(0, K, 250_000):
        ref += A[k0:k0 + 250_000].double().T @ B[k0:k0 + 250_000].double()
    check(A, M, B, M, N, K, ref, 6)
