"""GPU: the wgmma 3xTF32 GEMM (gemm_tf32x3.cu) against a float64 reference -- fp32-level accuracy
(1e-5 relative, an order tighter than the layer bar) at the layer's shapes, ragged edges included."""
import numpy as np
import pytest
import torch

from relationprediction_b200 import _lib, ops

pytestmark = pytest.mark.gpu


def rel(a, b):
    return float((a.double() - b).abs().max() / b.abs().max())


def walk_rows(m):
    """M itself, or for "<t>w" the rows that give every persistent CTA t tiles of a one-tile-wide output"""
    if isinstance(m, str):
        return 128 * int(m[:-1]) * torch.cuda.get_device_properties(0).multi_processor_count
    return m


def gemm_strided(A, B, b_is_nk, C, accumulate=False):
    """rgcn_gemm_tf32x3 on views whose leading dimensions (stride(0)) may exceed their widths"""
    M, K = A.shape
    N = B.shape[0] if b_is_nk else B.shape[1]
    ws = torch.empty(2 * N * K, device="cuda")
    _lib.check(_lib.load().rgcn_gemm_tf32x3(ops._ptr(A), A.stride(0), ops._ptr(B), B.stride(0), int(b_is_nk),
                                            ops._ptr(C), C.stride(0), M, N, K, int(accumulate), ops._ptr(ws),
                                            ws.numel() * 4, ops._stream(A.device)), "rgcn_gemm_tf32x3")
    return C


@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (128, 128, 128), (256, 256, 64), (14541, 500, 500),
                                   (1000, 512, 512), (77, 8, 8), (300, 200, 200), (129, 132, 36),
                                   (5000, 24, 40),
                                   # many tiles per persistent CTA (one / two / sixteen k-blocks per tile)
                                   (100000, 512, 512), (40000, 132, 32), (30000, 24, 40),
                                   # tile and k-block edges: one partial k-block, exactly one, and 1 / 2 / 3 / 4 / 16
                                   # k-blocks (total_g = 0, 1, 2 mod 3 for the producer's unroll and the stage ring)
                                   (1, 4, 4), (127, 124, 28), (128, 128, 96), (129, 132, 100), (1, 128, 512),
                                   # every CTA walks exactly 1, 2 or 16 tiles
                                   ("1w", 128, 32), ("2w", 124, 36), ("16w", 4, 96)])
@pytest.mark.parametrize("b_is_nk", [False, True])
def test_gemm_tf32x3_matches_float64(M, N, K, b_is_nk):
    M = walk_rows(M)
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N)
    A = torch.randn(M, K, device="cuda", generator=g)
    B = torch.randn(*((N, K) if b_is_nk else (K, N)), device="cuda", generator=g)
    ref = A.double() @ (B.double().T if b_is_nk else B.double())
    C = ops.gemm_tf32x3(A, B, b_is_nk=b_is_nk, out=torch.full((M, N), float("nan"), device="cuda"))   # overwritten
    assert torch.isfinite(C).all()
    assert rel(C, ref) < 1e-5, rel(C, ref)
    # accumulate form
    C0 = torch.randn(M, N, device="cuda", generator=g)
    C1 = ops.gemm_tf32x3(A, B, b_is_nk=b_is_nk, out=C0.clone(), accumulate=True)
    assert rel(C1, ref + C0.double()) < 1e-5


def test_gemm_tf32x3_is_tighter_than_single_tf32_and_handles_scales():
    g = torch.Generator(device="cuda").manual_seed(1)
    A = torch.randn(2048, 512, device="cuda", generator=g) * 1e3
    B = torch.randn(512, 512, device="cuda", generator=g) * 1e-3
    ref = A.double() @ B.double()
    assert rel(ops.gemm_tf32x3(A, B), ref) < 1e-5
    # strided A (leading dimension > K)
    big = torch.randn(700, 1000, device="cuda", generator=g)
    Av = big[:, :500]
    Bm = torch.randn(500, 500, device="cuda", generator=g)
    lib_out = gemm_strided(Av, Bm, False, torch.empty(700, 500, device="cuda"))
    assert rel(lib_out, Av.double() @ Bm.double()) < 1e-5


@pytest.mark.parametrize("M,N,K", [(1, 4, 4), (129, 132, 36), (300, 124, 100), (257, 128, 500)])
@pytest.mark.parametrize("b_is_nk", [False, True])
@pytest.mark.parametrize("accumulate", [False, True])
def test_gemm_tf32x3_padded_leading_dimensions(M, N, K, b_is_nk, accumulate):
    """lda > K, ldb > K (or > N for B [K, N]) and ldc > N, as ConvE and CompGCN call the NT kernel: the padding
    columns of C keep their bits.  Every operand has a spare row after it, so a read past K stays in its buffer."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(M + 1, K + 12, device="cuda", generator=g)[:M, :K]
    B = torch.randn(*((N + 1, K + 4) if b_is_nk else (K + 1, N + 8)), device="cuda", generator=g)
    B = B[:N, :K] if b_is_nk else B[:K, :N]
    Cbuf = torch.randn(M + 1, N + 8, device="cuda", generator=g)
    before = Cbuf.clone()
    ref = A.double() @ (B.double().T if b_is_nk else B.double()) + (Cbuf[:M, :N].double() if accumulate else 0)
    gemm_strided(A, B, b_is_nk, Cbuf[:M, :N], accumulate)
    assert rel(Cbuf[:M, :N], ref) < 1e-5
    assert torch.equal(Cbuf[:M, N:].view(torch.int32), before[:M, N:].view(torch.int32))
    assert torch.equal(Cbuf[M:].view(torch.int32), before[M:].view(torch.int32))


@pytest.mark.parametrize("K,M,N", [(128, 128, 128), (1000, 128, 128), (14541, 500, 500), (50000, 512, 512),
                                   (33, 8, 8), (4097, 132, 36), (3000, 2500, 500), (100, 200, 24)])
def test_gemm_tn_tf32x3_matches_float64(K, M, N):
    g = torch.Generator(device="cuda").manual_seed(K + M)
    A = torch.randn(K, M, device="cuda", generator=g)
    B = torch.randn(K, N, device="cuda", generator=g)
    ref = A.double().T @ B.double()
    C = ops.gemm_tn_tf32x3(A, B)
    assert torch.isfinite(C).all()
    assert rel(C, ref) < 1e-5, rel(C, ref)
    C0 = torch.randn(M, N, device="cuda", generator=g)
    C1 = ops.gemm_tn_tf32x3(A, B, out=C0.clone(), accumulate=True)
    assert rel(C1, ref + C0.double()) < 1e-5
