"""CPU: the kernel table of tests/gemm_kernels.py names exactly the `k_gemm_*` and `k_split_*` kernels the built library
contains.  Adding or deleting a GEMM kernel or epilogue therefore fails here until the table (and with it the GPU test
that runs every row against float64) is updated."""
import shutil

import pytest

import gemm_kernels as gk
from relationprediction_b200 import _lib
from test_block_walk_table_host import _library_kernels


def test_table_spelling():
    for k in gk.ROWS:
        assert gk.canonical(k) == k, k
    assert gk.canonical("void <unnamed>::k_gemm_ensemble<<unnamed>::EnsTopKEpi>(int, int, int, <unnamed>::EnsTopKEpi)") \
        == "k_gemm_ensemble<EnsTopKEpi>"
    assert gk.canonical("void (anonymous namespace)::k_gemm_ensemble<(anonymous namespace)::EnsRankEpi>(int, int, "
                        "int, (anonymous namespace)::EnsRankEpi)") == "k_gemm_ensemble<EnsRankEpi>"
    assert gk.canonical("void <unnamed>::k_gemm_tf32x3<(int)6>(const float *, long, const float *)") == \
        "k_gemm_tf32x3<6>"
    assert gk.canonical("void (anonymous namespace)::k_split_b(float const*, long, int)") == "k_split_b"
    assert gk.canonical("void <unnamed>::k_conve_split_w(const float *)") is None
    assert not set(gk.ROWS) & set(gk.UNREACHABLE)


def test_every_gemm_kernel_is_in_the_table():
    if shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not on PATH")
    _lib.load()
    built = {c for c in map(gk.canonical, _library_kernels(raw=True)) if c is not None}
    missing = sorted(built - gk.table_kernels())
    stale = sorted(gk.table_kernels() - built)
    assert not missing, "GEMM kernels no table row names: %s" % missing
    assert not stale, "table names kernels the library does not contain: %s" % stale
