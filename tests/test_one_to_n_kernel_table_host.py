"""CPU: the kernel table of tests/one_to_n_kernels.py names exactly the `k_onen_*` kernels the built library contains,
and every other kernel it names exists.  Adding or deleting a kernel of 1-N training therefore fails here until the
table (and with it the GPU launch check) is updated."""
import shutil

import pytest

import one_to_n_kernels as ok
from relationprediction_b200 import _lib
from test_block_walk_table_host import _library_kernels


def family(kernel):
    """a canonical() prefix that matches `kernel` (the prefix must be followed by at least one name character)"""
    return kernel.split("<")[0][:-1]


def test_table_spelling():
    for row in ok.ROWS.values():
        for k in row:
            assert ok.canonical(k, family(k)) == k, k
    assert ok.canonical("void <unnamed>::k_gemm_tf32x3<(int)5>(const float *, long)", family("k_gemm_tf32x3")) == \
        "k_gemm_tf32x3<5>"
    assert ok.canonical("void (anonymous namespace)::k_onen_labels(long const*, int)") == "k_onen_labels"


def test_every_one_to_n_kernel_is_in_the_table():
    if shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not on PATH")
    _lib.load()
    names = _library_kernels(raw=True)
    built = {c for c in map(ok.canonical, names) if c is not None}
    missing = sorted(built - ok.table_kernels())
    stale = sorted(ok.table_kernels() - built)
    assert not missing, "k_onen_* kernels no table row launches: %s" % missing
    assert not stale, "table names kernels the library does not contain: %s" % stale
    for k in ok.SHARED:
        assert k in {ok.canonical(n, family(k)) for n in names}, k
