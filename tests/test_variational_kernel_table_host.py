"""CPU: the kernel table of tests/variational_kernels.py names exactly the `k_var_*` kernels the built library contains,
and every other kernel it names exists.  Adding or deleting a kernel of the variational head therefore fails here until
the table (and with it the GPU launch check) is updated."""
import shutil

import pytest

import variational_kernels as vk
from relationprediction_b200 import _lib
from test_block_walk_table_host import _library_kernels


def family(kernel):
    """a canonical() prefix that matches `kernel` (the prefix must be followed by at least one name character)"""
    return kernel.split("<")[0][:-1]


def test_table_spelling():
    for row in vk.ROWS.values():
        for k in row:
            assert vk.canonical(k, family(k)) == k, k
    assert vk.canonical("void <unnamed>::k_gemm_tf32x3<(int)3>(const float *, long)", family("k_gemm_tf32x3")) == \
        "k_gemm_tf32x3<3>"
    assert vk.canonical("void (anonymous namespace)::k_var_prologue(float4 const*, long)") == "k_var_prologue"


def test_every_variational_kernel_is_in_the_table():
    if shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not on PATH")
    _lib.load()
    names = _library_kernels(raw=True)
    built = {c for c in map(vk.canonical, names) if c is not None}
    missing = sorted(built - vk.table_kernels())
    stale = sorted(vk.table_kernels() - built)
    assert not missing, "k_var_* kernels no table row launches: %s" % missing
    assert not stale, "table names kernels the library does not contain: %s" % stale
    for k in vk.SHARED:
        assert k in {vk.canonical(n, family(k)) for n in names}, k
