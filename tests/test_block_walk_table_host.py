"""CPU: the walk table of tests/block_walks.py names exactly the block-layer kernels the built library contains.

Every `k_block_*` instantiation in the library's SASS must be a walk kernel some table row launches, a listed
UNREACHABLE instantiation, or one of the non-walk kernels.  Adding or deleting a walk variant therefore fails here
until the table (and with it the GPU test that runs every row) is updated."""
import shutil
import subprocess

import pytest

import block_walks as bw
from relationprediction_b200 import _lib


def _library_kernels(raw=False):
    """canonical `k_block_*` names of the kernels in the library's SASS (raw=True: every demangled kernel name)"""
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    mangled = [f.split("\n", 1)[0].strip() for f in sass.split("Function : ")[1:]]
    names = subprocess.run(["cu++filt"], input="\n".join(mangled) + "\n", capture_output=True, text=True,
                           check=True).stdout.splitlines()
    assert len(names) == len(mangled)
    if raw:
        return names
    return {c for c in map(bw.canonical, names) if c is not None}


def test_table_rows_are_consistent():
    names = [r.name for r in bw.ROWS]
    assert len(names) == len(set(names))
    for r in bw.ROWS:
        assert r.d % 4 == 0 and r.d % r.s == 0, r
        assert r.algo in (-1, 0, 1, 3), r
        assert r.fwd and r.bwd, r
        assert all(k == bw.canonical(k) for k in r.kernels), r
        assert not set(r.kernels) & set(bw.NON_WALK), r
    assert not bw.table_kernels() & set(bw.UNREACHABLE)


def test_canonical_spelling_of_both_demanglers():
    assert bw.canonical("void <unnamed>::k_block_team<(int)8, (int)1, (bool)1, (bool)0, (int)4, (int)3, (int)2, "
                        "(int)8>(const WorkItem *, int)") == "k_block_team<8,1,true,false,4,3,2,8>"
    assert bw.canonical("void (anonymous namespace)::k_block_rel<4, 1, true>(WorkItem const*, int)") == \
        "k_block_rel<4,1,true>"
    assert bw.canonical("<unnamed>::k_block_relayout(const float *, int)") == "k_block_relayout"
    assert bw.canonical("void gemm_kernel<4>(float*)") is None


def test_every_walk_instantiation_is_in_the_table():
    if shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not on PATH")
    _lib.load()
    built = _library_kernels()
    known = bw.table_kernels() | set(bw.UNREACHABLE) | set(bw.NON_WALK)
    assert len(built) > 80
    missing = sorted(built - known)
    stale = sorted(known - built)
    assert not missing, "walk kernels no table row launches and not listed as unreachable: %s" % missing
    assert not stale, "table names kernels the library does not contain: %s" % stale
