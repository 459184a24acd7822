"""CPU: the walk table of tests/compgcn_walks.py names exactly the `k_compgcn_*` kernels the built library contains.

Every `k_compgcn_*` instantiation in the library's SASS must be a walk some table row launches, and every kernel the
table names must exist.  Adding or deleting a walk variant therefore fails here until the table (and with it the GPU
test that runs every row) is updated."""
import shutil

import pytest

import compgcn_walks as cw
from relationprediction_b200 import _lib
from test_block_walk_table_host import _library_kernels


def test_table_rows_are_consistent():
    names = [r.name for r in cw.ROWS]
    assert len(names) == len(set(names))
    for r in cw.ROWS:
        assert r.d % 4 == 0 and r.d > 0, r
        assert r.nv == cw.nv_rule(r.d), r
        assert all(k == cw.canonical(k) for k in r.kernels), r
    for c in cw.COMPOSITIONS:   # one row per distinct kernel set
        assert [r.nv for r in cw.ROWS if r.composition == c] == [1, 2, 3, 4]
    assert any(cw.slabs(r.d, r.nv) > 1 for r in cw.ROWS)


def test_canonical_spelling_of_both_demanglers():
    assert cw.canonical("void <unnamed>::k_compgcn_bwd<(int)4, (int)1>(const WorkItem *, int)") == "k_compgcn_bwd<4,1>"
    assert cw.canonical("void (anonymous namespace)::k_compgcn_fwd<3, 0>(WorkItem const*, int)") == "k_compgcn_fwd<3,0>"
    assert cw.canonical("void <unnamed>::k_diaggcn_fwd<(int)3>(const WorkItem *, int)") is None


def test_every_compgcn_instantiation_is_in_the_table():
    if shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not on PATH")
    _lib.load()
    built = {c for c in map(cw.canonical, _library_kernels(raw=True)) if c is not None}
    known = cw.table_kernels()
    missing = sorted(built - known)
    stale = sorted(known - built)
    assert not missing, "k_compgcn_* kernels no table row launches: %s" % missing
    assert not stale, "table names kernels the library does not contain: %s" % stale
