"""CPU: the walk table of tests/gcn_diag_walks.py names exactly the `k_diaggcn_*` kernels the built library contains.

Every `k_diaggcn_*` instantiation in the library's SASS must be a walk some table row launches, and every kernel the
table names must exist.  Adding or deleting a walk variant therefore fails here until the table (and with it the GPU
test that runs every row) is updated."""
import shutil

import pytest

import gcn_diag_walks as gw
from relationprediction_b200 import _lib
from test_block_walk_table_host import _library_kernels


def test_table_rows_are_consistent():
    names = [r.name for r in gw.ROWS]
    assert len(names) == len(set(names))
    for r in gw.ROWS:
        assert r.d % 4 == 0 and r.d > 0, r
        assert r.nv == gw.nv_rule(r.d), r
        assert all(k == gw.canonical(k) for k in r.kernels), r
    assert [r.nv for r in gw.ROWS] == [1, 2, 3, 4]          # one row per distinct kernel set
    assert any(gw.slabs(r.d, r.nv) > 1 for r in gw.ROWS)


def test_canonical_spelling_of_both_demanglers():
    assert gw.canonical("void <unnamed>::k_diaggcn_bwd<(int)4>(const WorkItem *, int)") == "k_diaggcn_bwd<4>"
    assert gw.canonical("void (anonymous namespace)::k_diaggcn_fwd<3>(WorkItem const*, int)") == "k_diaggcn_fwd<3>"
    assert gw.canonical("void <unnamed>::k_diagcoef_fwd<(int)3>(const WorkItem *, int)") is None


def test_every_diaggcn_instantiation_is_in_the_table():
    if shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not on PATH")
    _lib.load()
    built = {c for c in map(gw.canonical, _library_kernels(raw=True)) if c is not None}
    known = gw.table_kernels() | set(gw.HELPERS)
    missing = sorted(built - known)
    stale = sorted(known - built)
    assert not missing, "k_diaggcn_* kernels no table row launches: %s" % missing
    assert not stale, "table names kernels the library does not contain: %s" % stale
