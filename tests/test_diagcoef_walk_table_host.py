"""CPU: the walk table of tests/diagcoef_walks.py names exactly the `k_diagcoef_*` kernels the built library contains.

Every `k_diagcoef_*` instantiation in the library's SASS must be a walk some table row launches or one of the layer's
helpers, and every kernel the table names must exist.  Adding or deleting a walk variant therefore fails here until
the table (and with it the GPU test that runs every row) is updated."""
import shutil

import pytest

import diagcoef_walks as dw
from relationprediction_b200 import _lib
from test_block_walk_table_host import _library_kernels


def test_table_rows_are_consistent():
    names = [r.name for r in dw.ROWS]
    assert len(names) == len(set(names))
    for r in dw.ROWS:
        assert r.d % 4 == 0 and r.d > 0 and r.B > 0, r
        assert r.bc == dw.bc_rule(r.B) and r.nv == dw.nv_rule(r.d) and r.nvb == dw.nv_rule(r.d, cap=2), r
        assert all(k == dw.canonical(k) for k in r.kernels), r
        assert not set(r.kernels) & set(dw.HELPERS), r
    assert {r.nv for r in dw.ROWS} == {1, 2, 3, 4}
    assert {(r.bc, r.nvb) for r in dw.ROWS} == {(bc, nv) for bc in (1, 2, 4, 5) for nv in (1, 2)}
    assert any(r.B == 100 for r in dw.ROWS) and any(r.passes > 1 and r.B % r.bc for r in dw.ROWS)
    assert any(dw.slabs(r.d, r.nv) > 1 for r in dw.ROWS) and any(dw.slabs(r.d, r.nvb) > 2 for r in dw.ROWS)


def test_canonical_spelling_of_both_demanglers():
    assert dw.canonical("void <unnamed>::k_diagcoef_dp<(int)4, (int)2>(const WorkItem *, int)") == \
        "k_diagcoef_dp<4,2>"
    assert dw.canonical("void (anonymous namespace)::k_diagcoef_fwd<3>(WorkItem const*, int)") == "k_diagcoef_fwd<3>"
    assert dw.canonical("void <unnamed>::k_diagcoef_colsum(const float *, long, int, float *)") == "k_diagcoef_colsum"
    assert dw.canonical("void <unnamed>::k_basis_agg<(int)4, (int)2, (int)1, (bool)1>(AggLaunch)") is None


def test_every_diagcoef_instantiation_is_in_the_table():
    if shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not on PATH")
    _lib.load()
    built = {c for c in map(dw.canonical, _library_kernels(raw=True)) if c is not None}
    known = dw.table_kernels() | set(dw.HELPERS)
    missing = sorted(built - known)
    stale = sorted(known - built)
    assert not missing, "k_diagcoef_* kernels no table row launches: %s" % missing
    assert not stale, "table names kernels the library does not contain: %s" % stale
