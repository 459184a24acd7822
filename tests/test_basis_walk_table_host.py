"""CPU: the walk table of tests/basis_walks.py names exactly the basis-layer kernels the built library contains.

Every `k_basis_*` instantiation in the library's SASS must be a walk kernel some table row launches, and every
kernel the table names must exist.  Adding or deleting a walk variant therefore fails here until the table (and with
it the GPU test that runs every row) is updated."""
import shutil

import pytest

import basis_walks as bw
from relationprediction_b200 import _lib
from test_block_walk_table_host import _library_kernels


def test_table_rows_are_consistent():
    names = [r.name for r in bw.ROWS]
    assert len(names) == len(set(names))
    for r in bw.ROWS:
        assert r.kind in ("feat", "onehot"), r
        assert r.d % 4 == 0 and r.d > 0 and r.B > 0, r
        assert r.bc == bw.bc_rule(r.B), r
        assert r.nv == bw.nv_rule(r.d), r
        if r.onehot:
            assert r.nv_dc == bw.nv_rule(r.d, dc_variant=True), r
        assert r.fwd and r.bwd, r
        assert all(k == bw.canonical(k) for k in r.kernels), r
    feat = [r for r in bw.ROWS if not r.onehot]
    onehot = [r for r in bw.ROWS if r.onehot]
    pairs = [(bc, nv) for bc in (1, 2, 4, 5) for nv in (1, 2, 3, 4)]
    assert {(r.bc, r.nv) for r in feat} == set(pairs)
    assert {(r.bc, r.nv_dc) for r in onehot} == {p for p in pairs if p[1] <= 2}
    assert {r.nv for r in onehot} == {1, 2, 3, 4}
    # the boundaries the table exists for: partial and exact multi-pass, two slabs at two BC values, exact widths
    assert {r.B for r in feat} >= {3, 6, 8, 9} and any(r.passes == 3 for r in feat)
    assert len({r.bc for r in feat if bw.slabs(r.d, r.nv) > 1}) >= 2
    assert any(r.d % 512 == 4 for r in feat) and any(r.d == 1024 for r in feat)
    for nv in (1, 2, 3, 4):
        widths = {r.d for r in feat if r.nv == nv}
        assert any(w % 128 for w in widths) and any(w == 128 * nv for w in widths), nv


def test_canonical_spelling_of_both_demanglers():
    assert bw.canonical("void <unnamed>::k_basis_agg<(int)4, (int)2, (int)1, (bool)1>(AggLaunch, const float *, "
                        "int, int, float *, float *, long, const float *, const float *, float *)") == \
        "k_basis_agg<4,2,1,true>"
    assert bw.canonical("void (anonymous namespace)::k_basis_dc<5, 3>(AggLaunch, float const*, int, int, float*)") \
        == "k_basis_dc<5,3>"
    assert bw.canonical("void <unnamed>::k_basis_onehot_push<(int)3>(const WorkItem *, int)") == \
        "k_basis_onehot_push<3>"
    assert bw.canonical("void <unnamed>::k_block_rel<4, 1, true>(WorkItem const*, int)") is None


def test_every_basis_walk_instantiation_is_in_the_table():
    if shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None:
        pytest.skip("cuobjdump / cu++filt not on PATH")
    _lib.load()
    built = {c for c in map(bw.canonical, _library_kernels(raw=True)) if c is not None}
    assert len(built) >= 56
    known = bw.table_kernels()
    missing = sorted(built - known)
    stale = sorted(known - built)
    assert not missing, "basis walk kernels no table row launches: %s" % missing
    assert not stale, "table names kernels the library does not contain: %s" % stale
