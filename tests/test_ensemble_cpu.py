"""R-GCN+ ensemble without a GPU: the Ensemble's score-matrix path and the numpy oracle against the reference tool's
own ranks (tests/golden/reference_ensemble_golden.npz, see make_ensemble_golden.py), the C-ABI argument checks (they
run before any device work), the workspace size, Ensemble's constructor errors and the command's arguments."""
import ctypes
import math
import os

import numpy as np
import pytest

import ensemble_oracle as oracle
from relationprediction_b200 import _lib
from relationprediction_b200 import ensemble as ens
from relationprediction_b200.common import evaluation

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_ensemble_golden.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


class StubModel(object):
    """A member that returns stored float32 score matrices, rows by test triple."""

    def __init__(self, test, subj, obj, entity_count):
        self.row = {tuple(t): i for i, t in enumerate(np.asarray(test).tolist())}
        self.subj, self.obj, self.entity_count = subj, obj, entity_count

    def _rows(self, triples):
        return [self.row[tuple(t)] for t in np.asarray(triples).tolist()]

    def score_all_subjects(self, triples):
        return self.subj[self._rows(triples)]

    def score_all_objects(self, triples):
        return self.obj[self._rows(triples)]


def _scorer(g):
    scorer = evaluation.Scorer()
    for name in ("train", "valid", "test"):
        scorer.register_data(g[name])
    return scorer


def _members(g):
    V = int(g["V"])
    return (StubModel(g["test"], g["sa_subjects"], g["sa_objects"], V),
            StubModel(g["test"], g["sb_subjects"], g["sb_objects"], V))


def test_fallback_path_gives_the_reference_tool_ranks(golden):
    """The tool ranks subjects then objects of every test triple by #{others >= target} + 1; the Scorer's filtered
    ranks of an Ensemble are the same list (one chunk: under 1000 triples)."""
    a, b = _members(golden)
    scorer = _scorer(golden)
    for i, w in enumerate(golden["weights"]):
        model = ens.Ensemble(a, b, float(w))
        assert not model.supports_fused_ranking()
        scorer.register_model(model)
        score = scorer.compute_scores(golden["test"])
        np.testing.assert_array_equal(np.asarray(score.filtered_ranks), golden["ranks"][i])
        res = score.get_summary().results["Filtered"]
        got = [res["MRR"], res["H@1"], res["H@3"], res["H@10"]]
        np.testing.assert_allclose(got, golden["metrics"][i], rtol=0, atol=1e-12)
    np.testing.assert_allclose(golden["metrics"][0], golden["printed"], rtol=0, atol=1e-12)   # the tool's output


def test_numpy_oracle_gives_the_reference_tool_ranks(golden):
    scorer = _scorer(golden)
    test = golden["test"]
    tl = test.tolist()
    known = {0: [scorer.known_subject_triples[(t[2], t[1])] for t in tl],
             1: [scorer.known_object_triples[(t[0], t[1])] for t in tl]}
    for i, w in enumerate(golden["weights"]):
        got = []
        for side, key, col in ((0, "subjects", 0), (1, "objects", 2)):
            c = oracle.combine(w, golden["sa_" + key], golden["sb_" + key])
            raw, filt = oracle.ranks(c, test[:, col], known[side])
            assert np.all(raw >= filt)
            got.append(filt)
        np.testing.assert_array_equal(np.concatenate(got), golden["ranks"][i])


def test_golden_has_the_ties_it_was_made_for(golden):
    for key in ("sa_subjects", "sb_subjects", "sa_objects", "sb_objects"):
        s = golden[key]
        assert (s == 1.0).mean() > 0.05 and (s == 0.5).mean() > 0.05
    c = oracle.combine(0.5, golden["sa_subjects"], golden["sb_subjects"])
    gold = c[np.arange(len(c)), golden["test"][:, 0]]
    assert ((c == gold[:, None]).sum(1) > 1).mean() > 0.2     # the gold ties with another entity in many rows


def test_weight_one_and_zero_select_a_member_in_the_oracle(golden):
    sa, sb = golden["sa_subjects"], golden["sb_subjects"]
    gold = golden["test"][:, 0]
    np.testing.assert_array_equal(oracle.ranks(oracle.combine(1.0, sa, sb), gold)[0],
                                  oracle.ranks(sa.astype(np.float64), gold)[0])
    np.testing.assert_array_equal(oracle.ranks(oracle.combine(0.0, sa, sb), gold)[0],
                                  oracle.ranks(sb.astype(np.float64), gold)[0])
    for w in (0.0, 0.3, 0.5, 1.0):   # a model with itself: the combination of one float32 value is strictly monotone
        np.testing.assert_array_equal(oracle.ranks(oracle.combine(w, sa, sa), gold)[0],
                                      oracle.ranks(sa.astype(np.float64), gold)[0])


# ---- C-ABI ------------------------------------------------------------------------------------------------------
def _call(lib, dec_a=0, dec_b=1, d_a=8, d_b=12, V=300, weight=0.5, n=4, side=1, ws_bytes=None, known=False,
          filt=False, codes_a=True, codes_b=True, rel_a=True, X=True, raw=True, ws=True):
    buf = np.zeros(1 << 16, np.float32)
    p = ctypes.c_void_p(buf.ctypes.data)
    if ws_bytes is None:
        ws_bytes = max(lib.rgcn_ensemble_rank_workspace_bytes(V if V > 0 else 1, 8, 12, max(n, 0)), 0)
    return lib.rgcn_ensemble_rank(dec_a, p if codes_a else None, p if rel_a else None, 7, d_a,
                                  dec_b, p if codes_b else None, p, 7, d_b, V, weight, p if X else None, n, side,
                                  p if known else None, 0, p if raw else None, p if filt else None, p if ws else None,
                                  ws_bytes, None)


def test_entry_point_rejects_bad_arguments():
    lib = _lib.load()
    cases = ((dict(dec_a=2), b"unknown decoder"), (dict(dec_b=-1), b"unknown decoder"),
             (dict(d_a=6), b"d % 4"), (dict(d_b=10), b"d % 4"), (dict(d_a=0), b"d % 4"),
             (dict(weight=-0.01), b"weight"), (dict(weight=1.5), b"weight"), (dict(weight=math.nan), b"weight"),
             (dict(weight=math.inf), b"weight"), (dict(codes_a=False), b"null pointer"),
             (dict(codes_b=False), b"null pointer"), (dict(rel_a=False), b"null pointer"),
             (dict(X=False), b"null pointer"), (dict(raw=False), b"null pointer"), (dict(ws=False), b"null pointer"),
             (dict(V=0), b"bad size"), (dict(n=-1), b"bad size"), (dict(side=2), b"side"), (dict(side=-1), b"side"),
             (dict(filt=True), b"known mask"))
    for kw, needle in cases:
        assert _call(lib, **kw) == -1, kw
        msg = lib.rgcn_last_error()
        assert b"rgcn_ensemble_rank" in msg and needle in msg, (kw, msg)
    need = lib.rgcn_ensemble_rank_workspace_bytes(300, 8, 12, 4)
    assert _call(lib, ws_bytes=need - 1) == -4
    assert b"workspace too small" in lib.rgcn_last_error()
    assert _call(lib, dec_a=1, dec_b=1, ws_bytes=need - 1, known=True, filt=True) == -4   # valid otherwise


def test_workspace_bytes():
    lib = _lib.load()
    for args in ((0, 8, 8, 4), (100, 0, 8, 4), (100, 8, 6, 4), (100, 8, 8, -1), (100, 8, 8, 1 << 31)):
        assert lib.rgcn_ensemble_rank_workspace_bytes(*args) == -1, args
    V, da, db = 14541, 500, 200
    base = lib.rgcn_ensemble_rank_workspace_bytes(V, da, db, 0)
    assert base >= 2 * V * (da + db) * 4                                    # both members' hi/lo splits
    n1, n2 = 1000, 10000
    grow = lib.rgcn_ensemble_rank_workspace_bytes(V, da, db, n2) - lib.rgcn_ensemble_rank_workspace_bytes(V, da, db, n1)
    per_row = 2 * (da + db) * 4 + 5 * 4                                     # Q hi/lo of both members + five vectors
    assert abs(grow - (n2 - n1) * per_row) <= 2048


# ---- Python layer -----------------------------------------------------------------------------------------------
def test_ensemble_constructor_errors(golden):
    a, b = _members(golden)
    b.entity_count = a.entity_count + 1
    with pytest.raises(ValueError, match="entity set"):
        ens.Ensemble(a, b, 0.5)
    b.entity_count = a.entity_count
    for w in (-0.1, 1.01, math.nan, math.inf):
        with pytest.raises(ValueError, match="weight"):
            ens.Ensemble(a, b, w)
    assert ens.Ensemble(a, b, 1).weight == 1.0


def test_ensemble_ranker_refuses_other_rankers():
    from relationprediction_b200 import ops
    with pytest.raises(TypeError, match="DistMultRanker"):
        ops.EnsembleRanker(object(), object(), 0.5)


def test_command_arguments():
    args = ens.parse_args(["--dataset", "D", "--member", "gcn.exp", "gcn.pt", "--member", "dm.exp", "dm.pt"])
    assert args.member == [["gcn.exp", "gcn.pt"], ["dm.exp", "dm.pt"]]
    assert args.weight == 0.5 and args.split == "test" and args.limit is None and args.device == "cuda:0"
    args = ens.parse_args(["--dataset-npz", "F.npz", "--member", "a", "b", "--member", "c", "d", "--weight", "0.3",
                           "--split", "valid", "--limit", "7", "--device", "cuda:1"])
    assert (args.weight, args.split, args.limit, args.device, args.dataset_npz) == (0.3, "valid", 7, "cuda:1", "F.npz")
    for bad in (["--member", "a", "b", "--member", "c", "d"],                            # no dataset
                ["--dataset", "D", "--dataset-npz", "F", "--member", "a", "b", "--member", "c", "d"],
                ["--dataset", "D", "--member", "a", "b"],                                 # one member
                ["--dataset", "D"] + ["--member", "a", "b"] * 3,                          # three members
                ["--dataset", "D", "--member", "a", "b", "--member", "c", "d", "--weight", "1.5"],
                ["--dataset", "D", "--member", "a", "b", "--member", "c", "d", "--weight", "nan"],
                ["--dataset", "D", "--member", "a", "b", "--member", "c", "d", "--split", "train"],
                ["--dataset", "D", "--member", "a", "b", "--member", "c", "d", "--limit", "0"],
                ["--dataset", "D", "--member", "a"]):
        with pytest.raises(SystemExit):
            ens.parse_args(bad)
