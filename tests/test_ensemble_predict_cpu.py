"""R-GCN+ ensemble top-k and relation prediction without a GPU: the (u, id) order of the float64 restatement on
hand-built energies (saturated ones included), Ensemble's argument checks and RelationCount check, the Scorer's
wiring with a stub ranker, the ensemble command's query mode arguments, and the new C-ABI entry points' argument
checks (they run before any device work)."""
import ctypes
import math

import numpy as np
import pytest

import ensemble_topk_oracle as tko
from relationprediction_b200 import _lib
from relationprediction_b200 import ensemble as ens
from relationprediction_b200.common import evaluation


# ---- the (u, id) order --------------------------------------------------------------------------------------------
def test_saturated_energies_tie_in_float32_but_not_in_u():
    e = np.array([[20.0, 40.0, 200.0, 600.0, 40.0, -3.0]])
    s32 = 1.0 / (1.0 + np.exp(-e.astype(np.float32)))
    assert s32[0, 1] == s32[0, 2] == s32[0, 3] == 1.0                  # the float32 sigmoid cannot tell them apart
    u = tko.u_of(0.5, e, e)
    assert len(set(u[0, :4].tolist())) == 4 and np.all(u[0, :4] > 0)
    ids, uu, sc = tko.top_k(u, 4)
    assert ids.tolist() == [[3, 2, 1, 4]]                                # 600, 200, then the tie 40 / 40 by id
    np.testing.assert_array_equal(sc, 1.0 - uu)


def test_mixed_members_and_weights():
    ea = np.array([[1.0, 2.0, 3.0]])
    eb = np.array([[3.0, 2.0, 1.0]])
    assert tko.top_k(tko.u_of(1.0, ea, eb), 3)[0].tolist() == [[2, 1, 0]]
    assert tko.top_k(tko.u_of(0.0, ea, eb), 3)[0].tolist() == [[0, 1, 2]]
    assert tko.top_k(tko.u_of(0.5, ea, eb), 3)[0].tolist() == [[1, 0, 2]]   # u(1) < u(0) = u(2): ties by id


def test_padding_and_exclusions():
    u = tko.u_of(0.5, np.array([[1.0, 2.0, 3.0], [0.0, 0.0, 0.0]]), np.zeros((2, 3)))
    ids, uu, sc = tko.top_k(u, 5, [[2], [0, 1, 2]])
    assert ids.tolist() == [[1, 0, -1, -1, -1], [-1] * 5]
    assert np.all(np.isinf(uu[:, 2:])) and np.all(sc[:, 2:] == 0) and np.all(np.isinf(uu[1]))


def test_check_top_k_allows_only_near_ties_to_swap():
    u = np.array([[0.1, 0.1 * (1 + 1e-7), 0.5]])
    tko.check_top_k(np.array([[1, 0]]), u[:, [1, 0]], 1 - u[:, [1, 0]], u, 2)   # a 1e-7 swap is allowed
    with pytest.raises(AssertionError):
        v = np.array([[0.1, 0.2, 0.5]])
        tko.check_top_k(np.array([[1, 0]]), v[:, [1, 0]], 1 - v[:, [1, 0]], v, 2)


# ---- Ensemble and Scorer --------------------------------------------------------------------------------------------
class Member(object):
    def __init__(self, V=10, R=4):
        self.entity_count, self.relation_count = V, R


def test_relation_count_must_match():
    with pytest.raises(ValueError, match="relation set"):
        ens.Ensemble(Member(R=4), Member(R=5), 0.5)
    assert ens.Ensemble(Member(R=4), Member(R=4), 0.5).relation_count == 4


def test_argument_checks_come_before_the_fused_path():
    e = ens.Ensemble(Member(), Member(), 0.5)
    tri = np.array([[0, 1, 2]])
    for k in (0, 129):
        with pytest.raises(ValueError, match="k must be"):
            e.predict_top_k(tri, k, 1)
        with pytest.raises(ValueError, match="k must be"):
            e.predict_top_k_relations(tri, k)
    with pytest.raises(ValueError, match="side"):
        e.predict_top_k(tri, 5, 2)
    with pytest.raises(ValueError, match="entity ids"):
        e.predict_top_k(np.array([[0, 1, 10]]), 5, 1)
    with pytest.raises(ValueError, match="relation ids"):
        e.predict_top_k(np.array([[0, 4, 1]]), 5, 1)
    with pytest.raises(ValueError, match="relation ids"):
        e.rank_all_relations(np.array([[0, -1, 1]]), [[]])
    with pytest.raises(ValueError, match="entity ids"):
        e.predict_top_k_relations(np.array([[-1, 0, 1]]), 5)
    for call in (lambda: e.predict_top_k(tri, 5, 1), lambda: e.predict_top_k_relations(tri, 5),
                 lambda: e.rank_all_relations(tri, [[1]])):
        with pytest.raises(NotImplementedError, match="fused"):
            call()                                      # the stub members have no fused ranker


def test_scorer_wiring_with_a_stub_ranker(monkeypatch):
    """Scorer.predict_top_k / predict_top_k_relations / compute_relation_mrr_scores reach the Ensemble with the
    filtered exclusion lists and read (ids, u, scores) as they read a single model's (ids, energies, scores)."""
    import torch
    e = ens.Ensemble(Member(V=6, R=3), Member(V=6, R=3), 0.5)
    seen = {}

    class Ranker(object):
        a = type("A", (), {"codes": torch.zeros((6, 4))})()

        def top_k(self, X, side, k, mask):
            seen["top_k"] = (X.tolist(), side, k, None if mask is None else mask.tolist())
            n = X.shape[0]
            return (torch.arange(k, dtype=torch.int32).repeat(n, 1), torch.full((n, k), 0.25, dtype=torch.float64),
                    torch.full((n, k), 0.75, dtype=torch.float64))

        def top_k_relations(self, X, k, mask):
            seen["rel"] = (X.tolist(), k, None if mask is None else mask.tolist())
            n = X.shape[0]
            return (torch.zeros((n, k), dtype=torch.int32), torch.zeros((n, k), dtype=torch.float64),
                    torch.ones((n, k), dtype=torch.float64))

        def rank_relations(self, X, mask):
            seen["rank"] = (X.tolist(), mask.tolist())
            n = X.shape[0]
            return torch.full((n,), 2, dtype=torch.int32), torch.ones(n, dtype=torch.int32)

    monkeypatch.setattr(e, "_fused_ranker", lambda what, tri: Ranker())
    scorer = evaluation.Scorer()
    scorer.register_data(np.array([[0, 1, 2], [0, 2, 2], [3, 1, 2]]))
    scorer.register_model(e)
    ids, u, sc = scorer.predict_top_k(np.array([[0, 1, 0]]), 2, 1)
    assert ids.tolist() == [[0, 1]] and u.dtype == np.float64 and sc.tolist() == [[0.75, 0.75]]
    assert seen["top_k"][1:3] == (1, 2) and seen["top_k"][3] == [[1 << 2]]          # (0, 1, ?) knows object 2
    scorer.predict_top_k(np.array([[0, 1, 2]]), 2, 0)
    assert seen["top_k"][3] == [[(1 << 0) | (1 << 3)]]                             # (?, 1, 2) knows subjects 0, 3
    scorer.predict_top_k_relations(np.array([[0, 0, 2]]), 3)
    assert seen["rel"][2] == [[(1 << 1) | (1 << 2)]]                               # (0, ?, 2) knows relations 1, 2
    assert scorer.predict_top_k_relations(np.array([[0, 0, 2]]), 3, filtered=False) is not None
    assert seen["rel"][2] is None
    score = scorer.compute_relation_mrr_scores(np.array([[0, 1, 2], [3, 1, 2]]))
    assert score.raw_ranks == [2, 2] and score.filtered_ranks == [1, 1]
    assert seen["rank"][1] == [[(1 << 1) | (1 << 2)], [1 << 1]]
    from relationprediction_b200 import predict
    rows = predict.answer(scorer, [(0, 1, -1, 1), (0, -1, 2, 2)], 2, filtered=True)
    assert rows[0] == (0, 1, 0, 0.75) and rows[2][0] == 1


# ---- the command's query mode ------------------------------------------------------------------------------------
BASE = ["--dataset", "D", "--member", "a", "b", "--member", "c", "d"]


def test_query_mode_arguments():
    args = ens.parse_args(BASE + ["--queries", "q.txt", "--k", "10", "--out", "o.txt"])
    assert (args.queries, args.k, args.out, args.raw, args.relation_metrics) == ("q.txt", 10, "o.txt", False, False)
    assert ens.parse_args(BASE + ["--queries", "q", "--k", "1", "--out", "o", "--raw"]).raw
    assert ens.parse_args(BASE + ["--relation-metrics"]).relation_metrics
    args = ens.parse_args(BASE)
    assert (args.queries, args.k, args.out, args.raw, args.relation_metrics) == (None, None, None, False, False)
    for bad in (["--queries", "q", "--out", "o"], ["--queries", "q", "--k", "5"],
                ["--queries", "q", "--k", "0", "--out", "o"], ["--queries", "q", "--k", "129", "--out", "o"],
                ["--k", "5"], ["--out", "o"], ["--raw"],
                ["--queries", "q", "--k", "5", "--out", "o", "--relation-metrics"],
                ["--queries", "q", "--k", "5", "--out", "o", "--split", "test"],
                ["--queries", "q", "--k", "5", "--out", "o", "--limit", "3"]):
        with pytest.raises(SystemExit):
            ens.parse_args(BASE + bad)


def test_query_mode_reports_a_bad_query_file(tmp_path, monkeypatch):
    from relationprediction_b200 import train as driver
    monkeypatch.setattr(driver, "load_dataset", lambda d: ({}, {0: "e0", 1: "e1"}, {0: "r0"}))
    q = tmp_path / "q.txt"
    q.write_text("e0\tr0\t?\ne0\tnope\t?\n")
    with pytest.raises(SystemExit, match="line 2: unknown relation"):
        ens.main(BASE + ["--queries", str(q), "--k", "3", "--out", str(tmp_path / "o.txt")])


# ---- C-ABI --------------------------------------------------------------------------------------------------------
def _buf():
    buf = np.zeros(1 << 16, np.float32)
    return buf, ctypes.c_void_p(buf.ctypes.data)


def _topk(lib, dec_a=0, dec_b=1, d_a=8, d_b=12, V=300, weight=0.5, n=4, side=1, k=10, ws_bytes=None, codes_a=True,
          X=True, ids=True, u=True, ws=True):
    buf, p = _buf()
    if ws_bytes is None:
        ws_bytes = 1 << 40
    return lib.rgcn_ensemble_topk(dec_a, p if codes_a else None, p, 7, d_a, dec_b, p, p, 7, d_b, V, weight,
                                  p if X else None, n, side, k, None, 0, p if ids else None, p if u else None, p,
                                  p if ws else None, ws_bytes, None)


def _rel(lib, entry, dec_a=0, dec_b=1, d_a=8, d_b=12, V=300, R=7, Vrel_a=7, Vrel_b=7, weight=0.5, n=4, k=10,
         ws_bytes=None, X=True, out=True, known=False, filt=False, ws=True):
    buf, p = _buf()
    if ws_bytes is None:
        ws_bytes = 1 << 40
    if entry == "rank":
        return lib.rgcn_ensemble_relation_rank(dec_a, p, p, Vrel_a, d_a, dec_b, p, p, Vrel_b, d_b, V, R, weight,
                                               p if X else None, n, p if known else None, 0, p if out else None,
                                               p if filt else None, p if ws else None, ws_bytes, None)
    return lib.rgcn_ensemble_relation_topk(dec_a, p, p, Vrel_a, d_a, dec_b, p, p, Vrel_b, d_b, V, R, weight,
                                           p if X else None, n, k, None, 0, p if out else None, p, p,
                                           p if ws else None, ws_bytes, None)


def _rejects(lib, rc, who, needle):
    assert rc == -1
    msg = lib.rgcn_last_error()
    assert who in msg and needle in msg, msg


def test_topk_entry_point_rejects_bad_arguments():
    lib = _lib.load()
    who = b"rgcn_ensemble_topk"
    for kw, needle in ((dict(dec_a=2), b"unknown decoder"), (dict(dec_b=-1), b"unknown decoder"),
                       (dict(d_a=6), b"d % 4"), (dict(d_b=0), b"d % 4"), (dict(weight=-0.5), b"weight"),
                       (dict(weight=math.nan), b"weight"), (dict(k=0), b"k = 0"), (dict(k=129), b"k = 129"),
                       (dict(side=2), b"side"), (dict(codes_a=False), b"null pointer"), (dict(X=False), b"null pointer"),
                       (dict(ids=False), b"null pointer"), (dict(u=False), b"null pointer"),
                       (dict(ws=False), b"null pointer"), (dict(V=0), b"bad size")):
        _rejects(lib, _topk(lib, **kw), who, needle)
    need = lib.rgcn_ensemble_topk_workspace_bytes(300, 8, 12, 4, 10)
    assert need > 0
    assert _topk(lib, ws_bytes=need - 1) == -4 and b"workspace too small" in lib.rgcn_last_error()


@pytest.mark.parametrize("entry", ["rank", "topk"])
def test_relation_entry_points_reject_bad_arguments(entry):
    lib = _lib.load()
    who = b"rgcn_ensemble_relation_" + entry.encode()
    cases = [(dict(dec_a=3), b"unknown decoder"), (dict(d_b=10), b"d % 4"), (dict(weight=2.0), b"weight"),
             (dict(R=0), b"R = 0"), (dict(R=8), b"R = 8"), (dict(Vrel_b=6), b"R = 7"), (dict(X=False), b"null pointer"),
             (dict(out=False), b"null pointer"), (dict(ws=False), b"null pointer")]
    if entry == "rank":
        cases.append((dict(filt=True), b"known mask"))
    else:
        cases += [(dict(k=0), b"k = 0"), (dict(k=200), b"k = 200")]
    for kw, needle in cases:
        _rejects(lib, _rel(lib, entry, **kw), who, needle)
    need = (lib.rgcn_ensemble_relation_rank_workspace_bytes(7, 8, 12, 4) if entry == "rank"
            else lib.rgcn_ensemble_relation_topk_workspace_bytes(7, 8, 12, 4, 10))
    assert need > 0
    assert _rel(lib, entry, ws_bytes=need - 1) == -4 and b"workspace too small" in lib.rgcn_last_error()


def test_workspace_bytes():
    lib = _lib.load()
    for args in ((0, 8, 8, 4, 10), (100, 6, 8, 4, 10), (100, 8, 8, -1, 10), (100, 8, 8, 4, 0), (100, 8, 8, 4, 129)):
        assert lib.rgcn_ensemble_topk_workspace_bytes(*args) == -1, args
        assert lib.rgcn_ensemble_relation_topk_workspace_bytes(*args) == -1, args
    assert lib.rgcn_ensemble_relation_rank_workspace_bytes(0, 8, 8, 4) == -1
    V, da, db = 14541, 500, 200
    head = lib.rgcn_ensemble_rank_workspace_bytes(V, da, db, 0)
    assert lib.rgcn_ensemble_topk_workspace_bytes(V, da, db, 0, 10) == head        # the same split head
    n1, n2 = 1000, 2000
    for k, kt in ((10, 10), (128, 64)):
        grow = (lib.rgcn_ensemble_topk_workspace_bytes(V, da, db, n2, k)
                - lib.rgcn_ensemble_topk_workspace_bytes(V, da, db, n1, k))
        per_row = 2 * (da + db) * 4 + ((V + 63) // 64) * kt * 16                  # Q hi/lo + (u, id) candidates
        assert abs(grow - (n2 - n1) * per_row) <= 2048
    assert (lib.rgcn_ensemble_relation_rank_workspace_bytes(237, da, db, 100)
            == lib.rgcn_ensemble_rank_workspace_bytes(237, da, db, 100))
