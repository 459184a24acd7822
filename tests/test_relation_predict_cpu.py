"""Relation prediction without a GPU: argument checks of the relation C-ABI (they run before any device work), the
workspace sizes, the ops layer's refusal of CPU tensors, the Scorer's known-relation lists and what it hands the
model, and the predict command's relation queries with the model stubbed."""
import ctypes

import numpy as np
import pytest
import torch

from relationprediction_b200 import _lib, ops
from relationprediction_b200 import predict as predict_cmd
from relationprediction_b200.common import evaluation

RANKS = ("distmult_relation_rank", "rgcn_complex_relation_rank")
TOPKS = ("distmult_relation_topk", "rgcn_complex_relation_topk")


def _buf():
    buf = np.zeros(1 << 16, np.float32)
    return buf, ctypes.c_void_p(buf.ctypes.data)


def _rank(lib, name, V=300, Vrel=300, R=237, d=8, n=4, ws_bytes=None, codes=True, rel=True, X=True, raw=True,
          filt=False, mask=False, ws=True):
    buf, p = _buf()
    if ws_bytes is None:
        ws_bytes = max(lib.rgcn_relation_rank_workspace_bytes(max(R, 1), d if d > 0 and d % 4 == 0 else 8, n), 0)
    return getattr(lib, name)(p if codes else None, p if rel else None, V, Vrel, R, d, p if X else None, n,
                              p if mask else None, 0, p if raw else None, p if filt else None, p if ws else None,
                              ws_bytes, None)


def _topk(lib, name, V=300, Vrel=300, R=237, d=8, n=4, k=10, ws_bytes=None, codes=True, rel=True, X=True, ids=True,
          energies=True, ws=True):
    buf, p = _buf()
    if ws_bytes is None:
        ws_bytes = max(lib.rgcn_relation_topk_workspace_bytes(max(R, 1), d if d > 0 and d % 4 == 0 else 8, n,
                                                              min(max(k, 1), 128)), 0)
    return getattr(lib, name)(p if codes else None, p if rel else None, V, Vrel, R, d, p if X else None, n, k, None,
                              0, p if ids else None, p if energies else None, p if ws else None, ws_bytes, None)


COMMON = ((dict(R=0), b"R = 0"), (dict(R=301), b"R = 301"), (dict(R=-2), b"1 <= R <= Vrel"),
          (dict(R=20, Vrel=10), b"Vrel = 10"), (dict(d=6), b"d % 4"), (dict(d=0), b"bad arguments"),
          (dict(V=0), b"bad arguments"), (dict(codes=False), b"bad arguments"), (dict(rel=False), b"bad arguments"),
          (dict(X=False), b"bad arguments"), (dict(ws=False), b"bad arguments"))


@pytest.mark.parametrize("name", RANKS)
def test_rank_entry_points_reject_bad_arguments(name):
    lib = _lib.load()
    for kw, needle in COMMON + ((dict(raw=False), b"bad arguments"), (dict(filt=True), b"known mask")):
        assert _rank(lib, name, **kw) == -1, kw
        msg = lib.rgcn_last_error()
        assert name.encode() in msg and needle in msg, (kw, msg)
    need = lib.rgcn_relation_rank_workspace_bytes(237, 8, 4)
    assert _rank(lib, name, ws_bytes=need - 1) == -4
    assert b"workspace too small" in lib.rgcn_last_error()
    assert _rank(lib, name, filt=True, mask=True, ws_bytes=need - 1) == -4   # a filtered call passes the checks


@pytest.mark.parametrize("name", TOPKS)
def test_topk_entry_points_reject_bad_arguments(name):
    lib = _lib.load()
    for kw, needle in COMMON + ((dict(k=0), b"k = 0"), (dict(k=129), b"k = 129"), (dict(k=-3), b"out of range"),
                                (dict(ids=False), b"bad arguments"), (dict(energies=False), b"bad arguments")):
        assert _topk(lib, name, **kw) == -1, kw
        msg = lib.rgcn_last_error()
        assert name.encode() in msg and needle in msg, (kw, msg)
    need = lib.rgcn_relation_topk_workspace_bytes(237, 8, 4, 10)
    assert _topk(lib, name, ws_bytes=need - 1) == -4
    assert b"workspace too small" in lib.rgcn_last_error()


def test_workspace_bytes_reject_bad_input_and_grow_with_n_and_k():
    lib = _lib.load()
    for args in ((0, 8, 4), (-1, 8, 4), (100, 0, 4), (100, 6, 4), (100, 8, -1), (100, 512, 1 << 60)):
        assert lib.rgcn_relation_rank_workspace_bytes(*args) == -1, args
    for args in ((0, 8, 4, 10), (100, 0, 4, 10), (100, 6, 4, 10), (100, 8, -1, 10), (100, 8, 4, 0),
                 (100, 8, 4, 129), (1 << 30, 512, 1 << 40, 128)):
        assert lib.rgcn_relation_topk_workspace_bytes(*args) == -1, args
    R, d = 237, 500
    base = lib.rgcn_relation_rank_workspace_bytes(R, d, 0)
    assert base >= 2 * R * d * 4                                    # the hi/lo split of rel[0:R]
    assert base < 2 * 14541 * d * 4                                 # ... not of a [V, d] table
    by_n = [lib.rgcn_relation_rank_workspace_bytes(R, d, n) for n in (1, 100, 1000, 10000)]
    assert all(a < b for a, b in zip(by_n, by_n[1:]))
    assert abs((by_n[3] - by_n[2]) - 9000 * (4 * d + 16)) <= 2048    # query row + 4 ints per query
    by_n = [lib.rgcn_relation_topk_workspace_bytes(R, d, n, 10) for n in (1, 100, 1000, 10000)]
    assert all(a < b for a, b in zip(by_n, by_n[1:]))
    assert abs((by_n[3] - by_n[2]) - 9000 * (4 * d + 2 * 10 * 8)) <= 1024   # two 128-relation tiles of k pairs
    by_k = [lib.rgcn_relation_topk_workspace_bytes(R, d, 1000, k) for k in (1, 10, 100, 128)]
    assert all(a < b for a, b in zip(by_k, by_k[1:]))
    # the split sits in the same place in both, so one relation workspace serves rank and top-k
    assert lib.rgcn_relation_topk_workspace_bytes(R, d, 0, 1) == base


@pytest.mark.parametrize("cls", [ops.DistMultRanker, ops.ComplexRanker])
def test_ops_refuse_cpu_tensors(cls):
    with pytest.raises(_lib.RgcnError, match="CUDA"):
        cls(torch.zeros(10, 8), torch.zeros(10, 8), 3)


class StubModel(object):
    """Records what the Scorer hands the relation paths; answers top-k with relation ids in order and ranks 1, 2."""

    def __init__(self):
        self.calls = []

    def predict_top_k_relations(self, triples, k, exclude_lists=None):
        self.calls.append(("top", np.asarray(triples).copy(), k, exclude_lists))
        n = len(triples)
        ids = np.tile(np.arange(k, dtype=np.int64), (n, 1))
        energies = np.tile(-np.arange(k, dtype=np.float32), (n, 1))
        return ids, energies, 1.0 / (1.0 + np.exp(-energies))

    def rank_all_relations(self, triples, known_relation_lists):
        self.calls.append(("rank", np.asarray(triples).copy(), known_relation_lists))
        n = len(triples)
        return np.arange(n, dtype=np.int64) + 2, np.ones(n, np.int64)

    def predict_top_k(self, triples, k, side, exclude_lists=None):
        self.calls.append(("entity", np.asarray(triples).copy(), k, side, exclude_lists))
        n = len(triples)
        ids = np.tile(np.arange(k, dtype=np.int64) + 10, (n, 1))
        energies = np.tile(-np.arange(k, dtype=np.float32), (n, 1))
        return ids, energies, 1.0 / (1.0 + np.exp(-energies))


def _scorer():
    sc = evaluation.Scorer()
    sc.register_data(np.array([[0, 0, 1], [0, 2, 1], [0, 0, 1], [3, 1, 2]]))   # train (one duplicate)
    sc.register_data(np.array([[0, 2, 1], [0, 1, 1], [1, 0, 0]]))             # valid: repeats (0, 2, 1)
    sc.register_data(np.array([[0, 3, 1], [3, 1, 2]]))                        # test
    stub = StubModel()
    sc.register_model(stub)
    return sc, stub


def test_known_relation_triples_are_deduplicated_across_splits():
    sc, _ = _scorer()
    assert sc.known_relation_triples == {(0, 1): [0, 2, 1, 3], (3, 2): [1], (1, 0): [0]}
    # the entity-side lists are unchanged by the new ones
    assert sc.known_object_triples[(0, 0)] == [1] and sc.known_subject_triples[(1, 2)] == [0]


def test_scorer_hands_the_known_relations_to_the_model():
    sc, stub = _scorer()
    q = np.array([[0, 3, 1], [3, 1, 2], [2, 0, 5]])
    sc.predict_top_k_relations(q, 4)
    sc.predict_top_k_relations(q, 4, filtered=False)
    score = sc.compute_relation_mrr_scores(q)
    (t0, tri0, k0, ex0), (t1, _, _, ex1), (t2, tri2, known) = stub.calls
    assert (t0, t1, t2, k0) == ("top", "top", "rank", 4)
    assert tri0.tolist() == q.tolist() and tri2.tolist() == q.tolist()
    assert [sorted(e) for e in ex0] == [[0, 1, 2, 3], [1], []]
    assert ex1 is None
    assert [sorted(e) for e in known] == [[0, 1, 2, 3], [1], []]
    assert score.raw_ranks == [2, 3, 4] and score.filtered_ranks == [1, 1, 1]
    res = score.get_summary().results
    assert res['Filtered']['MRR'] == 1.0 and res['Raw']['H@1'] == 0.0


def test_relation_paths_refuse_a_model_off_cuda():
    from relationprediction_b200.model import Model

    class CpuModel(Model):
        def rank_relations_all(self, *a):
            raise AssertionError("not reached")

        def top_k_relations_all(self, *a):
            raise AssertionError("not reached")
    m = CpuModel(None, {'EntityCount': 5, 'RelationCount': 3, 'EdgeCount': 1})
    m.set_device("cpu")
    with pytest.raises(NotImplementedError, match="relation prediction"):
        m.rank_all_relations(np.array([[0, 1, 2]]), [[1]])
    with pytest.raises(NotImplementedError, match="relation prediction"):
        m.predict_top_k_relations(np.array([[0, 1, 2]]), 3)
    bare = Model(None, {'EntityCount': 5, 'RelationCount': 3, 'EdgeCount': 1})
    bare.set_device("cpu")
    with pytest.raises(NotImplementedError):
        bare.predict_top_k_relations(np.array([[0, 1, 2]]), 3)


def test_parse_queries_handles_relation_queries_by_name_and_id():
    ents = {"alice": 0, "bob": 1, "carol": 2}
    rels = {"knows": 0, "likes": 1}
    q = predict_cmd.parse_queries(["alice\t?\tbob\n", "alice\tknows\t?", "\n", "carol\t?\talice\r\n"], ents, rels)
    assert q == [(0, -1, 1, 2), (0, 0, -1, 1), (2, -1, 0, 2)]
    ids = {str(i): i for i in range(5)}
    assert predict_cmd.parse_queries(["3\t?\t4", "?\t0\t4"], ids, {"0": 0}) == [(3, -1, 4, 2), (-1, 0, 4, 0)]


@pytest.mark.parametrize("line,needle", [
    ("alice\t?\t?", "exactly one"), ("?\t?\tbob", "exactly one"), ("?\t?\t?", "exactly one"),
    ("alice\tknows\tbob", "exactly one"), ("alice\t?", "expected head"),
    ("alice\t?\tdave", "unknown entity 'dave'"), ("dave\t?\tbob", "unknown entity 'dave'"),
])
def test_parse_queries_rejects_malformed_relation_queries(line, needle):
    with pytest.raises(predict_cmd.QueryError, match="line 2: " + needle):
        predict_cmd.parse_queries(["alice\t?\tbob", line], {"alice": 0, "bob": 1}, {"knows": 0})


def test_answer_interleaves_entity_and_relation_queries_in_query_order():
    sc, stub = _scorer()
    queries = [(0, -1, 1, 2), (0, 0, -1, 1), (-1, 1, 2, 0), (3, -1, 2, 2)]
    rows = predict_cmd.answer(sc, queries, 2, filtered=True)
    assert [r[:3] for r in rows] == [(0, 1, 0), (0, 2, 1), (1, 1, 10), (1, 2, 11), (2, 1, 10), (2, 2, 11),
                                     (3, 1, 0), (3, 2, 1)]
    (e0, t0, _, s0, _), (e1, t1, _, s1, _), (r2, t2, k2, ex2) = stub.calls
    assert (e0, s0, e1, s1, r2, k2) == ("entity", 0, "entity", 1, "top", 2)
    assert t2.tolist() == [[0, 0, 1], [3, 0, 2]]                # the relation column holds an id in range
    assert [sorted(e) for e in ex2] == [[0, 1, 2, 3], [1]]
    predict_cmd.answer(sc, queries, 2, filtered=False)
    assert stub.calls[-1][0] == "top" and stub.calls[-1][3] is None


def test_answer_without_relation_queries_never_calls_the_relation_path():
    class EntityOnly(StubModel):
        def predict_top_k_relations(self, *a, **kw):
            raise AssertionError("relation path called without relation queries")
    sc = evaluation.Scorer()
    sc.register_data(np.array([[0, 0, 1]]))
    sc.register_model(EntityOnly())
    rows = predict_cmd.answer(sc, [(0, 0, -1, 1), (-1, 0, 1, 0)], 1, filtered=True)
    assert [r[:3] for r in rows] == [(0, 1, 10), (1, 1, 10)]


def test_predict_command_writes_relation_rows_with_the_model_stubbed(tmp_path, monkeypatch):
    from relationprediction_b200 import train as driver
    splits = {"train": np.array([[0, 0, 1], [1, 1, 2]], np.int32), "valid": np.zeros((0, 3), np.int32),
              "test": np.zeros((0, 3), np.int32)}
    ents, rels = {0: "alice", 1: "bob", 2: "carol"}, {0: "knows", 1: "likes"}
    monkeypatch.setattr(driver, "load_dataset", lambda path: (splits, ents, rels))

    class Chain(StubModel):
        def load(self, path):
            pass

        def predict_top_k(self, triples, k, side, exclude_lists=None):
            ids, energies, scores = StubModel.predict_top_k(self, triples, k, side, exclude_lists)
            return ids - 10, energies, scores
    model, sc = Chain(), evaluation.Scorer()
    for part in splits.values():
        sc.register_data(part)
    sc.register_model(model)
    monkeypatch.setattr(driver, "build_chain", lambda *a: (None, model, sc))
    monkeypatch.setattr(predict_cmd.settings_reader, "read", lambda path: {})
    (tmp_path / "q.tsv").write_text("alice\t?\tbob\nalice\tknows\t?\n")
    out = tmp_path / "out.tsv"
    predict_cmd.main(["--settings", "x.exp", "--dataset", "d", "--checkpoint", "m-3.pt", "--queries",
                      str(tmp_path / "q.tsv"), "--k", "2", "--out", str(out)])
    lines = [l.split("\t") for l in out.read_text().splitlines()]
    # relation answers by relation name, entity answers by entity name, in query order
    assert [l[:3] for l in lines] == [["0", "1", "knows"], ["0", "2", "likes"], ["1", "1", "alice"],
                                      ["1", "2", "bob"]]
    assert abs(float(lines[1][3]) - 1.0 / (1.0 + np.exp(1.0))) < 1e-7
    assert model.calls[-1][0] == "top" and [sorted(e) for e in model.calls[-1][3]] == [[0]]
