"""Top-k entity prediction without a GPU: argument checks of the C-ABI (they run before any device work), the ops
layer's refusal of CPU tensors, the exclusion lists Scorer.predict_top_k builds, and the predict command's query
parsing and output with the model stubbed."""
import ctypes

import numpy as np
import pytest
import torch

from relationprediction_b200 import _lib, ops
from relationprediction_b200 import predict as predict_cmd
from relationprediction_b200.common import evaluation

ENTRIES = ("distmult_topk", "rgcn_complex_topk")


def _call(lib, name, V=300, d=8, n=4, side=1, k=10, ws_bytes=None, codes=True, X=True, ids=True, energies=True,
          ws=True):
    buf = np.zeros(1 << 16, np.float32)
    p = ctypes.c_void_p(buf.ctypes.data)
    if ws_bytes is None:
        ws_bytes = max(lib.rgcn_topk_workspace_bytes(V, d if d > 0 and d % 4 == 0 else 8, n, min(max(k, 1), 128)), 0)
    return getattr(lib, name)(p if codes else None, p, V, 7, d, p if X else None, n, side, k, None, 0,
                              p if ids else None, p if energies else None, p if ws else None, ws_bytes, None)


@pytest.mark.parametrize("name", ENTRIES)
def test_entry_points_reject_bad_arguments(name):
    lib = _lib.load()
    for kw, needle in ((dict(k=0), b"k = 0"), (dict(k=129), b"k = 129"), (dict(k=-3), b"out of range"),
                       (dict(codes=False), b"bad arguments"), (dict(X=False), b"bad arguments"),
                       (dict(ids=False), b"bad arguments"), (dict(energies=False), b"bad arguments"),
                       (dict(ws=False), b"bad arguments"), (dict(d=6), b"d % 4"), (dict(side=2), b"side"),
                       (dict(side=-1), b"side"), (dict(V=0), b"bad arguments")):
        assert _call(lib, name, **kw) == -1, kw
        msg = lib.rgcn_last_error()
        assert name.encode() in msg and needle in msg, (kw, msg)
    need = lib.rgcn_topk_workspace_bytes(300, 8, 4, 10)
    assert _call(lib, name, ws_bytes=need - 1) == -4
    assert b"workspace too small" in lib.rgcn_last_error()


def test_workspace_bytes_rejects_bad_input_and_grows_with_n_and_k():
    lib = _lib.load()
    for args in ((0, 8, 4, 10), (100, 0, 4, 10), (100, 6, 4, 10), (100, 8, -1, 10), (100, 8, 4, 0),
                 (100, 8, 4, 129), (1 << 30, 512, 1 << 40, 128)):
        assert lib.rgcn_topk_workspace_bytes(*args) == -1, args
    base = lib.rgcn_topk_workspace_bytes(14541, 500, 0, 10)
    assert base >= 2 * 14541 * 500 * 4                          # the hi/lo split of the codes
    by_n = [lib.rgcn_topk_workspace_bytes(14541, 500, n, 10) for n in (1, 100, 1000, 10000)]
    assert all(a < b for a, b in zip(by_n, by_n[1:]))
    per_row = 500 * 4 + 114 * 10 * 8                            # query row + one (energy, id) pair per tile and k
    assert abs((by_n[3] - by_n[2]) - 9000 * per_row) <= 1024     # linear in n up to alignment
    by_k = [lib.rgcn_topk_workspace_bytes(14541, 500, 1000, k) for k in (1, 10, 100, 128)]
    assert all(a < b for a, b in zip(by_k, by_k[1:]))
    # the split sits where distmult_rank's workspace has it, so one workspace serves both
    assert lib.rgcn_topk_workspace_bytes(14541, 500, 0, 1) == lib.distmult_rank_workspace_bytes(14541, 500, 0)


@pytest.mark.parametrize("cls", [ops.DistMultRanker, ops.ComplexRanker])
def test_ops_refuse_cpu_tensors(cls):
    with pytest.raises(_lib.RgcnError, match="CUDA"):
        cls(torch.zeros(10, 8), torch.zeros(3, 8))


class StubModel(object):
    """Records the exclusion lists handed to predict_top_k; answers with the entity ids in order."""

    def __init__(self):
        self.calls = []

    def predict_top_k(self, triples, k, side, exclude_lists=None):
        self.calls.append((np.asarray(triples).copy(), k, side, exclude_lists))
        n = len(triples)
        ids = np.tile(np.arange(k, dtype=np.int64), (n, 1))
        energies = np.tile(-np.arange(k, dtype=np.float32), (n, 1))
        return ids, energies, 1.0 / (1.0 + np.exp(-energies))


def test_scorer_excludes_every_known_completion_of_the_registered_splits():
    sc = evaluation.Scorer()
    train = np.array([[0, 0, 1], [0, 0, 2], [3, 1, 2]])
    valid = np.array([[0, 0, 4], [5, 0, 2]])
    test = np.array([[6, 0, 2], [0, 1, 7]])
    for part in (train, valid, test):
        sc.register_data(part)
    stub = StubModel()
    sc.register_model(stub)
    q = np.array([[0, 0, 9], [9, 0, 2], [0, 1, 9]])
    sc.predict_top_k(q, 3, 1)                                   # objects of (0, 0, ?), (9, 0, ?), (0, 1, ?)
    sc.predict_top_k(q, 3, 0)                                   # subjects of (?, 0, 9), (?, 0, 2), (?, 1, 9)
    sc.predict_top_k(q, 3, 1, filtered=False)
    (_, k1, s1, ex1), (_, _, s0, ex0), (_, _, _, raw) = stub.calls
    assert (k1, s1, s0) == (3, 1, 0)
    assert [sorted(e) for e in ex1] == [[1, 2, 4], [], [7]]
    assert [sorted(e) for e in ex0] == [[], [0, 5, 6], []]
    assert raw is None


def test_predict_parses_names_and_ids():
    ents = {"alice": 0, "bob": 1, "carol": 2}
    rels = {"knows": 0, "likes": 1}
    q = predict_cmd.parse_queries(["alice\tknows\t?\n", "\n", "?\tlikes\tcarol\r\n", "bob\tlikes\t?"], ents, rels)
    assert q == [(0, 0, -1, 1), (-1, 1, 2, 0), (1, 1, -1, 1)]
    ids = {str(i): i for i in range(5)}
    assert predict_cmd.parse_queries(["3\t1\t?", "?\t0\t4"], ids, {"0": 0, "1": 1}) == [(3, 1, -1, 1), (-1, 0, 4, 0)]


@pytest.mark.parametrize("line,needle", [
    ("alice\tknows", "expected head"), ("alice\tknows\tbob", "exactly one"), ("?\tknows\t?", "exactly one"),
    ("alice\thates\t?", "unknown relation 'hates'"), ("?\tknows\tdave", "unknown entity 'dave'"),
])
def test_predict_rejects_malformed_queries(line, needle):
    with pytest.raises(predict_cmd.QueryError, match="line 2: " + needle):
        predict_cmd.parse_queries(["alice\tknows\t?", line], {"alice": 0, "bob": 1}, {"knows": 0})


def test_predict_answers_both_sides_in_query_order():
    sc = evaluation.Scorer()
    sc.register_data(np.array([[0, 0, 1]]))
    stub = StubModel()
    sc.register_model(stub)
    queries = [(0, 0, -1, 1), (-1, 1, 2, 0), (1, 1, -1, 1)]
    rows = predict_cmd.answer(sc, queries, 2, filtered=True)
    assert [r[:3] for r in rows] == [(0, 1, 0), (0, 2, 1), (1, 1, 0), (1, 2, 1), (2, 1, 0), (2, 2, 1)]
    (t0, _, s0, ex0), (t1, _, s1, ex1) = stub.calls
    assert s0 == 0 and t0.tolist() == [[2, 1, 2]]               # the unknown end holds the known entity's id
    assert s1 == 1 and t1.tolist() == [[0, 0, 0], [1, 1, 1]]
    assert [sorted(e) for e in ex1] == [[1], []] and ex0 == [[]]
    predict_cmd.answer(sc, queries, 2, filtered=False)
    assert stub.calls[-1][3] is None


def test_predict_command_writes_rows_with_the_model_stubbed(tmp_path, monkeypatch):
    """The command end to end on the host: names in, names out, the checkpoint handed to Model.load."""
    from relationprediction_b200 import train as driver
    splits = {"train": np.array([[0, 0, 1], [1, 1, 2]], np.int32), "valid": np.zeros((0, 3), np.int32),
              "test": np.zeros((0, 3), np.int32)}
    ents, rels = {0: "alice", 1: "bob", 2: "carol"}, {0: "knows", 1: "likes"}
    monkeypatch.setattr(driver, "load_dataset", lambda path: (splits, ents, rels))
    loaded = []

    class Chain(StubModel):
        def load(self, path):
            loaded.append(path)
    model, sc = Chain(), evaluation.Scorer()
    for part in splits.values():
        sc.register_data(part)
    sc.register_model(model)
    monkeypatch.setattr(driver, "build_chain", lambda *a: (None, model, sc))
    monkeypatch.setattr(predict_cmd.settings_reader, "read", lambda path: {})
    (tmp_path / "q.tsv").write_text("alice\tknows\t?\n?\tlikes\tcarol\n")
    out = tmp_path / "out.tsv"
    predict_cmd.main(["--settings", "x.exp", "--dataset", "d", "--checkpoint", "m-3.pt", "--queries",
                      str(tmp_path / "q.tsv"), "--k", "2", "--out", str(out)])
    assert loaded == ["m-3.pt"]
    lines = [l.split("\t") for l in out.read_text().splitlines()]
    assert [l[:3] for l in lines] == [["0", "1", "alice"], ["0", "2", "bob"], ["1", "1", "alice"], ["1", "2", "bob"]]
    assert abs(float(lines[1][3]) - 1.0 / (1.0 + np.exp(1.0))) < 1e-7
    with pytest.raises(SystemExit):
        predict_cmd.main(["--settings", "x.exp", "--dataset", "d", "--checkpoint", "m", "--queries",
                          str(tmp_path / "q.tsv"), "--k", "129", "--out", str(out)])
