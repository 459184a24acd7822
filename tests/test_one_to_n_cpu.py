"""CPU: 1-N training -- the float64 oracle, the label CSR and query de-duplication, the settings keys, and the C-ABI
argument checks, which all return before any device work."""
import ctypes

import numpy as np
import pytest
import torch

import one_to_n_oracle as oo
from relationprediction_b200 import _lib, ops
from relationprediction_b200.common import model_builder
from relationprediction_b200.decoders.bilinear_diag import parse_training_objective


def skewed_graph(seed=0, V=300, R=7, m=4000):
    """a few hub entities and one dominant relation: long and empty label rows side by side"""
    rng = np.random.default_rng(seed)
    s = np.minimum(rng.zipf(1.5, m) - 1, V - 1)
    o = rng.integers(0, V, m)
    r = np.where(rng.random(m) < 0.7, 0, rng.integers(0, R, m))
    return np.stack([s, r, o], 1).astype(np.int32)


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
def test_oracle_gradcheck(decoder):
    g = torch.Generator().manual_seed(1)
    V, R, d = 9, 3, 8
    codes = torch.randn(V, d, dtype=torch.float64, generator=g, requires_grad=True)
    rel = torch.randn(R, d, dtype=torch.float64, generator=g, requires_grad=True)
    qs = np.array([[0, 1, 0], [3, 2, 0], [4, 0, 1], [8, 1, 1]], np.int32)
    y = (torch.rand(4, V, generator=g) < 0.3).double().numpy()
    f = lambda c, r: sum(oo.loss(c, r, qs, torch.as_tensor(y), 0.1, decoder))
    assert torch.autograd.gradcheck(f, (codes, rel))


def _csr_entities(labels, a, r, side):
    key = (2 * r + side) * labels.V + a
    keys = labels.keys.numpy()
    i = np.searchsorted(keys, key)
    if i == len(keys) or keys[i] != key:
        return set()
    off = labels.offsets.numpy()
    return set(labels.entities.numpy()[off[i]:off[i + 1]].tolist())


@pytest.mark.parametrize("graph", ["toy", "skewed"])
def test_label_csr_matches_numpy(toy, graph):
    train = np.asarray(toy["train"], np.int32) if graph == "toy" else skewed_graph()
    V = int(train[:, [0, 2]].max()) + 1
    R = int(train[:, 1].max()) + 1
    labels = ops.OneToNLabels(train, V, R, "cpu")
    keys = labels.keys.numpy()
    assert np.all(np.diff(keys) > 0) and labels.offsets.numpy()[-1] == len(labels.entities)
    qs = oo.queries(train)
    y = oo.dense_labels(train, qs, V)
    for t, (a, r, side) in enumerate(qs.tolist()):
        assert _csr_entities(labels, a, r, side) == set(np.flatnonzero(y[t]).tolist())
    assert len(keys) == len(qs)   # one key per distinct training query
    assert oo.unbits(oo.bits(y), V).tolist() == y.tolist()


def test_query_deduplication():
    tri = np.array([[0, 1, 2], [0, 1, 3], [0, 1, 2], [2, 1, 0], [5, 0, 2]], np.int32)
    q = ops.one_to_n_queries(tri)
    assert q.dtype == np.int32 and q.flags.c_contiguous
    assert q.tolist() == oo.queries(tri).tolist()
    assert q.tolist() == [[2, 0, 0], [0, 1, 0], [2, 1, 0], [3, 1, 0], [5, 0, 1], [0, 1, 1], [2, 1, 1]]
    assert len(q) == len({tuple(x) for x in q.tolist()})
    assert (np.diff(q[:, 2]) >= 0).all()   # subject queries first
    skew = skewed_graph()
    assert ops.one_to_n_queries(skew).tolist() == oo.queries(skew).tolist()


def test_settings_parsing_and_rejections():
    assert parse_training_objective({}) == ('NegativeSampling', 0.0)
    assert parse_training_objective({'TrainingObjective': 'NegativeSampling'}) == ('NegativeSampling', 0.0)
    assert parse_training_objective({'TrainingObjective': '1-N', 'LabelSmoothing': '0.1'}) == ('1-N', 0.1)
    with pytest.raises(ValueError, match="TrainingObjective"):
        parse_training_objective({'TrainingObjective': 'KvsAll'})
    for eps in ('1', '1.5', '-0.1', 'nan'):
        with pytest.raises(ValueError, match="LabelSmoothing"):
            parse_training_objective({'TrainingObjective': '1-N', 'LabelSmoothing': eps})
    with pytest.raises(ValueError, match="TrainingObjective=1-N"):
        model_builder.build_decoder(None, {'Name': 'nonlinear-transform', 'TrainingObjective': '1-N'})
    assert model_builder.build_decoder(None, {'Name': 'nonlinear-transform'}) is None   # unchanged without the key


def test_ops_rejects_unknown_decoder():
    with pytest.raises(ValueError, match="decoder"):
        ops.one_to_n_loss(None, None, np.zeros((0, 3), np.int32), None, 0.0, "transe")


# ---- C-ABI: every bad argument is refused before any device work (fake device pointers are never touched) ----
P = ctypes.c_void_p(256)


def _args(**kw):
    a = dict(codes=P, rel=P, V=10, Vrel=10, R=4, d=8, queries=None, n=3, labels=P, eps=0.1, g=None, loss=P,
             dcodes=P, drel=P, chunk=2, ws=P, wsb=1 << 40)
    a.update(kw)
    return a


def _call(entry, a, q=((0, 1, 0), (9, 3, 1), (2, 0, 1))):
    qs = np.ascontiguousarray(np.array(q, np.int32).reshape(-1, 3)) if a["queries"] is None else a["queries"]
    qp = ctypes.c_void_p(qs.ctypes.data) if qs is not False else None
    return getattr(_lib.load(), entry)(a["codes"], a["rel"], a["V"], a["Vrel"], a["R"], a["d"], qp, a["n"],
                                       a["labels"], a["eps"], a["g"], a["loss"], a["dcodes"], a["drel"], a["chunk"],
                                       a["ws"], a["wsb"], None)


INVALID = [
    dict(codes=None), dict(rel=None), dict(loss=None), dict(ws=None), dict(labels=None), dict(queries=False),
    dict(dcodes=None), dict(drel=None), dict(V=0), dict(Vrel=0), dict(R=0), dict(R=11), dict(d=0), dict(d=6),
    dict(n=-1), dict(chunk=0), dict(eps=1.0), dict(eps=-0.01), dict(eps=float("nan")),
]


@pytest.mark.parametrize("entry", ["distmult_one_to_n", "rgcn_complex_one_to_n"])
@pytest.mark.parametrize("bad", INVALID, ids=lambda b: "-".join("%s=%s" % kv for kv in b.items()))
def test_cabi_rejects_bad_arguments(entry, bad):
    assert _call(entry, _args(**bad)) == -1, _lib.load().rgcn_last_error()


@pytest.mark.parametrize("entry", ["distmult_one_to_n", "rgcn_complex_one_to_n"])
@pytest.mark.parametrize("q", [((10, 0, 0),), ((-1, 0, 1),), ((0, 4, 1),), ((0, -1, 0),), ((0, 0, 2),), ((0, 0, -1),)])
def test_cabi_rejects_bad_queries(entry, q):
    assert _call(entry, _args(n=1), q) == -1
    assert b"query 0" in _lib.load().rgcn_last_error()


def test_cabi_workspace_and_device():
    lib = _lib.load()
    need = lib.rgcn_one_to_n_workspace_bytes(10, 8, 3, 2)
    assert need > 0 and lib.rgcn_one_to_n_workspace_bytes(10, 8, 3, 0) == -1
    assert lib.rgcn_one_to_n_workspace_bytes(10, 6, 3, 1) == -1 and lib.rgcn_one_to_n_workspace_bytes(0, 8, 3, 1) == -1
    # the per-pass buffers grow with the chunk, not with n
    assert lib.rgcn_one_to_n_workspace_bytes(14541, 500, 60000, 4096) < 2 * lib.rgcn_one_to_n_workspace_bytes(
        14541, 500, 4096, 4096)
    assert _call("distmult_one_to_n", _args(wsb=need - 1)) == -4
    if torch.cuda.is_available():
        pytest.skip("a device is present: valid arguments would run")
    assert _call("distmult_one_to_n", _args(wsb=need)) == -5


def test_cabi_label_entry_checks():
    lib = _lib.load()
    q = np.array([[0, 1, 0], [3, 2, 1]], np.int32)
    qp = ctypes.c_void_p(q.ctypes.data)
    nb = lib.rgcn_one_to_n_labels_workspace_bytes(2)
    assert nb > 0 and lib.rgcn_one_to_n_labels_workspace_bytes(-1) == -1
    call = lambda **k: lib.rgcn_one_to_n_labels(k.get("keys", P), P, P, 5, 10, k.get("R", 3), k.get("q", qp), 2,
                                                k.get("bits", P), P, k.get("wsb", nb), None)
    assert call(keys=None) == -1 and call(bits=None) == -1 and call(q=None) == -1 and call(R=0) == -1
    assert call(R=2) == -1   # relation 2 out of range
    assert call(wsb=nb - 1) == -4
    if not torch.cuda.is_available():
        assert call() == -5


def test_label_csr_rejects_out_of_range_triples():
    tri = np.array([[0, 1, 2], [3, 0, 4]], np.int32)
    ops.OneToNLabels(tri, 5, 2, "cpu")
    for bad, V, R in ((tri, 4, 2), (tri, 5, 1), (np.array([[-1, 0, 1]], np.int32), 5, 2)):
        with pytest.raises(ValueError, match="OneToNLabels"):
            ops.OneToNLabels(bad, V, R, "cpu")


def test_cabi_finish_checks():
    lib = _lib.load()
    q = np.array([[0, 1, 0], [3, 2, 1]], np.int32)
    qp = ctypes.c_void_p(q.ctypes.data)
    nb = lib.rgcn_one_to_n_finish_workspace_bytes(2)
    assert nb > 0 and lib.rgcn_one_to_n_finish_workspace_bytes(-1) == -1
    call = lambda **k: lib.rgcn_one_to_n_finish(P, P, 10, 10, k.get("R", 3), k.get("d", 8), k.get("q", qp), 2,
                                                k.get("g", P), P, P, k.get("out", P), P, P, k.get("wsb", nb), None)
    assert call(g=None) == -1 and call(out=None) == -1 and call(q=None) == -1 and call(d=6) == -1
    assert call(R=2) == -1   # relation 2 out of range
    assert call(wsb=nb - 1) == -4
    if not torch.cuda.is_available():
        assert call() == -5
