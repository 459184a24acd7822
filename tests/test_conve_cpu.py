"""CPU: the ConvE decoder -- the float64 oracle (gradcheck in every weight), the [Decoder] keys and every refusal, the
factory with both encoder families, the host plugin chain and the training driver with the library calls replaced by
the oracle (the substitution lives in this file; the product has no CPU path), a checkpoint round trip that includes
the decoder's weights, and the C-ABI argument checks, which all return before any device work."""
import ctypes

import numpy as np
import pytest
import torch

import conve_oracle as co
import one_to_n_oracle as oo
from relationprediction_b200 import _lib, ops
from relationprediction_b200 import ensemble as ens_mod
from relationprediction_b200 import train as driver
from relationprediction_b200.common import evaluation, model_builder
from relationprediction_b200.decoders.conve import ConvE, parse_conve_settings
from test_gpu_train import TOY_EXP, write_toy
from test_plugin_chain_cpu import oracle_backed_ops  # noqa: F401  (fixture)
from test_plugin_host import merged_settings
from test_train_loop_cpu import cpu_driver  # noqa: F401  (fixture)

DT = torch.float64


def tables(V, R, h, w, C, seed=0):
    d, F = h * w, C * (2 * h - 2) * (w - 2)
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(s, dtype=DT, generator=g) * sc for s, sc in
            (((V, d), 0.5), ((R, d), 0.5), ((R, d), 0.5), ((C, 3, 3), 0.5), ((C,), 0.1), ((F, d), F ** -0.5),
             ((d,), 0.1))]


# ---- the oracle ----
@pytest.mark.parametrize("masked", [False, True])
def test_oracle_gradcheck_in_every_weight(masked):
    V, R, h, w, C = 7, 3, 3, 4, 2
    ts = [t.requires_grad_(True) for t in tables(V, R, h, w, C)]
    q = np.array([[0, 1, 0], [3, 2, 0], [5, 0, 1], [6, 2, 1]], np.int32)
    y = torch.rand(4, V, generator=torch.Generator().manual_seed(2)) < 0.3
    masks, keeps = None, (1.0, 1.0, 1.0)
    if masked:
        g = torch.Generator().manual_seed(3)
        masks = tuple((torch.rand(4, n, generator=g) < 0.7).to(torch.uint8) for n in (2 * h * w, C, h * w))
        keeps = (0.7, 0.7, 0.7)
    f = lambda *a: sum(co.one_to_n_loss(*a, h, q, y, 0.1, masks, keeps))
    assert torch.autograd.gradcheck(f, tuple(ts))


def test_oracle_reciprocal_rows_and_ranks():
    V, R, h, w, C = 9, 2, 2, 4, 3
    ts = tables(V, R, h, w, C)
    a, r = torch.tensor([1, 4]), torch.tensor([0, 1])
    q1 = co.query_rows(*ts, h, a, r, [1, 1])
    ts2 = list(ts)
    ts2[2] = ts[1]   # rel_inv = rel: a subject query is then the object query
    assert torch.equal(co.query_rows(*ts2, h, a, r, [0, 0]), q1)
    scores = torch.tensor([[0.5, 0.9, 0.5, 0.1]])
    raw, filt = co.ranks(scores, torch.tensor([0]), torch.tensor([[False, True, False, False]]))
    assert raw.tolist() == [3] and filt.tolist() == [3]   # 3 - 1 known + 1


# ---- settings, factory, refusals ----
def _decoder_settings(toy, settings_file="complex.exp", d="16", **keys):
    enc, dec = merged_settings(toy, settings_file, toy["V"], toy["R"], len(toy["train"]))
    for s in (enc, dec):
        s.put("CodeDimension", d)
        s.put("InternalEncoderDimension", d)
    dec.put("Name", "conve")
    dec.put("TrainingObjective", "1-N")
    dec.put("EmbeddingHeight", "4")
    for k, v in keys.items():
        dec.put(k, v)
    return enc, dec


def test_settings_defaults_and_refusals():
    assert parse_conve_settings({}, 500) == (20, 32, (0.8, 0.8, 0.7))
    assert parse_conve_settings({'EmbeddingHeight': '10', 'ConvFilters': '8', 'InputDropoutKeepProbability': '1',
                                 'FeatureDropoutKeepProbability': '0.5', 'HiddenDropoutKeepProbability': '0.25'},
                                200) == (10, 8, (1.0, 0.5, 0.25))
    for d, h in ((16, 3), (16, 1), (12, 6), (10, 2)):   # d % h, h < 2, w < 3, d % 4
        with pytest.raises(ValueError, match="CodeDimension"):
            parse_conve_settings({'EmbeddingHeight': str(h)}, d)
    with pytest.raises(ValueError, match="ConvFilters"):
        parse_conve_settings({'EmbeddingHeight': '4', 'ConvFilters': '0'}, 16)
    for key in ('InputDropoutKeepProbability', 'FeatureDropoutKeepProbability', 'HiddenDropoutKeepProbability'):
        for bad in ('0', '1.5', 'nan', '-0.2'):
            with pytest.raises(ValueError, match=key):
                parse_conve_settings({'EmbeddingHeight': '4', key: bad}, 16)


@pytest.mark.parametrize("settings_file", ["complex.exp", "gcn_basis.exp"])
def test_factory_builds_conve(toy, settings_file):
    enc, dec = _decoder_settings(toy, settings_file, ConvFilters="3")
    encoder = model_builder.build_encoder(enc, np.array(toy["train"]))
    model = model_builder.build_decoder(encoder, dec)
    assert type(model) is ConvE and model.next_component is encoder and model.ensemble_fused is False
    assert (model.height, model.filter_count, model.keeps, model.feature_count) == (4, 3, (0.8, 0.8, 0.7), 36)
    model.set_device("cpu")
    model.initialize_train()
    shapes = [tuple(w.shape) for w in model.get_weights()[-5:]]
    assert shapes == [(toy["R"], 16), (3, 3, 3), (3,), (36, 16), (16,)]


def test_factory_refusals(toy):
    for objective in ("NegativeSampling", "SelfAdversarial"):
        _, dec = _decoder_settings(toy, TrainingObjective=objective)
        with pytest.raises(ValueError, match="conve decoder trains under TrainingObjective=1-N only"):
            model_builder.build_decoder(None, dec)
    with pytest.raises(ValueError, match="1-N only, not 'NegativeSampling'"):   # the default objective
        model_builder.build_decoder(None, {'Name': 'conve', 'CodeDimension': '16', 'EmbeddingHeight': '4'})
    _, dec = _decoder_settings(toy, EmbeddingHeight="3")
    with pytest.raises(ValueError, match="EmbeddingHeight"):
        model_builder.build_decoder(None, dec)
    # the other decoders' messages are unchanged
    assert model_builder.build_decoder(None, {'Name': 'nonlinear-transform'}) is None
    with pytest.raises(ValueError, match=r"TrainingObjective=1-N needs the bilinear-diag or complex decoder, "
                                         r"not 'rotate'"):
        model_builder.build_decoder(None, {'Name': 'rotate', 'TrainingObjective': '1-N'})
    with pytest.raises(ValueError, match="decoder"):
        ops.one_to_n_loss(None, None, np.zeros((0, 3), np.int32), None, 0.0, "transe")


# ---- the host plugin chain with the library calls replaced by the oracle ----
class DenseLabels(object):
    def __init__(self, train, V):
        self.train, self.V = train, V

    def rows(self, queries):
        return torch.as_tensor(oo.dense_labels(self.train, queries, self.V)).bool()


def oracle_loss(codes, rel, weights, queries, labels, smoothing, masks=None, keeps=(1.0, 1.0, 1.0),
                relation_count=None):
    rel, ws = rel.to(codes.dtype), [w.to(codes.dtype) for w in weights]
    return co.one_to_n_loss(codes, rel, *ws, weights.h, queries, labels, smoothing, masks, keeps)


def oracle_rows(codes, rel, weights, X, side, relation_count=None):
    X = torch.as_tensor(X).long()
    anchors = X[:, 0] if side == 1 else X[:, 2]
    rel, ws = rel.to(codes.dtype), [w.to(codes.dtype) for w in weights]
    return co.query_rows(codes, rel, *ws, weights.h, anchors, X[:, 1], [side] * len(X))


class OracleConvERanker(object):
    def __init__(self, codes, rel, weights, relation_count=None):
        self.codes, self.rel, self.weights = codes, rel, weights

    def _scores(self, X, side):
        return torch.sigmoid((oracle_rows(self.codes, self.rel, self.weights, X, side) @ self.codes.T).float())

    def rank(self, X, side, known_mask=None):
        X = torch.as_tensor(X).long()
        known = None
        if known_mask is not None:
            known = torch.as_tensor(oo.unbits(np.asarray(known_mask.cpu()).view(np.uint32), len(self.codes))).bool()
        return co.ranks(self._scores(X, side), X[:, 2] if side == 1 else X[:, 0], known)

    def top_k(self, X, side, k, exclude_mask=None):
        E = oracle_rows(self.codes, self.rel, self.weights, X, side) @ self.codes.T
        top = torch.topk(E, k, dim=1)
        return top.indices.int(), top.values.float()

    def rank_relations(self, X, known_mask=None):
        raise NotImplementedError("the ConvE decoder has no relation prediction")

    top_k_relations = rank_relations


@pytest.fixture
def oracle_conve(monkeypatch, oracle_backed_ops):  # noqa: F811
    calls = []

    def fake_loss(*a, **kw):
        calls.append((len(a[3]), a[6] if len(a) > 6 else kw.get("masks")))
        return oracle_loss(*a, **kw)
    monkeypatch.setattr(ops, "conve_one_to_n_loss", fake_loss)
    monkeypatch.setattr(ops, "conve_query_rows", oracle_rows)
    monkeypatch.setattr(ops, "ConvERanker", OracleConvERanker)
    return calls


@pytest.mark.parametrize("settings_file", ["complex.exp", "gcn_basis.exp"])
def test_host_chain(toy, oracle_conve, settings_file):
    train = np.asarray(toy["train"], np.int32)
    V, R = int(toy["V"]), int(toy["R"])
    enc, dec = _decoder_settings(toy, settings_file, ConvFilters="3", LabelSmoothing="0.1")
    model = model_builder.build_decoder(model_builder.build_encoder(enc, train), dec)
    model.set_device("cpu")
    model.initialize_train()
    model.set_one_to_n_labels(DenseLabels(train, V))
    torch.manual_seed(0)
    ws = model.get_weights()
    for w in ws:
        w.data = torch.randn(w.shape, dtype=DT) * 0.3
    X = train[:12]
    feed = (train[:20], X, np.ones(len(X), np.float32)) if model.needs_graph() else (X, np.ones(len(X), np.float32))
    total = model.train_loss(*feed)
    total.backward()
    n, masks = oracle_conve[0]
    queries = ops.one_to_n_queries(X)
    assert n == len(queries) and [tuple(m.shape) for m in masks] == [(n, 32), (n, 3), (n, 16)]
    codes, relt = [t.detach() for t in model.next_component.get_all_codes(mode='train')[:2]]
    weights = ops.ConvEWeights(*[w.detach() for w in ws[-5:]], h=4)
    L, reg = co.one_to_n_loss(codes, relt, *weights, 4, queries,
                              torch.as_tensor(oo.dense_labels(train, queries, V)).bool(), 0.1, masks, model.keeps)
    param = float(dec["RegularizationParameter"])
    assert abs(total.item() - (L.item() + param * reg.item())) <= 1e-12 * abs(total.item())
    assert all(w.grad is not None and torch.isfinite(w.grad).all() for w in ws[-5:])
    # test mode: no dropout; predict, both score matrices, fused ranks equal to matrix ranks, top-k
    model.preprocess(train)
    model.register_for_test(train)
    test = np.asarray(toy["test"], np.int32)
    p = np.asarray(model.score(test))
    with torch.no_grad():
        codes, relt = [t.detach() for t in model.next_component.get_all_codes(mode='test')[:2]]
        T = torch.as_tensor(test).long()
        q1 = co.query_rows(codes, relt, *weights, 4, T[:, 0], T[:, 1], [1] * len(T))
        q0 = co.query_rows(codes, relt, *weights, 4, T[:, 2], T[:, 1], [0] * len(T))
    np.testing.assert_allclose(p, torch.sigmoid((q1 * codes[T[:, 2]]).sum(1)).numpy(), rtol=1e-12)
    np.testing.assert_allclose(model.score_all_objects(test), torch.sigmoid(q1 @ codes.T).numpy(), rtol=1e-12)
    np.testing.assert_allclose(model.score_all_subjects(test), torch.sigmoid(q0 @ codes.T).numpy(), rtol=1e-12)
    sc = evaluation.Scorer({'Metric': 'MRR'})
    sc.register_data(train)
    sc.register_data(test)
    sc.register_model(model)
    matrices = sc.compute_scores(test)
    fused = model.rank_all(test, [sc.known_subject_triples.get((t[2], t[1]), []) for t in test.tolist()],
                           [sc.known_object_triples.get((t[0], t[1]), []) for t in test.tolist()])
    assert np.concatenate([fused[0], fused[2]]).tolist() == matrices.raw_ranks
    assert np.concatenate([fused[1], fused[3]]).tolist() == matrices.filtered_ranks
    with torch.no_grad():
        ids, energies = model.top_k_all(test, 3, 1)
    np.testing.assert_allclose(energies, torch.topk(q1 @ codes.T, 3, dim=1).values.float().numpy(), rtol=1e-6)


def test_checkpoint_round_trip_includes_the_decoder_weights(toy, tmp_path):
    enc, dec = _decoder_settings(toy)
    model = model_builder.build_decoder(model_builder.build_encoder(enc, np.array(toy["train"])), dec)
    model.set_device("cpu")
    model.initialize_train()
    assert [w is v for w, v in zip(model.get_weights()[-5:], model.local_get_weights())] == [True] * 5
    saved = [torch.randn(w.shape) for w in model.get_weights()]
    for w, v in zip(model.get_weights(), saved):
        w.data = v.clone()
    model.save(str(tmp_path / "rt"))
    for w in model.get_weights():
        w.data.zero_()
    model.load(str(tmp_path / "rt-0.pt"))
    assert all(torch.equal(a, w.detach()) for a, w in zip(saved, model.get_weights()))


def test_no_relation_prediction_or_fused_ensemble(toy, oracle_conve):
    enc, dec = _decoder_settings(toy)
    model = model_builder.build_decoder(model_builder.build_encoder(enc, np.array(toy["train"])), dec)
    model.set_device("cpu")
    model.initialize_train()
    model.register_for_test(np.array(toy["train"]))
    tri = np.array(toy["test"])[:3]
    with pytest.raises(NotImplementedError):
        model.rank_all_relations(tri, [[]] * 3)
    with pytest.raises(NotImplementedError):
        model.predict_top_k_relations(tri, 5)
    ensemble = ens_mod.Ensemble(model, model, 0.5)
    assert not ensemble.supports_fused_ranking() and ensemble.rank_all_entities(tri, [[]] * 3, [[]] * 3) is None

    with pytest.raises(NotImplementedError, match="ConvE"):
        ops.ConvERanker.rank_relations(None, None)
    with pytest.raises(NotImplementedError, match="ConvE"):
        ops.ConvERanker.top_k_relations(None, None, 5)


def test_conve_ranker_is_no_fused_ensemble_member():
    ranker = ops.ConvERanker.__new__(ops.ConvERanker)
    for call in (lambda: ranker.rank_relations(None), lambda: ranker.top_k_relations(None, 5)):
        with pytest.raises(NotImplementedError, match="ConvE"):
            call()
    with pytest.raises(TypeError, match="DistMultRanker"):
        ops.EnsembleRanker(ranker, ranker, 0.5)


def test_driver_trains_and_refuses_relation_metrics(toy, tmp_path, capsys, cpu_driver, oracle_conve,  # noqa: F811
                                                    monkeypatch):
    monkeypatch.setattr(ops, "OneToNLabels", lambda train, V, R, device: DenseLabels(np.asarray(train, np.int32), V))
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(TOY_EXP.format(layers=1, concat="No").replace(
        "Name=bilinear-diag", "Name=conve\n\tEmbeddingHeight=4\n\tConvFilters=2").replace(
        "[General]\n", "[General]\n\tTrainingObjective=1-N\n"))
    np.random.seed(0)
    torch.manual_seed(0)
    driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "40", "--device", "cpu",
                 "--no-save"])
    losses = [float(l.split(":")[-1]) for l in capsys.readouterr().out.splitlines()
              if l.startswith("Average train loss")]
    assert len(losses) == 2 and all(np.isfinite(losses))
    with pytest.raises(SystemExit, match="relation-metrics: the ConvE decoder"):
        driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "40", "--device", "cpu",
                     "--no-save", "--relation-metrics"])
    assert "Initial loss" not in capsys.readouterr().out


# ---- C-ABI: every bad argument is refused before any device work (fake device pointers are never touched) ----
P = ctypes.c_void_p(256)
Q3 = np.array([[0, 1, 0], [9, 3, 1], [2, 0, 1]], np.int32)


def _net(**kw):
    a = dict(h=2, C=3, rel_inv=256, filters=256, conv_bias=256, W_fc=256, b_fc=256, input_mask=None,
             feature_mask=None, hidden_mask=None, input_keep=0.8, feature_keep=0.8, hidden_keep=0.7)
    a.update({k: v for k, v in kw.items() if k in a})
    return _lib.ConvENet(*a.values())


GRADS = _lib.ConvEGrads(256, 256, 256, 256, 256)


def _onen(**kw):
    a = dict(codes=P, rel=P, V=10, Vrel=10, R=4, d=8, q=Q3, n=3, labels=P, eps=0.1, g=None, loss=P, dcodes=P,
             drel=P, grads=GRADS, chunk=2, ws=P, wsb=1 << 40)
    a.update({k: v for k, v in kw.items() if k in a})
    qp = None if a["q"] is None else ctypes.c_void_p(a["q"].ctypes.data)
    g = None if a["grads"] is None else ctypes.byref(a["grads"])
    return _lib.load().rgcn_conve_one_to_n(a["codes"], a["rel"], a["V"], a["Vrel"], a["R"], a["d"],
                                           ctypes.byref(_net(**kw)), qp, a["n"], a["labels"], a["eps"], a["g"],
                                           a["loss"], a["dcodes"], a["drel"], g, a["chunk"], a["ws"], a["wsb"], None)


def _finish(**kw):
    a = dict(codes=P, rel=P, V=10, Vrel=10, R=4, d=8, q=Q3, n=3, g=P, dl=P, drl=P, lg=GRADS, dcodes=P, drel=P,
             grads=GRADS, ws=P, wsb=1 << 40)
    a.update({k: v for k, v in kw.items() if k in a})
    qp = None if a["q"] is None else ctypes.c_void_p(a["q"].ctypes.data)
    lg = None if a["lg"] is None else ctypes.byref(a["lg"])
    g = None if a["grads"] is None else ctypes.byref(a["grads"])
    return _lib.load().rgcn_conve_one_to_n_finish(a["codes"], a["rel"], a["V"], a["Vrel"], a["R"], a["d"],
                                                  ctypes.byref(_net(**kw)), qp, a["n"], a["g"], a["dl"], a["drl"], lg,
                                                  a["dcodes"], a["drel"], g, a["ws"], a["wsb"], None)


def _eval(entry):
    def call(**kw):
        a = dict(codes=P, rel=P, V=10, Vrel=10, R=4, d=8, X=P, n=5, side=1, ws=P, wsb=1 << 40)
        a.update({k: v for k, v in kw.items() if k in a})
        head = (a["codes"], a["rel"], a["V"], a["Vrel"], a["R"], a["d"], ctypes.byref(_net(**kw)), a["X"], a["n"],
                a["side"])
        lib = _lib.load()
        if entry == "rows":
            return lib.rgcn_conve_query_rows(*head, P, a["ws"], a["wsb"], None)
        if entry == "rank":
            return lib.rgcn_conve_rank(*head, P, 0, P, P, a["ws"], a["wsb"], None)
        return lib.rgcn_conve_topk(*head, kw.get("k", 5), None, 0, P, P, a["ws"], a["wsb"], None)
    call.__name__ = entry
    return call


NET_BAD = [dict(h=1), dict(h=3), dict(h=4), dict(C=0), dict(d=6), dict(d=16, h=8), dict(rel_inv=None),
           dict(filters=None), dict(conv_bias=None), dict(W_fc=None), dict(b_fc=None), dict(input_keep=0.0),
           dict(feature_keep=1.5), dict(hidden_keep=float("nan"))]
SIZE_BAD = [dict(V=0), dict(Vrel=0), dict(R=0), dict(R=11), dict(n=-1)]
INVALID = ([(_onen, b) for b in NET_BAD + SIZE_BAD + [
               dict(codes=None), dict(rel=None), dict(loss=None), dict(ws=None), dict(labels=None), dict(q=None),
               dict(dcodes=None), dict(drel=None), dict(grads=None), dict(chunk=0), dict(eps=1.0),
               dict(eps=float("nan"))]] +
           [(_finish, b) for b in NET_BAD + SIZE_BAD + [
               dict(codes=None), dict(g=None), dict(dl=None), dict(lg=None), dict(grads=None), dict(ws=None),
               dict(q=None)]] +
           [(_eval(e), b) for e in ("rows", "rank", "topk") for b in NET_BAD + SIZE_BAD + [
               dict(codes=None), dict(rel=None), dict(X=None), dict(ws=None), dict(side=2), dict(side=-1)]] +
           [(_eval("topk"), dict(k=0)), (_eval("topk"), dict(k=129))])


@pytest.mark.parametrize("fn,bad", INVALID, ids=lambda x: x.__name__ if callable(x) else
                         "-".join("%s=%s" % kv for kv in x.items()))
def test_cabi_rejects_bad_arguments(fn, bad):
    assert fn(**bad) == -1, _lib.load().rgcn_last_error()


@pytest.mark.parametrize("q", [((10, 0, 0),), ((-1, 0, 1),), ((0, 4, 1),), ((0, 0, 2),)])
def test_cabi_rejects_bad_queries(q):
    qs = np.ascontiguousarray(np.array(q, np.int32))
    assert _onen(q=qs, n=1) == -1 and b"query 0" in _lib.load().rgcn_last_error()
    assert _finish(q=qs, n=1) == -1 and b"query 0" in _lib.load().rgcn_last_error()


def test_cabi_workspace_and_device():
    lib = _lib.load()
    need = lib.rgcn_conve_one_to_n_workspace_bytes(10, 4, 8, 2, 3, 3, 2)
    assert need > lib.rgcn_one_to_n_workspace_bytes(10, 8, 3, 2)
    for bad in ((10, 4, 8, 3, 3, 3, 2), (10, 0, 8, 2, 3, 3, 2), (10, 4, 8, 2, 0, 3, 2), (10, 4, 8, 2, 3, 3, 0)):
        assert lib.rgcn_conve_one_to_n_workspace_bytes(*bad) == -1
    assert _onen(wsb=need - 1) == -4
    assert _finish(wsb=lib.rgcn_conve_one_to_n_finish_workspace_bytes(3) - 1) == -4
    rows = lib.rgcn_conve_query_rows_workspace_bytes(8, 2, 3, 5)
    rank = lib.rgcn_conve_rank_workspace_bytes(10, 8, 2, 3, 5)
    topk = lib.rgcn_conve_topk_workspace_bytes(10, 8, 2, 3, 5, 5)
    assert min(rows, rank, topk) > 0 and rank > lib.distmult_rank_workspace_bytes(10, 8, 5)
    assert _eval("rows")(wsb=rows - 1) == -4 and _eval("rank")(wsb=rank - 1) == -4
    assert _eval("topk")(wsb=topk - 1) == -4
    if torch.cuda.is_available():
        pytest.skip("a device is present: valid arguments would run")
    assert _onen() == -5 and _finish() == -5 and _eval("rows")() == -5
