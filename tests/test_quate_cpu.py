"""CPU: the QuatE decoder -- the float64 oracle (the three-way identity of the energy, gradcheck of all three
objectives, the normalisation below eps, ranks and top-k), the factory and its refusals, the host plugin chain and the
training driver with the library calls replaced by the oracle (the substitution lives in this file; the product has
no CPU path), a checkpoint round trip, an ensemble with a QuatE member, and the C-ABI argument checks, which all
return before any device work."""
import ctypes

import numpy as np
import pytest
import torch

import one_to_n_oracle as oo
import quate_oracle as qo
import self_adversarial_oracle as so
from relationprediction_b200 import _lib, ops
from relationprediction_b200 import ensemble as ens_mod
from relationprediction_b200 import train as driver
from relationprediction_b200.common import evaluation, model_builder
from relationprediction_b200.decoders.quate import QuatE
from test_compgcn_cpu import compgcn_settings, oracle_compgcn  # noqa: F401  (fixture)
from test_gpu_train import TOY_EXP, write_toy
from test_plugin_chain_cpu import oracle_backed_ops  # noqa: F401  (fixture)
from test_plugin_host import merged_settings
from test_train_loop_cpu import cpu_driver  # noqa: F401  (fixture)

DT = torch.float64


def tables(d, V, R, seed=0, scale=0.5):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(V, d, dtype=DT, generator=g) * scale, torch.randn(R, d, dtype=DT, generator=g) * scale


def triples(rng, V, R, N):
    return np.stack([rng.integers(0, V, N), rng.integers(0, R, N), rng.integers(0, V, N)], 1).astype(np.int32)


# ---- the oracle ----
def test_three_way_identity():
    """<h (x) rh, t> = <h, t (x) conj(rh)> = <rh, conj(h) (x) t>, quaternion by quaternion"""
    g = torch.Generator().manual_seed(0)
    h, r, t = (torch.randn(50, 4, dtype=DT, generator=g) for _ in range(3))
    rh = qo.quats(qo.normalize(r.reshape(50, 4)))
    a = (qo.qmul(h, rh) * t).sum(-1)
    b = (h * qo.qmul(t, qo.qconj(rh))).sum(-1)
    c = (rh * qo.qmul(qo.qconj(h), t)).sum(-1)
    torch.testing.assert_close(a, b, rtol=1e-13, atol=1e-13)
    torch.testing.assert_close(a, c, rtol=1e-13, atol=1e-13)
    # and the energies are the query rows against their gold
    codes, relt = tables(12, 7, 3, seed=1)
    X = triples(np.random.default_rng(1), 7, 3, 20)
    e = qo.energies(codes, relt, X)
    for side in (0, 1, "relation"):
        S, Sg, _ = qo.scores(codes, relt, X, side)
        torch.testing.assert_close(Sg, e, rtol=1e-12, atol=1e-12)


def test_hamilton_product_and_normalisation():
    i, j, k = (torch.eye(4, dtype=DT)[n] for n in (1, 2, 3))
    assert torch.equal(qo.qmul(i, j), k) and torch.equal(qo.qmul(j, i), -k) and torch.equal(qo.qmul(i, i), -torch.eye(
        4, dtype=DT)[0])
    # norms that are powers of two normalise exactly, in float32 too
    r = torch.tensor([[1.0, -1.0, 1.0, 1.0, 0.0, 0.0, -2.0, 0.0, 0.0, 0.0, 0.0, 0.0]])
    assert torch.equal(qo.normalize(r), torch.tensor([[0.5, -0.5, 0.5, 0.5, 0.0, 0.0, -1.0, 0.0, 0.0, 0.0, 0.0, 0.0]]))
    # a zero quaternion stays zero; below eps the row is divided by eps
    tiny = torch.tensor([[1e-13, 0.0, 0.0, 0.0]], dtype=DT)
    torch.testing.assert_close(qo.normalize(tiny), tiny / qo.EPS)


def test_oracle_gradcheck():
    """the oracle's gradients are the derivatives of its losses (all three objectives, L2 included)"""
    codes, relt = tables(8, 7, 3, seed=3)
    codes.requires_grad_(True)
    relt.requires_grad_(True)
    rng = np.random.default_rng(0)
    X = triples(rng, 7, 3, 12)
    Y = torch.as_tensor(rng.integers(0, 2, 12), dtype=DT)
    assert torch.autograd.gradcheck(lambda c, r: sum(qo.ns_loss(c, r, X, Y)[:2]), (codes, relt))
    p = so.weights(qo.self_adversarial_loss(codes, relt, X, 2, 1.3)[2], 2, 1.3)
    assert torch.autograd.gradcheck(lambda c, r: sum(qo.self_adversarial_loss(c, r, X, 2, 1.3, p=p)[:2]),
                                    (codes, relt))
    qs = oo.queries(X)
    y = torch.as_tensor(oo.dense_labels(X, qs, 7))
    assert torch.autograd.gradcheck(lambda c, r: sum(qo.one_to_n_loss(c, r, qs, y, 0.1)), (codes, relt))


def test_normalisation_gradient_below_eps():
    """a relation quaternion below eps: the gradient is g / eps, finite, and the gradcheck holds in that regime (steps
    of 1e-15 stay below eps); the rule (g - rh <rh, g>) / |r| holds above it"""
    g = torch.tensor([0.3, -0.7, 1.1, 0.2], dtype=DT)
    tiny = torch.tensor([2e-13, -1e-13, 0.0, 3e-13], dtype=DT, requires_grad=True)
    (qo.normalize(tiny) * g).sum().backward()
    torch.testing.assert_close(tiny.grad, g / qo.EPS, rtol=1e-14, atol=0)
    zero = torch.zeros(4, dtype=DT, requires_grad=True)
    (qo.normalize(zero) * g).sum().backward()
    assert torch.isfinite(zero.grad).all()
    assert torch.autograd.gradcheck(lambda r: (qo.normalize(r) * g).sum(), (tiny.detach().requires_grad_(True),),
                                    eps=1e-15, atol=1e-3, rtol=1e-6)
    r = torch.tensor([0.5, -1.5, 0.25, 2.0], dtype=DT, requires_grad=True)
    (qo.normalize(r) * g).sum().backward()
    rh = r.detach() / r.detach().norm()
    torch.testing.assert_close(r.grad, (g - rh * (rh @ g)) / r.detach().norm(), rtol=1e-13, atol=1e-15)


def test_oracle_self_adversarial_k1_is_negative_sampling():
    codes, relt = tables(8, 9, 3, seed=5)
    rng = np.random.default_rng(2)
    n = 6
    X1 = triples(rng, 9, 3, 2 * n)
    for alpha in (0.0, 1.0, 5.0):
        L, _, _ = qo.self_adversarial_loss(codes, relt, X1, 1, alpha)
        y = torch.cat([torch.ones(n, dtype=DT), torch.zeros(n, dtype=DT)])
        assert abs(float(L - qo.ns_loss(codes, relt, X1, y)[0])) < 1e-12


def test_oracle_ranks_and_top_k_follow_the_rules():
    codes, relt = tables(8, 12, 5, seed=6, scale=1.0)
    X = triples(np.random.default_rng(3), 12, 5, 20)
    for side in (0, 1, "relation"):
        S, Sg, gold = qo.scores(codes, relt, X, side)
        C = S.shape[1]
        known = [[int(g), (int(g) + 1) % C] for g in gold]
        raw, filt = qo.ranks(S, gold, known)
        np.testing.assert_array_equal(raw, (S >= Sg[:, None]).sum(1).numpy())
        assert (raw >= 1).all() and (filt >= 1).all() and (filt <= raw).all()
        ids, en = qo.top_k(S, 4, known)
        for t in range(len(X)):
            assert not set(ids[t].tolist()) & set(known[t])
            assert (np.diff(en[t]) <= 0).all()
    ids, en = qo.top_k(np.array([[1.0, 0.5, 1.0, 0.5]]), 4, [[0]])
    assert ids.tolist() == [[2, 1, 3, -1]] and en.tolist() == [[1.0, 0.5, 0.5, -np.inf]]


# ---- settings, factory, refusals ----
def _decoder_settings(toy, **keys):
    enc, dec = merged_settings(toy, "complex.exp", toy["V"], toy["R"], len(toy["train"]))
    d = keys.pop("d", "16")
    for s in (enc, dec):
        s.put("CodeDimension", d)
    dec.put("Name", keys.pop("Name", "quate"))
    for k, v in keys.items():
        dec.put(k, v)
    return enc, dec


@pytest.mark.parametrize("objective", ["NegativeSampling", "SelfAdversarial", "1-N"])
def test_factory_builds_quate(toy, objective):
    enc, dec = _decoder_settings(toy, TrainingObjective=objective)
    encoder = model_builder.build_encoder(enc, np.array(toy["train"]))
    model = model_builder.build_decoder(encoder, dec)
    assert type(model) is QuatE and model.dimension == 16 and model.next_component is encoder
    assert model.training_objective == objective and model.ensemble_fused is False and model.ONE_TO_N == "quate"
    model.set_device("cpu")
    model.initialize_train()
    assert [tuple(w.shape) for w in model.get_weights()] == [(toy["V"], 16), (16,), (toy["V"], 16)]


def test_factory_refusals(toy):
    for d in ("6", "10", "18"):
        _, dec = _decoder_settings(toy, d=d)
        with pytest.raises(ValueError, match=r"the QuatE decoder needs CodeDimension %% 4 == 0, got %s$" % d):
            model_builder.build_decoder(None, dec)
    _, dec = _decoder_settings(toy, TrainingObjective="1-N", LabelSmoothing="1.5")
    with pytest.raises(ValueError, match="LabelSmoothing"):
        model_builder.build_decoder(None, dec)
    # the other decoders keep their messages
    for name in ("rotate", "transe"):
        _, dec = _decoder_settings(toy, Name=name, TrainingObjective="1-N")
        with pytest.raises(ValueError, match=r"TrainingObjective=1-N needs the bilinear-diag or complex decoder, "
                                             r"not '%s'" % name):
            model_builder.build_decoder(None, dec)
    _, dec = _decoder_settings(toy, Name="conve", TrainingObjective="NegativeSampling")
    with pytest.raises(ValueError, match="the conve decoder trains under TrainingObjective=1-N only"):
        model_builder.build_decoder(None, dec)


def test_ops_kinds():
    assert "quate" in ops.ONE_TO_N_DECODERS and "quate" in ops.SELF_ADVERSARIAL_DECODERS
    assert ops.MARGIN_DECODERS == ("rotate", "transe")
    with pytest.raises(ValueError, match="gamma"):   # QuatE has no margin
        ops.self_adversarial_loss(None, None, None, 10, 1.0, "quate", gamma=1.0)
    assert not issubclass(ops.QuatERanker, ops.DistMultRanker)


# ---- the host plugin chain with the library calls replaced by the oracle ----
def oracle_quate_score(codes, rel_table, X, Y=None):
    X = np.asarray(X.cpu() if torch.is_tensor(X) else X)
    if Y is None:
        return qo.energies(codes, rel_table, X), torch.zeros((), dtype=codes.dtype), qo.l2(codes, rel_table, X)
    L, reg, e = qo.ns_loss(codes, rel_table, X, Y)
    return e, L, reg


def oracle_query_rows(codes, rel_table, X, side):
    return qo.queries(codes, rel_table.to(codes.dtype), np.asarray(X.cpu()), side)[0]


def _lists(mask, count):
    if mask is None:
        return None
    bits = np.asarray(mask.cpu()).view(np.uint32)
    return [[v for v in range(count) if (bits[t, v >> 5] >> (v & 31)) & 1] for t in range(len(bits))]


class OracleQuatERanker(object):
    def __init__(self, codes, rel_table, relation_count=None):
        self.codes, self.rel = codes.detach(), rel_table.detach()
        self.relation_count = rel_table.shape[0] if relation_count is None else relation_count

    def _scores(self, X, side, count=None):
        return qo.scores(self.codes, self.rel, np.asarray(X.cpu()), side, count)

    def rank(self, X, side, known_mask=None):
        S, _, gold = self._scores(X, side)
        raw, filt = qo.ranks(S, gold, _lists(known_mask, len(self.codes)))
        return torch.as_tensor(raw), None if filt is None else torch.as_tensor(filt)

    def top_k(self, X, side, k, exclude_mask=None):
        ids, en = qo.top_k(self._scores(X, side)[0], k, _lists(exclude_mask, len(self.codes)))
        return torch.as_tensor(ids), torch.as_tensor(en, dtype=torch.float32)

    def rank_relations(self, X, known_mask=None):
        S, _, gold = self._scores(X, "relation", self.relation_count)
        raw, filt = qo.ranks(S, gold, _lists(known_mask, self.relation_count))
        return torch.as_tensor(raw), None if filt is None else torch.as_tensor(filt)

    def top_k_relations(self, X, k, exclude_mask=None):
        S = self._scores(X, "relation", self.relation_count)[0]
        ids, en = qo.top_k(S, k, _lists(exclude_mask, self.relation_count))
        return torch.as_tensor(ids), torch.as_tensor(en, dtype=torch.float32)


class DenseLabels(object):
    def __init__(self, train, V):
        self.train, self.V = train, V

    def rows(self, queries):
        return torch.as_tensor(oo.dense_labels(self.train, queries, self.V))


@pytest.fixture
def oracle_quate(monkeypatch, oracle_backed_ops):  # noqa: F811
    calls = []

    def fake_sa(codes, rel_table, X, K, alpha, decoder, *, gamma=None):
        calls.append(("SelfAdversarial", K, alpha, decoder, gamma))
        return qo.self_adversarial_loss(codes, rel_table, np.asarray(X.cpu()), K, alpha)

    def fake_one_to_n(codes, rel_table, queries, labels, smoothing, decoder, relation_count=None):
        calls.append(("1-N", len(queries), smoothing, decoder, relation_count))
        return qo.one_to_n_loss(codes, rel_table, queries, labels.to(codes.dtype), smoothing)
    monkeypatch.setattr(ops, "quate_score", oracle_quate_score)
    monkeypatch.setattr(ops, "self_adversarial_loss", fake_sa)
    monkeypatch.setattr(ops, "one_to_n_loss", fake_one_to_n)
    monkeypatch.setattr(ops, "quate_query_rows", oracle_query_rows)
    monkeypatch.setattr(ops, "QuatERanker", OracleQuatERanker)
    monkeypatch.setattr(ops, "OneToNLabels", lambda train, V, R, device: DenseLabels(np.asarray(train, np.int32), V))
    return calls


def _chain_settings(toy, settings_file):
    if settings_file == "compgcn":
        enc, dec = compgcn_settings(toy, decoder="quate")
    else:
        enc, dec = merged_settings(toy, settings_file, toy["V"], toy["R"], len(toy["train"]))
        dec.put("Name", "quate")
    for s in (enc, dec):
        s.put("CodeDimension", "16")
        s.put("InternalEncoderDimension", "16")
    return enc, dec


@pytest.mark.parametrize("settings_file", ["complex.exp", "gcn_basis.exp", "compgcn"])
@pytest.mark.parametrize("objective", ["NegativeSampling", "SelfAdversarial", "1-N"])
def test_host_chain(toy, oracle_quate, oracle_compgcn, settings_file, objective):  # noqa: F811
    train = np.asarray(toy["train"], np.int32)
    V, R = int(toy["V"]), int(toy["R"])
    enc, dec = _chain_settings(toy, settings_file)
    dec.put("TrainingObjective", objective)
    if objective == "1-N":
        dec.put("LabelSmoothing", "0.1")
    model = model_builder.build_decoder(model_builder.build_encoder(enc, train), dec)
    model.set_device("cpu")
    model.initialize_train()
    if objective == "1-N":
        model.set_one_to_n_labels(DenseLabels(train, V))
    torch.manual_seed(0)
    ws = model.get_weights()
    for w in ws:
        w.data = torch.randn(w.shape, dtype=DT) * 0.3
    K = int(dec["NegativeSampleRate"])
    rng = np.random.default_rng(7)
    X = np.concatenate([triples(rng, V, R, 9)] * (K + 1))
    X[9:, 2] = rng.integers(0, V, 9 * K)
    Y = np.concatenate([np.ones(9), np.zeros(9 * K)]).astype(np.float32)
    feed = (train[:20], X, Y) if model.needs_graph() else (X, Y)
    torch.manual_seed(1)
    total = model.train_loss(*feed)
    total.backward()
    codes, relt = [t.detach() for t in model.next_component.get_all_codes(mode='train')[:2]]
    if objective == "SelfAdversarial":
        assert oracle_quate == [("SelfAdversarial", K, 1.0, "quate", None)]
        L, reg, _ = qo.self_adversarial_loss(codes, relt, X, K, 1.0)
    elif objective == "1-N":
        qs = oo.queries(X)
        assert oracle_quate == [("1-N", len(qs), 0.1, "quate", R)]
        L, reg = qo.one_to_n_loss(codes, relt, qs, torch.as_tensor(oo.dense_labels(train, qs, V)), 0.1)
    else:
        L, reg, _ = qo.ns_loss(codes, relt, X, torch.as_tensor(Y))
    param = float(dec["RegularizationParameter"])
    assert abs(total.item() - (L.item() + param * reg.item())) <= 1e-12 * abs(total.item())
    assert all(w.grad is None or torch.isfinite(w.grad).all() for w in ws)
    assert any(w.grad is not None and float(w.grad.abs().max()) > 0 for w in ws)
    # test mode: predict, the score matrices, the ranks, the top-k and the relation queries
    model.preprocess(train)
    model.register_for_test(train)
    test = np.asarray(toy["test"], np.int32)
    p = np.asarray(model.score(test))
    with torch.no_grad():
        codes, relt = [t.detach() for t in model.next_component.get_all_codes(mode='test')[:2]]
        e = qo.energies(codes, relt, test)
    np.testing.assert_allclose(p, torch.sigmoid(e).numpy(), rtol=1e-12)
    S1 = qo.scores(codes, relt, test, 1)[0]
    S0 = qo.scores(codes, relt, test, 0)[0]
    np.testing.assert_allclose(model.score_all_objects(test), torch.sigmoid(S1).numpy(), rtol=1e-12)
    np.testing.assert_allclose(model.score_all_subjects(test), torch.sigmoid(S0).numpy(), rtol=1e-12)
    sc = evaluation.Scorer({'Metric': 'MRR'})
    sc.register_data(train)
    sc.register_data(test)
    sc.register_model(model)
    matrices = sc.compute_scores(test)
    fused = model.rank_all(test, [sc.known_subject_triples.get((t[2], t[1]), []) for t in test.tolist()],
                           [sc.known_object_triples.get((t[0], t[1]), []) for t in test.tolist()])
    assert np.concatenate([fused[0], fused[2]]).tolist() == matrices.raw_ranks
    assert np.concatenate([fused[1], fused[3]]).tolist() == matrices.filtered_ranks
    ids, en = model.top_k_all(test, 3, 1)
    want_ids, want_en = qo.top_k(S1, 3)
    np.testing.assert_array_equal(ids, want_ids)
    np.testing.assert_allclose(en, want_en, rtol=1e-6)
    known_rel = [[int(t[1])] for t in test]
    raw, filt = model.rank_relations_all(test, known_rel)
    Sr, Srg, gold = qo.scores(codes, relt, test, "relation", R)
    np.testing.assert_array_equal(raw, (Sr >= Srg[:, None]).sum(1).numpy())
    np.testing.assert_array_equal(filt, raw)   # only the gold is known: it counts once either way
    ids, _ = model.top_k_relations_all(test, 2, known_rel)
    np.testing.assert_array_equal(ids, qo.top_k(Sr, 2, known_rel)[0])


def test_checkpoint_round_trip(toy, tmp_path):
    enc, dec = _decoder_settings(toy)
    model = model_builder.build_decoder(model_builder.build_encoder(enc, np.array(toy["train"])), dec)
    model.set_device("cpu")
    model.initialize_train()
    saved = [torch.randn(w.shape) for w in model.get_weights()]
    for w, v in zip(model.get_weights(), saved):
        w.data = v.clone()
    model.save(str(tmp_path / "rt"))
    for w in model.get_weights():
        w.data.zero_()
    model.load(str(tmp_path / "rt-0.pt"))
    assert all(torch.equal(a, w.detach()) for a, w in zip(saved, model.get_weights()))


def test_ensemble_member_is_not_fused(toy, oracle_quate):
    enc, dec = _decoder_settings(toy)
    model = model_builder.build_decoder(model_builder.build_encoder(enc, np.array(toy["train"])), dec)
    model.set_device("cpu")
    model.initialize_train()
    model.register_for_test(np.array(toy["train"]))
    tri = np.array(toy["test"])[:3]
    ensemble = ens_mod.Ensemble(model, model, 0.5)
    assert not ensemble.supports_fused_ranking() and ensemble.rank_all_entities(tri, [[]] * 3, [[]] * 3) is None
    with pytest.raises(NotImplementedError, match="fused path"):
        ensemble.predict_top_k(tri, 5, 1)
    # the score matrices still rank it: the weighted sum of the members' float32 sigmoid scores
    s = np.asarray(ensemble.score_all_objects(tri))
    np.testing.assert_allclose(s, np.asarray(model.score_all_objects(tri)), rtol=1e-6)


@pytest.mark.parametrize("objective", ["NegativeSampling", "SelfAdversarial", "1-N"])
def test_driver_trains(toy, tmp_path, capsys, cpu_driver, oracle_quate, objective):  # noqa: F811
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(TOY_EXP.format(layers=1, concat="No").replace(
        "Name=bilinear-diag", "Name=quate\n\tTrainingObjective=%s" % objective))
    np.random.seed(0)
    torch.manual_seed(0)
    driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "40", "--device", "cpu",
                 "--no-save"])
    text = capsys.readouterr().out
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 2 and all(np.isfinite(losses)) and "Validation filtered MRR" in text
    assert all(c[0] == objective and c[3] == "quate" for c in oracle_quate)
    assert bool(oracle_quate) == (objective != "NegativeSampling")


# ---- C-ABI: every bad argument is refused before any device work (fake device pointers are never touched) ----
P = ctypes.c_void_p(256)


def _call(entry, a, kw):
    a.update(kw)
    return getattr(_lib.load(), entry)(*a.values(), None)


def _fwd(**kw):
    return _call("rgcn_quate_forward", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, N=33, Y=P, energies=P, loss=P), kw)


def _bwd(**kw):
    return _call("rgcn_quate_backward", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, N=33, Y=P, energies=P,
                                             g_loss=1.0, g_reg=1.0, g_scale=None, g_energy=None, dcodes=P, drel=P,
                                             ss=None), kw)


def _sa(**kw):
    return _call("rgcn_quate_self_adversarial_forward", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, N=33, K=10,
                                                             alpha=1.0, energies=P, coef=P, loss=P, ws=P,
                                                             wsb=1 << 40), kw)


def _rank(**kw):
    return _call("rgcn_quate_rank", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, n=5, side=1, known=P, reuse=0,
                                         raw=P, filt=P, ws=P, wsb=1 << 40), kw)


def _topk(**kw):
    return _call("rgcn_quate_topk", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, n=5, side=1, k=4, excl=None,
                                         reuse=0, ids=P, energies=P, ws=P, wsb=1 << 40), kw)


def _rrank(**kw):
    return _call("rgcn_quate_relation_rank", dict(codes=P, rel=P, V=10, Vrel=10, R=4, d=8, X=P, n=5, known=P,
                                                  reuse=0, raw=P, filt=P, ws=P, wsb=1 << 40), kw)


def _rtopk(**kw):
    return _call("rgcn_quate_relation_topk", dict(codes=P, rel=P, V=10, Vrel=10, R=4, d=8, X=P, n=5, k=4, excl=None,
                                                  reuse=0, ids=P, energies=P, ws=P, wsb=1 << 40), kw)


QUERIES = np.array([[1, 2, 1], [3, 0, 0]], np.int32)


def _onen(**kw):
    q = kw.pop("queries", QUERIES)
    return _call("rgcn_quate_one_to_n", dict(codes=P, rel=P, V=10, Vrel=10, R=4, d=8, queries=q.ctypes.data,
                                             n=len(q), labels=P, eps=0.0, g_scale=None, loss=P, dcodes=P, drel=P,
                                             chunk=64, ws=P, wsb=1 << 40), kw)


def _rows(**kw):
    return _call("rgcn_quate_query_rows", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, n=5, side=1, Q=P), kw)


SIZES = [dict(V=0), dict(Vrel=0), dict(d=0), dict(d=6), dict(d=-4), dict(d=10)]
QUERY = SIZES + [dict(codes=None), dict(rel=None), dict(X=None), dict(ws=None), dict(n=-1)]
INVALID = ([(_fwd, b) for b in SIZES + [dict(codes=None), dict(rel=None), dict(X=None), dict(energies=None),
                                        dict(loss=None), dict(N=-1)]] +
           [(_bwd, b) for b in SIZES + [dict(codes=None), dict(rel=None), dict(X=None), dict(dcodes=None),
                                        dict(drel=None), dict(energies=None), dict(N=-1)]] +
           [(_sa, b) for b in SIZES + [dict(codes=None), dict(X=None), dict(coef=None), dict(ws=None), dict(N=34),
                                       dict(K=0), dict(alpha=-1.0), dict(alpha=float("nan"))]] +
           [(_rank, b) for b in QUERY + [dict(raw=None), dict(side=2), dict(side=-1), dict(known=None)]] +
           [(_topk, b) for b in QUERY + [dict(ids=None), dict(energies=None), dict(side=2), dict(side=-1), dict(k=0),
                                         dict(k=129)]] +
           [(_rrank, b) for b in QUERY + [dict(raw=None), dict(known=None), dict(R=0), dict(R=11)]] +
           [(_rtopk, b) for b in QUERY + [dict(ids=None), dict(energies=None), dict(k=0), dict(k=129), dict(R=0),
                                          dict(R=11)]] +
           [(_onen, b) for b in SIZES + [dict(codes=None), dict(labels=None), dict(loss=None), dict(dcodes=None),
                                         dict(ws=None), dict(R=0), dict(R=11), dict(chunk=0), dict(eps=1.0),
                                         dict(eps=float("nan")), dict(queries=np.array([[10, 0, 1]], np.int32)),
                                         dict(queries=np.array([[1, 4, 1]], np.int32)),
                                         dict(queries=np.array([[1, 0, 2]], np.int32))]] +
           [(_rows, b) for b in SIZES + [dict(codes=None), dict(rel=None), dict(X=None), dict(Q=None), dict(side=2),
                                         dict(side=-1)]])


@pytest.mark.parametrize("fn,bad", INVALID, ids=lambda x: x.__name__ if callable(x) else
                         "-".join("%s=%s" % (k, "array" if isinstance(v, np.ndarray) else v) for k, v in x.items()))
def test_cabi_rejects_bad_arguments(fn, bad):
    assert fn(**bad) == -1, _lib.load().rgcn_last_error()


def test_cabi_workspace_and_device():
    lib = _lib.load()
    rank_need = lib.distmult_rank_workspace_bytes(10, 8, 5)
    topk_need = lib.rgcn_topk_workspace_bytes(10, 8, 5, 4)
    rrank_need = lib.rgcn_quate_relation_rank_workspace_bytes(4, 8, 5)
    rtopk_need = lib.rgcn_quate_relation_topk_workspace_bytes(4, 8, 5, 4)
    # the relation workspaces carry the normalised table ahead of the DistMult ones
    assert rrank_need >= lib.rgcn_relation_rank_workspace_bytes(4, 8, 5) + 4 * 8 * 4
    assert rtopk_need >= lib.rgcn_relation_topk_workspace_bytes(4, 8, 5, 4) + 4 * 8 * 4
    for bad in ((0, 8, 5), (4, 6, 5), (4, 8, -1)):
        assert lib.rgcn_quate_relation_rank_workspace_bytes(*bad) == -1
    for bad in ((0, 8, 5, 4), (4, 6, 5, 4), (4, 8, -1, 4), (4, 8, 5, 0), (4, 8, 5, 129)):
        assert lib.rgcn_quate_relation_topk_workspace_bytes(*bad) == -1
    assert _rank(wsb=rank_need - 1) == -4 and _topk(wsb=topk_need - 1) == -4
    assert _rrank(wsb=rrank_need - 1) == -4 and _rtopk(wsb=rtopk_need - 1) == -4
    assert _sa(wsb=lib.rgcn_self_adversarial_workspace_bytes(33, 10) - 1) == -4
    assert _onen(wsb=lib.rgcn_one_to_n_workspace_bytes(10, 8, 2, 64) - 1) == -4
    if torch.cuda.is_available():
        pytest.skip("a device is present: valid arguments would run")
    assert _fwd() == -5 and _bwd() == -5 and _sa() == -5 and _rows() == -5
    assert _onen(wsb=lib.rgcn_one_to_n_workspace_bytes(10, 8, 2, 64)) == -5


def test_ranker_workspace_entries():
    """QuatERanker runs DistMultRanker's bodies over the QuatE entry points and the QuatE relation workspaces"""
    assert ops.QuatERanker._RANK == "rgcn_quate_rank" and ops.QuatERanker._TOPK == "rgcn_quate_topk"
    assert ops.QuatERanker._REL_RANK_WORKSPACE == "rgcn_quate_relation_rank_workspace_bytes"
    assert ops.DistMultRanker._REL_RANK_WORKSPACE == "rgcn_relation_rank_workspace_bytes"
    assert ops.QuatERanker.rank is ops.DistMultRanker.rank
    assert ops.QuatERanker.rank_relations is ops.DistMultRanker.rank_relations
