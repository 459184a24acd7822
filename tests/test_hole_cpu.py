"""CPU: the HolE decoder -- the float64 oracle (the direct correlation against numpy's FFT, the Fourier-basis energy and
the three query-row identities, U^T U = I, gradcheck of all three objectives), the factory and its refusals, the host
plugin chain and the training driver with the library calls replaced by the oracle (the substitution lives in this
file; the product has no CPU path), a checkpoint round trip, an ensemble with a HolE member, and the C-ABI argument
checks, which all return before any device work."""
import ctypes

import numpy as np
import pytest
import torch

import hole_oracle as ho
import one_to_n_oracle as oo
import self_adversarial_oracle as so
from relationprediction_b200 import _lib, ops
from relationprediction_b200 import ensemble as ens_mod
from relationprediction_b200 import train as driver
from relationprediction_b200.common import evaluation, model_builder
from relationprediction_b200.decoders.hole import HolE
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
@pytest.mark.parametrize("d", [4, 8, 200, 500, 516])
def test_basis_is_orthogonal(d):
    U = ho.basis(d)
    torch.testing.assert_close(U.T @ U, torch.eye(d, dtype=DT), rtol=0, atol=1e-13)


@pytest.mark.parametrize("d", [4, 8, 12, 200, 500, 516])
def test_direct_sum_fft_and_basis_agree(d):
    """the direct O(d^2) sum, irfft(conj(rfft(h)) rfft(t)) read by r, and the energy of the transformed rows"""
    codes, relt = tables(d, 9, 4, seed=d)
    X = triples(np.random.default_rng(d), 9, 4, 30)
    e = ho.energies(codes, relt, X)
    h, r, t = (np.asarray(x) for x in ho.gather(codes, relt, X))
    fft = (r * np.fft.irfft(np.conj(np.fft.rfft(h)) * np.fft.rfft(t), n=d)).sum(1)
    np.testing.assert_allclose(e.numpy(), fft, rtol=1e-11, atol=1e-11 * d)
    direct = (torch.as_tensor(r) * ho.correlate_direct(torch.as_tensor(h), torch.as_tensor(t))).sum(1)
    np.testing.assert_allclose(direct.numpy(), fft, rtol=1e-11, atol=1e-11 * d)
    torch.testing.assert_close(ho.fourier_energies(ho.transform(codes), ho.transform(relt), X), e,
                               rtol=1e-11, atol=1e-11 * d)
    # the correlation itself, column by column, written out and by FFT
    direct = ho.correlate_direct(torch.as_tensor(h), torch.as_tensor(t))
    torch.testing.assert_close(ho.correlate(torch.as_tensor(h), torch.as_tensor(t)), direct, rtol=1e-11,
                               atol=1e-11 * d)
    np.testing.assert_allclose(direct.numpy(),
                               np.fft.irfft(np.conj(np.fft.rfft(h)) * np.fft.rfft(t), n=d), rtol=1e-11,
                               atol=1e-11 * d)


def test_query_row_identities():
    """each query row scored against its table gives the gold's energy: objects w (h r), subjects w conj(r) t,
    relations w conj(h) t"""
    codes, relt = tables(12, 7, 3, seed=1)
    X = triples(np.random.default_rng(1), 7, 3, 20)
    e = ho.energies(codes, relt, X)
    for side in (0, 1, "relation"):
        S, Sg, _ = ho.scores(ho.transform(codes), ho.transform(relt), X, side)
        torch.testing.assert_close(Sg, e, rtol=1e-12, atol=1e-12)


def test_invariance_of_the_l2_term():
    codes, relt = tables(16, 7, 3, seed=2)
    X = triples(np.random.default_rng(2), 7, 3, 10)
    torch.testing.assert_close(ho.l2(ho.transform(codes), ho.transform(relt), X), ho.l2(codes, relt, X),
                               rtol=1e-13, atol=0)


def test_oracle_gradcheck():
    """the oracle's gradients are the derivatives of its losses (all three objectives, L2 included)"""
    codes, relt = tables(8, 7, 3, seed=3)
    codes.requires_grad_(True)
    relt.requires_grad_(True)
    rng = np.random.default_rng(0)
    X = triples(rng, 7, 3, 12)
    Y = torch.as_tensor(rng.integers(0, 2, 12), dtype=DT)
    assert torch.autograd.gradcheck(lambda c, r: sum(ho.ns_loss(c, r, X, Y)[:2]), (codes, relt))
    p = so.weights(ho.self_adversarial_loss(codes, relt, X, 2, 1.3)[2], 2, 1.3)
    assert torch.autograd.gradcheck(lambda c, r: sum(ho.self_adversarial_loss(c, r, X, 2, 1.3, p=p)[:2]),
                                    (codes, relt))
    qs = oo.queries(X)
    y = torch.as_tensor(oo.dense_labels(X, qs, 7))
    assert torch.autograd.gradcheck(lambda c, r: sum(ho.one_to_n_loss(c, r, qs, y, 0.1)), (codes, relt))


def test_oracle_one_to_n_is_the_direct_energy():
    """the 1-N oracle scores through the basis; its logits are the correlation energies"""
    codes, relt = tables(8, 6, 3, seed=4)
    X = triples(np.random.default_rng(4), 6, 3, 5)
    qs = oo.queries(X)
    y = torch.as_tensor(oo.dense_labels(X, qs, 6))
    full = []
    for a, r, side in qs.tolist():
        tri = [[a, r, v] if side == 1 else [v, r, a] for v in range(6)]
        full.append(ho.energies(codes, relt, np.array(tri)))
    z = torch.stack(full)
    want = (torch.clamp(z, min=0) - z * (0.9 * y + 0.1 / 6) + torch.log1p(torch.exp(-z.abs()))).mean()
    torch.testing.assert_close(ho.one_to_n_loss(codes, relt, qs, y, 0.1)[0], want, rtol=1e-12, atol=0)


# ---- settings, factory, refusals ----
def _decoder_settings(toy, **keys):
    enc, dec = merged_settings(toy, "complex.exp", toy["V"], toy["R"], len(toy["train"]))
    d = keys.pop("d", "16")
    for s in (enc, dec):
        s.put("CodeDimension", d)
    dec.put("Name", keys.pop("Name", "hole"))
    for k, v in keys.items():
        dec.put(k, v)
    return enc, dec


@pytest.mark.parametrize("objective", ["NegativeSampling", "SelfAdversarial", "1-N"])
def test_factory_builds_hole(toy, objective):
    enc, dec = _decoder_settings(toy, TrainingObjective=objective)
    encoder = model_builder.build_encoder(enc, np.array(toy["train"]))
    model = model_builder.build_decoder(encoder, dec)
    assert type(model) is HolE and model.dimension == 16 and model.next_component is encoder
    assert model.training_objective == objective and model.ensemble_fused is False and model.ONE_TO_N == "hole"
    model.set_device("cpu")
    model.initialize_train()
    # no weights of its own: the encoder's
    assert [tuple(w.shape) for w in model.get_weights()] == [(toy["V"], 16), (16,), (toy["V"], 16)]


def test_factory_refusals(toy):
    for d in ("6", "10", "18"):
        _, dec = _decoder_settings(toy, d=d)
        with pytest.raises(ValueError, match=r"the HolE decoder needs CodeDimension %% 4 == 0, got %s$" % d):
            model_builder.build_decoder(None, dec)
    _, dec = _decoder_settings(toy, TrainingObjective="1-N", LabelSmoothing="1.5")
    with pytest.raises(ValueError, match="LabelSmoothing"):
        model_builder.build_decoder(None, dec)
    _, dec = _decoder_settings(toy, TrainingObjective="Margin")
    with pytest.raises(ValueError, match="TrainingObjective must be one of"):
        model_builder.build_decoder(None, dec)
    _, dec = _decoder_settings(toy, TrainingObjective="SelfAdversarial", LabelSmoothing="0.1")
    with pytest.raises(ValueError, match="LabelSmoothing applies to TrainingObjective=1-N only"):
        model_builder.build_decoder(None, dec)
    _, dec = _decoder_settings(toy, TrainingObjective="SelfAdversarial", AdversarialTemperature="-1")
    with pytest.raises(ValueError, match="AdversarialTemperature"):
        model_builder.build_decoder(None, dec)


def test_ops_kinds():
    assert "hole" in ops.ONE_TO_N_DECODERS and "hole" in ops.SELF_ADVERSARIAL_DECODERS
    assert ops.MARGIN_DECODERS == ("rotate", "transe")
    with pytest.raises(ValueError, match="gamma"):   # HolE has no margin
        ops.self_adversarial_loss(None, None, None, 10, 1.0, "hole", gamma=1.0)
    assert not issubclass(ops.HolERanker, ops.DistMultRanker)
    assert ops.HolERanker._RANK == "rgcn_hole_rank" and ops.HolERanker._TOPK == "rgcn_hole_topk"
    # the relation candidates are the transformed relation rows themselves: DistMult's relation workspaces
    assert ops.HolERanker._REL_RANK_WORKSPACE == "rgcn_relation_rank_workspace_bytes"
    assert ops.HolERanker._REL_TOPK_WORKSPACE == "rgcn_relation_topk_workspace_bytes"
    assert ops.HolERanker.rank is ops.DistMultRanker.rank
    assert ops.HolERanker.rank_relations is ops.DistMultRanker.rank_relations


def test_slice_norms_follow_the_transform():
    """a slice norm the HolE backward leaves on a transformed table lands on the table it was made from"""
    param = torch.zeros(3)
    made = torch.zeros(3)
    made._slice_source = param
    ops._add_slice_sumsq(made, torch.tensor(2.0))
    ops._add_slice_sumsq(made, torch.tensor(1.5))
    assert float(param._slice_sumsq) == 3.5 and getattr(made, "_slice_sumsq", None) is None
    plain = torch.zeros(3)
    ops._add_slice_sumsq(plain, torch.tensor(1.0))
    assert float(plain._slice_sumsq) == 1.0


# ---- the host plugin chain with the library calls replaced by the oracle ----
# Every fake receives tables in the basis, as the library does, and takes them back to raw rows with U^T for the
# direct oracle; so the chain is checked against the O(d^2) correlation of the encoder's raw codes.
def oracle_transform(x, inverse=False):
    U = ho.basis(x.shape[-1], x.dtype)
    return x @ (U.T if inverse else U)


def _raw(*xs):
    return [oracle_transform(x, inverse=True) for x in xs]


def oracle_hole_score(codes, rel_table, X, Y=None):
    X = np.asarray(X.cpu() if torch.is_tensor(X) else X)
    codes, rel_table = _raw(codes, rel_table)
    if Y is None:
        return ho.energies(codes, rel_table, X), torch.zeros((), dtype=codes.dtype), ho.l2(codes, rel_table, X)
    L, reg, e = ho.ns_loss(codes, rel_table, X, Y)
    return e, L, reg


def oracle_query_rows(codes, rel_table, X, side):
    return ho.queries(codes, rel_table.to(codes.dtype), np.asarray(X.cpu()), side)[0]


def _lists(mask, count):
    if mask is None:
        return None
    bits = np.asarray(mask.cpu()).view(np.uint32)
    return [[v for v in range(count) if (bits[t, v >> 5] >> (v & 31)) & 1] for t in range(len(bits))]


class OracleHolERanker(object):
    def __init__(self, codes, rel_table, relation_count=None):
        self.codes, self.rel = codes.detach(), rel_table.detach()
        self.relation_count = rel_table.shape[0] if relation_count is None else relation_count

    def _scores(self, X, side, count=None):
        return ho.scores(self.codes, self.rel, np.asarray(X.cpu()), side, count)

    def rank(self, X, side, known_mask=None):
        S, _, gold = self._scores(X, side)
        raw, filt = ho.ranks(S, gold, _lists(known_mask, len(self.codes)))
        return torch.as_tensor(raw), None if filt is None else torch.as_tensor(filt)

    def top_k(self, X, side, k, exclude_mask=None):
        ids, en = ho.top_k(self._scores(X, side)[0], k, _lists(exclude_mask, len(self.codes)))
        return torch.as_tensor(ids), torch.as_tensor(en, dtype=torch.float32)

    def rank_relations(self, X, known_mask=None):
        S, _, gold = self._scores(X, "relation", self.relation_count)
        raw, filt = ho.ranks(S, gold, _lists(known_mask, self.relation_count))
        return torch.as_tensor(raw), None if filt is None else torch.as_tensor(filt)

    def top_k_relations(self, X, k, exclude_mask=None):
        S = self._scores(X, "relation", self.relation_count)[0]
        ids, en = ho.top_k(S, k, _lists(exclude_mask, self.relation_count))
        return torch.as_tensor(ids), torch.as_tensor(en, dtype=torch.float32)


class DenseLabels(object):
    def __init__(self, train, V):
        self.train, self.V = train, V

    def rows(self, queries):
        return torch.as_tensor(oo.dense_labels(self.train, queries, self.V))


@pytest.fixture
def oracle_hole(monkeypatch, oracle_backed_ops):  # noqa: F811
    calls = []

    def fake_sa(codes, rel_table, X, K, alpha, decoder, *, gamma=None):
        calls.append(("SelfAdversarial", K, alpha, decoder, gamma))
        return ho.self_adversarial_loss(*_raw(codes, rel_table), np.asarray(X.cpu()), K, alpha)

    def fake_one_to_n(codes, rel_table, queries, labels, smoothing, decoder, relation_count=None):
        calls.append(("1-N", len(queries), smoothing, decoder, relation_count))
        return ho.one_to_n_loss(*_raw(codes, rel_table), queries, labels.to(codes.dtype), smoothing)
    monkeypatch.setattr(ops, "hole_transform", oracle_transform)
    monkeypatch.setattr(ops, "hole_score", oracle_hole_score)
    monkeypatch.setattr(ops, "self_adversarial_loss", fake_sa)
    monkeypatch.setattr(ops, "one_to_n_loss", fake_one_to_n)
    monkeypatch.setattr(ops, "hole_query_rows", oracle_query_rows)
    monkeypatch.setattr(ops, "HolERanker", OracleHolERanker)
    monkeypatch.setattr(ops, "OneToNLabels", lambda train, V, R, device: DenseLabels(np.asarray(train, np.int32), V))
    return calls


def _chain_settings(toy, settings_file):
    if settings_file == "compgcn":
        enc, dec = compgcn_settings(toy, decoder="hole")
    else:
        enc, dec = merged_settings(toy, settings_file, toy["V"], toy["R"], len(toy["train"]))
        dec.put("Name", "hole")
    for s in (enc, dec):
        s.put("CodeDimension", "16")
        s.put("InternalEncoderDimension", "16")
    return enc, dec


@pytest.mark.parametrize("settings_file", ["complex.exp", "gcn_basis.exp", "compgcn"])
@pytest.mark.parametrize("objective", ["NegativeSampling", "SelfAdversarial", "1-N"])
def test_host_chain(toy, oracle_hole, oracle_compgcn, settings_file, objective):  # noqa: F811
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
        assert oracle_hole == [("SelfAdversarial", K, 1.0, "hole", None)]
        L, reg, _ = ho.self_adversarial_loss(codes, relt, X, K, 1.0)
    elif objective == "1-N":
        qs = oo.queries(X)
        assert oracle_hole == [("1-N", len(qs), 0.1, "hole", R)]
        L, reg = ho.one_to_n_loss(codes, relt, qs, torch.as_tensor(oo.dense_labels(train, qs, V)), 0.1)
    else:
        L, reg, _ = ho.ns_loss(codes, relt, X, torch.as_tensor(Y))
    param = float(dec["RegularizationParameter"])
    assert abs(total.item() - (L.item() + param * reg.item())) <= 1e-11 * abs(total.item())
    assert all(w.grad is None or torch.isfinite(w.grad).all() for w in ws)
    assert any(w.grad is not None and float(w.grad.abs().max()) > 0 for w in ws)
    # test mode: predict, the score matrices, the ranks, the top-k and the relation queries
    model.preprocess(train)
    model.register_for_test(train)
    test = np.asarray(toy["test"], np.int32)
    p = np.asarray(model.score(test))
    with torch.no_grad():
        codes, relt = [t.detach() for t in model.next_component.get_all_codes(mode='test')[:2]]
        e = ho.energies(codes, relt, test)
    np.testing.assert_allclose(p, torch.sigmoid(e).numpy(), rtol=1e-12)
    ct, rt = ho.transform(codes), ho.transform(relt)
    S1 = ho.scores(ct, rt, test, 1)[0]
    S0 = ho.scores(ct, rt, test, 0)[0]
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
    want_ids, want_en = ho.top_k(S1, 3)
    np.testing.assert_array_equal(ids, want_ids)
    np.testing.assert_allclose(en, want_en, rtol=1e-6)
    known_rel = [[int(t[1])] for t in test]
    raw, filt = model.rank_relations_all(test, known_rel)
    Sr, Srg, gold = ho.scores(ct, rt, test, "relation", R)
    np.testing.assert_array_equal(raw, (Sr >= Srg[:, None]).sum(1).numpy())
    np.testing.assert_array_equal(filt, raw)   # only the gold is known: it counts once either way
    ids, _ = model.top_k_relations_all(test, 2, known_rel)
    np.testing.assert_array_equal(ids, ho.top_k(Sr, 2, known_rel)[0])


def test_transforms_once_per_mode(toy, oracle_hole, monkeypatch):
    """the decoder transforms the entity and relation tables once per mode and feed, not once per use"""
    seen = []
    monkeypatch.setattr(ops, "hole_transform", lambda x, inverse=False: seen.append(tuple(x.shape)) or
                        oracle_transform(x, inverse))
    enc, dec = _decoder_settings(toy)
    model = model_builder.build_decoder(model_builder.build_encoder(enc, np.array(toy["train"])), dec)
    model.set_device("cpu")
    model.initialize_train()
    model.register_for_test(np.array(toy["train"]))
    test = np.array(toy["test"])[:4]
    model.score(test)
    assert len(seen) == 2
    with torch.no_grad():   # the same feed: the cached tables serve every path
        model.predict()
        model.predict_all_object_scores()
        model.predict_all_subject_scores()
    assert len(seen) == 2
    model.score(test)   # a new feed clears the caches
    assert len(seen) == 4


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


def test_ensemble_member_is_not_fused(toy, oracle_hole):
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
def test_driver_trains(toy, tmp_path, capsys, cpu_driver, oracle_hole, objective):  # noqa: F811
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(TOY_EXP.format(layers=1, concat="No").replace(
        "Name=bilinear-diag", "Name=hole\n\tTrainingObjective=%s" % objective))
    np.random.seed(0)
    torch.manual_seed(0)
    driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "40", "--device", "cpu",
                 "--no-save"])
    text = capsys.readouterr().out
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 2 and all(np.isfinite(losses)) and "Validation filtered MRR" in text
    assert all(c[0] == objective and c[3] == "hole" for c in oracle_hole)
    assert bool(oracle_hole) == (objective != "NegativeSampling")


# ---- C-ABI: every bad argument is refused before any device work (fake device pointers are never touched) ----
P = ctypes.c_void_p(256)


def _call(entry, a, kw):
    a.update(kw)
    return getattr(_lib.load(), entry)(*a.values(), None)


def _xf(**kw):
    return _call("rgcn_hole_transform", dict(x=P, rows=33, d=8, inverse=0, basis=ctypes.c_void_p(512), ready=0,
                                             out=ctypes.c_void_p(768), ws=P, wsb=1 << 40), kw)


def _fwd(**kw):
    return _call("rgcn_hole_forward", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, N=33, Y=P, energies=P, loss=P), kw)


def _bwd(**kw):
    return _call("rgcn_hole_backward", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, N=33, Y=P, energies=P,
                                            g_loss=1.0, g_reg=1.0, g_scale=None, g_energy=None, dcodes=P, drel=P,
                                            ss=None), kw)


def _sa(**kw):
    return _call("rgcn_hole_self_adversarial_forward", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, N=33, K=10,
                                                            alpha=1.0, energies=P, coef=P, loss=P, ws=P,
                                                            wsb=1 << 40), kw)


def _rank(**kw):
    return _call("rgcn_hole_rank", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, n=5, side=1, known=P, reuse=0,
                                        raw=P, filt=P, ws=P, wsb=1 << 40), kw)


def _topk(**kw):
    return _call("rgcn_hole_topk", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, n=5, side=1, k=4, excl=None,
                                        reuse=0, ids=P, energies=P, ws=P, wsb=1 << 40), kw)


def _rrank(**kw):
    return _call("rgcn_hole_relation_rank", dict(codes=P, rel=P, V=10, Vrel=10, R=4, d=8, X=P, n=5, known=P,
                                                 reuse=0, raw=P, filt=P, ws=P, wsb=1 << 40), kw)


def _rtopk(**kw):
    return _call("rgcn_hole_relation_topk", dict(codes=P, rel=P, V=10, Vrel=10, R=4, d=8, X=P, n=5, k=4, excl=None,
                                                 reuse=0, ids=P, energies=P, ws=P, wsb=1 << 40), kw)


QUERIES = np.array([[1, 2, 1], [3, 0, 0]], np.int32)


def _onen(**kw):
    q = kw.pop("queries", QUERIES)
    return _call("rgcn_hole_one_to_n", dict(codes=P, rel=P, V=10, Vrel=10, R=4, d=8, queries=q.ctypes.data,
                                            n=len(q), labels=P, eps=0.0, g_scale=None, loss=P, dcodes=P, drel=P,
                                            chunk=64, ws=P, wsb=1 << 40), kw)


def _rows(**kw):
    return _call("rgcn_hole_query_rows", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, n=5, side=1, Q=P), kw)


SIZES = [dict(V=0), dict(Vrel=0), dict(d=0), dict(d=6), dict(d=-4), dict(d=10)]
QUERY = SIZES + [dict(codes=None), dict(rel=None), dict(X=None), dict(ws=None), dict(n=-1)]
INVALID = ([(_xf, b) for b in [dict(d=0), dict(d=6), dict(d=-4), dict(rows=-1), dict(rows=1 << 31), dict(inverse=2),
                               dict(inverse=-1), dict(x=None), dict(out=None), dict(basis=None), dict(ws=None),
                               dict(out=P)]] +
           [(_fwd, b) for b in SIZES + [dict(codes=None), dict(rel=None), dict(X=None), dict(energies=None),
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
    assert lib.rgcn_hole_transform_workspace_bytes(8) >= 2 * 8 * 8 * 4
    assert lib.rgcn_hole_transform_workspace_bytes(500) >= 2 * 500 * 500 * 4
    for bad in (0, 6, -4):
        assert lib.rgcn_hole_transform_workspace_bytes(bad) == -1
    rank_need = lib.distmult_rank_workspace_bytes(10, 8, 5)
    topk_need = lib.rgcn_topk_workspace_bytes(10, 8, 5, 4)
    rrank_need = lib.rgcn_relation_rank_workspace_bytes(4, 8, 5)
    rtopk_need = lib.rgcn_relation_topk_workspace_bytes(4, 8, 5, 4)
    assert _xf(wsb=lib.rgcn_hole_transform_workspace_bytes(8) - 1) == -4
    assert _rank(wsb=rank_need - 1) == -4 and _topk(wsb=topk_need - 1) == -4
    assert _rrank(wsb=rrank_need - 1) == -4 and _rtopk(wsb=rtopk_need - 1) == -4
    assert _sa(wsb=lib.rgcn_self_adversarial_workspace_bytes(33, 10) - 1) == -4
    assert _onen(wsb=lib.rgcn_one_to_n_workspace_bytes(10, 8, 2, 64) - 1) == -4
    if torch.cuda.is_available():
        pytest.skip("a device is present: valid arguments would run")
    assert _xf() == -5 and _fwd() == -5 and _bwd() == -5 and _sa() == -5 and _rows() == -5
    assert _onen(wsb=lib.rgcn_one_to_n_workspace_bytes(10, 8, 2, 64)) == -5
