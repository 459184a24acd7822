"""CPU: the TransE decoder -- the float64 oracle (gradcheck, the zero-residual subgradient, the self-adversarial
identities, ranks and top-k), the Margin key and every refusal, the factory, the host plugin chain and the training
driver with the library calls replaced by the oracle (the substitution lives in this file; the product has no CPU
path), a checkpoint round trip, and the C-ABI argument checks, which all return before any device work."""
import ctypes

import numpy as np
import pytest
import torch

import self_adversarial_oracle as so
import transe_oracle as to
from relationprediction_b200 import _lib, ops
from relationprediction_b200 import ensemble as ens_mod
from relationprediction_b200 import train as driver
from relationprediction_b200.common import evaluation, model_builder
from relationprediction_b200.decoders.rotate import Rotate
from relationprediction_b200.decoders.transe import TransE
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
def test_oracle_energy_is_the_l1_translation_distance():
    codes, relt = tables(8, 6, 3, seed=1)
    X = triples(np.random.default_rng(1), 6, 3, 10)
    e = to.energies(codes, relt, X, 5.0)
    want = [5.0 - float((codes[s] + relt[r] - codes[o]).abs().sum()) for s, r, o in X]
    np.testing.assert_allclose(e.numpy(), want, rtol=1e-13)


def test_oracle_gradcheck():
    """away from u = 0 the oracle's gradients are the derivatives of its loss (both objectives, L2 included)"""
    codes, relt = tables(8, 7, 3, seed=3)
    codes.requires_grad_(True)
    relt.requires_grad_(True)
    rng = np.random.default_rng(0)
    X = triples(rng, 7, 3, 12)
    Y = torch.as_tensor(rng.integers(0, 2, 12), dtype=DT)
    assert torch.autograd.gradcheck(lambda c, r: sum(to.ns_loss(c, r, X, Y, 2.0)[:2]), (codes, relt))
    p = so.weights(to.self_adversarial_loss(codes, relt, X, 2, 1.3, 2.0)[2], 2, 1.3)
    assert torch.autograd.gradcheck(lambda c, r: sum(to.self_adversarial_loss(c, r, X, 2, 1.3, 2.0, p=p)[:2]),
                                    (codes, relt))


def test_oracle_zero_residual_subgradient():
    """u = 0 in every column (r = 0, s = o): the distance contributes nothing, the L2 term alone moves the rows"""
    codes, relt = tables(8, 4, 2, seed=4)
    relt[0] = 0.0
    codes.requires_grad_(True)
    relt.requires_grad_(True)
    X = np.array([[2, 0, 2]], np.int32)
    L, reg, e = to.ns_loss(codes, relt, X, torch.ones(1, dtype=DT), 3.0)
    assert float(e[0].detach()) == 3.0
    (L + reg).backward()
    # reg = mean(h^2) + mean(r^2) + mean(t^2) with h = t = codes[2], r = 0
    torch.testing.assert_close(codes.grad[2], 4.0 * codes[2].detach() / 8, rtol=1e-14, atol=0)
    assert float(relt.grad.abs().max()) == 0.0


def test_oracle_gradient_is_the_sign():
    codes, relt = tables(8, 5, 2, seed=7)
    codes.requires_grad_(True)
    relt.requires_grad_(True)
    X = np.array([[0, 1, 3]], np.int32)
    to.energies(codes, relt, X, 1.0).sum().backward()
    s = torch.sign(codes[0] + relt[1] - codes[3]).detach()
    assert torch.equal(codes.grad[0], -s) and torch.equal(relt.grad[1], -s) and torch.equal(codes.grad[3], s)


def test_oracle_self_adversarial_identities():
    codes, relt = tables(8, 9, 3, seed=5)
    rng = np.random.default_rng(2)
    n = 6
    X1 = triples(rng, 9, 3, 2 * n)
    for alpha in (0.0, 1.0, 5.0):   # K = 1: the NegativeSampling loss
        L, _, e = to.self_adversarial_loss(codes, relt, X1, 1, alpha, 4.0)
        y = torch.cat([torch.ones(n, dtype=DT), torch.zeros(n, dtype=DT)])
        assert abs(float(L - to.ns_loss(codes, relt, X1, y, 4.0)[0])) < 1e-12
    K = 4
    X = triples(rng, 9, 3, n * (K + 1))
    L, _, e = to.self_adversarial_loss(codes, relt, X, K, 0.0, 4.0)   # alpha = 0: p = 1/K
    b = e.reshape(K + 1, n)
    assert abs(float(L - (so.softplus(-b[0]).sum() + so.softplus(b[1:]).sum() / K) / (2 * n))) < 1e-12


def test_oracle_ranks_and_top_k_follow_the_rules():
    codes, relt = tables(8, 12, 5, seed=6, scale=1.0)
    X = triples(np.random.default_rng(3), 12, 5, 20)
    for side in (0, 1, "relation"):
        D, Dg, gold = to.distances(codes, relt, X, side)
        C = D.shape[1]
        known = [[int(g), (int(g) + 1) % C] for g in gold]
        raw, filt = to.ranks(codes, relt, X, side, known)
        np.testing.assert_array_equal(raw, (D <= Dg[:, None]).sum(1).numpy())
        assert (raw >= 1).all() and (filt >= 1).all() and (filt <= raw).all()
        # every query's gold distance is the triple's own: gamma - D_gold is the energy
        np.testing.assert_allclose(Dg.numpy(), 7.0 - to.energies(codes, relt, X, 7.0).numpy(), rtol=1e-12)
        ids, en = to.top_k(D, 4, 7.0, known)
        for t in range(len(X)):
            assert not set(ids[t].tolist()) & set(known[t])
            assert (np.diff(en[t]) <= 0).all()
    # ties go to the smaller id; short rows end in (-1, -inf)
    ids, en = to.top_k(np.array([[1.0, 0.5, 1.0, 0.5]]), 4, 2.0, [[1]])
    assert ids.tolist() == [[3, 0, 2, -1]] and en.tolist() == [[1.5, 1.0, 1.0, -np.inf]]


# ---- settings, factory, refusals ----
def _decoder_settings(toy, **keys):
    enc, dec = merged_settings(toy, "complex.exp", toy["V"], toy["R"], len(toy["train"]))
    d = keys.pop("d", "16")
    for s in (enc, dec):
        s.put("CodeDimension", d)
    dec.put("Name", "transe")
    for k, v in keys.items():
        dec.put(k, v)
    return enc, dec


def test_factory_builds_transe(toy):
    enc, dec = _decoder_settings(toy, Margin="9")
    encoder = model_builder.build_encoder(enc, np.array(toy["train"]))
    model = model_builder.build_decoder(encoder, dec)
    assert type(model) is TransE and not isinstance(model, Rotate)
    assert model.margin == 9.0 and model.dimension == 16 and model.next_component is encoder
    assert model.training_objective == 'NegativeSampling' and model.ensemble_fused is False
    model.set_device("cpu")
    model.initialize_train()
    ws = model.get_weights()
    assert [tuple(w.shape) for w in ws] == [(toy["V"], 16), (16,), (toy["V"], 16)]   # the relation table keeps [V, d]
    _, dec = _decoder_settings(toy)
    assert model_builder.build_decoder(encoder, dec).margin == 12.0
    _, dec = _decoder_settings(toy, Margin="-2.5")
    assert model_builder.build_decoder(encoder, dec).margin == -2.5
    _, dec = _decoder_settings(toy, TrainingObjective="SelfAdversarial", AdversarialTemperature="0.5")
    m = model_builder.build_decoder(encoder, dec)
    assert m.training_objective == 'SelfAdversarial' and m.adversarial_temperature == 0.5


def test_factory_refusals(toy):
    for d in ("6", "10", "18"):
        enc, dec = _decoder_settings(toy, d=d)
        with pytest.raises(ValueError, match="CodeDimension % 4"):
            model_builder.build_decoder(None, dec)
    for bad in ("nan", "inf"):
        _, dec = _decoder_settings(toy, Margin=bad)
        with pytest.raises(ValueError, match="Margin"):
            model_builder.build_decoder(None, dec)
    _, dec = _decoder_settings(toy, TrainingObjective="1-N")
    with pytest.raises(ValueError, match=r"TrainingObjective=1-N needs the bilinear-diag or complex decoder, "
                                         r"not 'transe'"):
        model_builder.build_decoder(None, dec)


def test_ops_refusals():
    with pytest.raises(ValueError, match="gamma"):
        ops.self_adversarial_loss(None, None, None, 10, 1.0, "transe", gamma=float("nan"))
    with pytest.raises(ValueError, match="gamma"):
        ops.self_adversarial_loss(None, None, None, 10, 1.0, "complex", gamma=1.0)
    with pytest.raises(ValueError, match="gamma"):
        ops.transe_score(None, None, None, gamma=float("inf"))
    with pytest.raises(ValueError, match="decoder"):   # TransE has no 1-N objective
        ops.one_to_n_loss(None, None, np.zeros((1, 3), np.int32), None, 0.0, "transe")
    assert "transe" not in ops.ONE_TO_N_DECODERS and "transe" in ops.SELF_ADVERSARIAL_DECODERS


# ---- the host plugin chain with the library calls replaced by the oracle ----
def oracle_transe_score(codes, rel_table, X, Y=None, *, gamma):
    X = np.asarray(X.cpu() if torch.is_tensor(X) else X)
    if Y is None:
        e = to.energies(codes, rel_table, X, gamma)
        return e, torch.zeros((), dtype=codes.dtype), to.l2(codes, rel_table, X)
    L, reg, e = to.ns_loss(codes, rel_table, X, Y, gamma)
    return e, L, reg


def _lists(mask, count):
    if mask is None:
        return None
    bits = np.asarray(mask.cpu()).view(np.uint32)
    return [[v for v in range(count) if (bits[t, v >> 5] >> (v & 31)) & 1] for t in range(len(bits))]


class OracleTransERanker(object):
    def __init__(self, codes, rel_table, relation_count=None, gamma=0.0):
        self.codes, self.rel, self.gamma = codes.detach(), rel_table.detach(), gamma
        self.relation_count = rel_table.shape[0] if relation_count is None else relation_count

    def rank(self, X, side, known_mask=None):
        raw, filt = to.ranks(self.codes, self.rel, np.asarray(X.cpu()), side, _lists(known_mask, len(self.codes)))
        return torch.as_tensor(raw), None if filt is None else torch.as_tensor(filt)

    def top_k(self, X, side, k, exclude_mask=None):
        D = to.distances(self.codes, self.rel, np.asarray(X.cpu()), side)[0]
        ids, en = to.top_k(D, k, self.gamma, _lists(exclude_mask, len(self.codes)))
        return torch.as_tensor(ids), torch.as_tensor(en, dtype=torch.float32)

    def rank_relations(self, X, known_mask=None):
        R = self.relation_count
        raw, filt = to.ranks(self.codes, self.rel, np.asarray(X.cpu()), "relation", _lists(known_mask, R), R)
        return torch.as_tensor(raw), None if filt is None else torch.as_tensor(filt)

    def top_k_relations(self, X, k, exclude_mask=None):
        R = self.relation_count
        D = to.distances(self.codes, self.rel, np.asarray(X.cpu()), "relation", R)[0]
        ids, en = to.top_k(D, k, self.gamma, _lists(exclude_mask, R))
        return torch.as_tensor(ids), torch.as_tensor(en, dtype=torch.float32)


@pytest.fixture
def oracle_transe(monkeypatch, oracle_backed_ops):  # noqa: F811
    calls = []

    def fake_sa(codes, rel_table, X, K, alpha, decoder, *, gamma=None):
        calls.append((K, alpha, decoder, gamma))
        return to.self_adversarial_loss(codes, rel_table, np.asarray(X.cpu()), K, alpha, gamma)
    monkeypatch.setattr(ops, "transe_score", oracle_transe_score)
    monkeypatch.setattr(ops, "self_adversarial_loss", fake_sa)
    monkeypatch.setattr(ops, "TransERanker", OracleTransERanker)
    return calls


def _chain_settings(toy, settings_file):
    if settings_file == "compgcn":
        enc, dec = compgcn_settings(toy, decoder="transe")
    else:
        enc, dec = merged_settings(toy, settings_file, toy["V"], toy["R"], len(toy["train"]))
        dec.put("Name", "transe")
    for s in (enc, dec):
        s.put("CodeDimension", "16")
        s.put("InternalEncoderDimension", "16")
    return enc, dec


@pytest.mark.parametrize("settings_file", ["complex.exp", "gcn_basis.exp", "compgcn"])
@pytest.mark.parametrize("objective", ["NegativeSampling", "SelfAdversarial"])
def test_host_chain(toy, oracle_transe, oracle_compgcn, settings_file, objective):  # noqa: F811
    train = np.asarray(toy["train"], np.int32)
    V, R = int(toy["V"]), int(toy["R"])
    enc, dec = _chain_settings(toy, settings_file)
    dec.put("Margin", "4")
    dec.put("TrainingObjective", objective)
    model = model_builder.build_decoder(model_builder.build_encoder(enc, train), dec)
    model.set_device("cpu")
    model.initialize_train()
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
        assert oracle_transe == [(K, 1.0, "transe", 4.0)]
        L, reg, _ = to.self_adversarial_loss(codes, relt, X, K, 1.0, 4.0)
    else:
        L, reg, _ = to.ns_loss(codes, relt, X, torch.as_tensor(Y), 4.0)
    param = float(dec["RegularizationParameter"])
    assert abs(total.item() - (L.item() + param * reg.item())) <= 1e-12 * abs(total.item())
    assert all(w.grad is None or torch.isfinite(w.grad).all() for w in ws)
    assert any(w.grad is not None and float(w.grad.abs().max()) > 0 for w in ws)
    # test mode: predict, the score matrices (float32 sigmoid of the energy), the ranks and the top-k
    model.preprocess(train)
    model.register_for_test(train)
    test = np.asarray(toy["test"], np.int32)
    p = np.asarray(model.score(test))
    with torch.no_grad():
        codes, relt = [t.detach() for t in model.next_component.get_all_codes(mode='test')[:2]]
        e = to.energies(codes, relt, test, 4.0)
    np.testing.assert_allclose(p, torch.sigmoid(e).numpy(), rtol=1e-12)
    D1, _, _ = to.distances(codes, relt, test, 1)
    D0, _, _ = to.distances(codes, relt, test, 0)
    np.testing.assert_allclose(model.score_all_objects(test), torch.sigmoid(4.0 - D1).numpy(), rtol=1e-12)
    np.testing.assert_allclose(model.score_all_subjects(test), torch.sigmoid(4.0 - D0).numpy(), rtol=1e-12)
    sc = evaluation.Scorer({'Metric': 'MRR'})
    sc.register_data(train)
    sc.register_data(test)
    sc.register_model(model)
    matrices = sc.compute_scores(test)
    fused = model.rank_all(test, [sc.known_subject_triples.get((t[2], t[1]), []) for t in test.tolist()],
                           [sc.known_object_triples.get((t[0], t[1]), []) for t in test.tolist()])
    assert np.concatenate([fused[0], fused[2]]).tolist() == matrices.raw_ranks
    assert np.concatenate([fused[1], fused[3]]).tolist() == matrices.filtered_ranks
    # top-k through the decoder's hooks: the oracle's order, energies gamma - D
    ids, en = model.top_k_all(test, 3, 1)
    want_ids, want_en = to.top_k(D1, 3, 4.0)
    np.testing.assert_array_equal(ids, want_ids)
    np.testing.assert_allclose(en, want_en, rtol=1e-6)
    known_rel = [[int(t[1])] for t in test]
    raw, filt = model.rank_relations_all(test, known_rel)
    Dr, Drg, _ = to.distances(codes, relt, test, "relation", R)
    np.testing.assert_array_equal(raw, (Dr <= Drg[:, None]).sum(1).numpy())
    np.testing.assert_array_equal(filt, raw)   # only the gold is known: it counts once either way
    ids, _ = model.top_k_relations_all(test, 2, known_rel)
    np.testing.assert_array_equal(ids, to.top_k(Dr, 2, 4.0, known_rel)[0])


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


def test_no_fused_ensemble(toy, oracle_transe):
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


@pytest.mark.parametrize("objective", ["NegativeSampling", "SelfAdversarial"])
def test_driver_trains(toy, tmp_path, capsys, cpu_driver, oracle_transe, objective):  # noqa: F811
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(TOY_EXP.format(layers=1, concat="No").replace(
        "Name=bilinear-diag", "Name=transe\n\tMargin=6\n\tTrainingObjective=%s" % objective))
    np.random.seed(0)
    torch.manual_seed(0)
    driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "40", "--device", "cpu",
                 "--no-save"])
    text = capsys.readouterr().out
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 2 and all(np.isfinite(losses)) and "Validation filtered MRR" in text
    assert all(c[2:] == ("transe", 6.0) for c in oracle_transe)
    assert bool(oracle_transe) == (objective == "SelfAdversarial")


# ---- C-ABI: every bad argument is refused before any device work (fake device pointers are never touched) ----
P = ctypes.c_void_p(256)


def _call(entry, a, kw):
    a.update(kw)
    return getattr(_lib.load(), entry)(*a.values(), None)


def _fwd(**kw):
    return _call("rgcn_transe_forward", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, N=33, Y=P, gamma=12.0,
                                             energies=P, loss=P), kw)


def _bwd(**kw):
    return _call("rgcn_transe_backward", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, N=33, Y=P, gamma=12.0,
                                              energies=P, g_loss=1.0, g_reg=1.0, g_scale=None, g_energy=None,
                                              dcodes=P, drel=P, ss=None), kw)


def _sa(**kw):
    return _call("rgcn_transe_self_adversarial_forward", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, N=33, K=10,
                                                              alpha=1.0, gamma=12.0, energies=P, coef=P, loss=P, ws=P,
                                                              wsb=1 << 40), kw)


def _rank(**kw):
    return _call("rgcn_transe_rank", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, n=5, side=1, known=P, raw=P,
                                          filt=P, ws=P, wsb=1 << 40), kw)


def _topk(**kw):
    return _call("rgcn_transe_topk", dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, n=5, side=1, k=4, excl=None,
                                          gamma=12.0, ids=P, energies=P, ws=P, wsb=1 << 40), kw)


def _rrank(**kw):
    return _call("rgcn_transe_relation_rank", dict(codes=P, rel=P, V=10, Vrel=10, R=4, d=8, X=P, n=5, known=P, raw=P,
                                                   filt=P, ws=P, wsb=1 << 40), kw)


def _rtopk(**kw):
    return _call("rgcn_transe_relation_topk", dict(codes=P, rel=P, V=10, Vrel=10, R=4, d=8, X=P, n=5, k=4, excl=None,
                                                   gamma=12.0, ids=P, energies=P, ws=P, wsb=1 << 40), kw)


SIZES = [dict(V=0), dict(Vrel=0), dict(d=0), dict(d=6), dict(d=-4), dict(d=10)]
GAMMAS = [dict(gamma=float("inf")), dict(gamma=float("-inf")), dict(gamma=float("nan"))]
QUERY = SIZES + [dict(codes=None), dict(rel=None), dict(X=None), dict(ws=None), dict(n=-1)]
INVALID = ([(_fwd, b) for b in SIZES + GAMMAS + [dict(codes=None), dict(rel=None), dict(X=None), dict(energies=None),
                                                   dict(loss=None), dict(N=-1)]] +
           [(_bwd, b) for b in SIZES + GAMMAS + [dict(codes=None), dict(rel=None), dict(X=None), dict(dcodes=None),
                                                   dict(drel=None), dict(energies=None), dict(N=-1)]] +
           [(_sa, b) for b in SIZES + GAMMAS + [dict(codes=None), dict(X=None), dict(coef=None), dict(ws=None),
                                                   dict(N=34), dict(K=0), dict(alpha=-1.0), dict(alpha=float("nan"))]] +
           [(_rank, b) for b in QUERY + [dict(raw=None), dict(side=2), dict(side=-1), dict(known=None)]] +
           [(_topk, b) for b in QUERY + GAMMAS + [dict(ids=None), dict(energies=None), dict(side=2), dict(side=-1),
                                                  dict(k=0), dict(k=129)]] +
           [(_rrank, b) for b in QUERY + [dict(raw=None), dict(known=None), dict(R=0), dict(R=11)]] +
           [(_rtopk, b) for b in QUERY + GAMMAS + [dict(ids=None), dict(energies=None), dict(k=0), dict(k=129),
                                                   dict(R=0), dict(R=11)]])


@pytest.mark.parametrize("fn,bad", INVALID, ids=lambda x: x.__name__ if callable(x) else
                         "-".join("%s=%s" % kv for kv in x.items()))
def test_cabi_rejects_bad_arguments(fn, bad):
    assert fn(**bad) == -1, _lib.load().rgcn_last_error()


def test_cabi_workspace_and_device():
    lib = _lib.load()
    rank_need = lib.rgcn_transe_rank_workspace_bytes(10, 8, 5)
    topk_need = lib.rgcn_transe_topk_workspace_bytes(10, 8, 5, 4)
    rrank_need = lib.rgcn_transe_relation_rank_workspace_bytes(4, 8, 5)
    rtopk_need = lib.rgcn_transe_relation_topk_workspace_bytes(4, 8, 5, 4)
    assert rank_need >= 5 * 8 * 4 + 4 * 5 * 4 and topk_need >= 5 * 8 * 4 + 5 * 4 * 8
    assert rrank_need >= 5 * 8 * 4 + 4 * 5 * 4 and rtopk_need >= 5 * 8 * 4 + 5 * 4 * 8
    for fn in (lib.rgcn_transe_rank_workspace_bytes, lib.rgcn_transe_relation_rank_workspace_bytes):
        for bad in ((0, 8, 5), (10, 6, 5), (10, 8, -1)):
            assert fn(*bad) == -1
    for fn in (lib.rgcn_transe_topk_workspace_bytes, lib.rgcn_transe_relation_topk_workspace_bytes):
        for bad in ((0, 8, 5, 4), (10, 6, 5, 4), (10, 8, -1, 4), (10, 8, 5, 0), (10, 8, 5, 129)):
            assert fn(*bad) == -1
    assert _rank(wsb=rank_need - 1) == -4 and _topk(wsb=topk_need - 1) == -4
    assert _rrank(wsb=rrank_need - 1) == -4 and _rtopk(wsb=rtopk_need - 1) == -4
    assert _sa(wsb=lib.rgcn_self_adversarial_workspace_bytes(33, 10) - 1) == -4
    if torch.cuda.is_available():
        pytest.skip("a device is present: valid arguments would run")
    assert _fwd() == -5 and _bwd() == -5 and _sa() == -5
    assert _rank(wsb=rank_need) == -5 and _topk(wsb=topk_need) == -5
    assert _rrank(wsb=rrank_need) == -5 and _rtopk(wsb=rtopk_need) == -5
