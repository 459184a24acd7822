"""CPU: the RotatE decoder -- the float64 oracle (gradcheck, the zero-residual subgradient, the two self-adversarial
identities, the ranks), the Margin key and every refusal, the factory, the host plugin chain and the training driver
with the library calls replaced by the oracle (the substitution lives in this file; the product has no CPU path), a
checkpoint round trip, and the C-ABI argument checks, which all return before any device work."""
import ctypes

import numpy as np
import pytest
import torch

import rotate_oracle as ro
import self_adversarial_oracle as so
from relationprediction_b200 import _lib, ops
from relationprediction_b200 import ensemble as ens_mod
from relationprediction_b200 import train as driver
from relationprediction_b200.common import evaluation, model_builder
from relationprediction_b200.decoders.rotate import Rotate, parse_margin
from test_gpu_train import TOY_EXP, write_toy
from test_plugin_chain_cpu import oracle_backed_ops  # noqa: F401  (fixture)
from test_plugin_host import merged_settings
from test_train_loop_cpu import cpu_driver  # noqa: F401  (fixture)

DT = torch.float64


def tables(d, V, R, seed=0, scale=0.5):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(V, d, dtype=DT, generator=g) * scale, torch.randn(R, d, dtype=DT, generator=g) * 2.0


def triples(rng, V, R, N):
    return np.stack([rng.integers(0, V, N), rng.integers(0, R, N), rng.integers(0, V, N)], 1).astype(np.int32)


# ---- the oracle ----
def test_oracle_energy_is_the_complex_distance():
    codes, relt = tables(8, 6, 3, seed=1)
    X = triples(np.random.default_rng(1), 6, 3, 10)
    e = ro.energies(codes, relt, X, 5.0)
    z = codes[:, :4] + 1j * codes[:, 4:]
    th = relt[:, :4]
    want = [5.0 - float(torch.abs(z[s] * torch.exp(1j * th[r]) - z[o]).sum()) for s, r, o in X]
    np.testing.assert_allclose(e.numpy(), want, rtol=1e-13)


def test_oracle_gradcheck():
    """away from u = 0 the oracle's gradients are the derivatives of its loss (both objectives, L2 included)"""
    codes, relt = tables(8, 7, 3, seed=3)
    codes.requires_grad_(True)
    relt.requires_grad_(True)
    rng = np.random.default_rng(0)
    X = triples(rng, 7, 3, 12)
    Y = torch.as_tensor(rng.integers(0, 2, 12), dtype=DT)
    assert torch.autograd.gradcheck(lambda c, r: sum(ro.ns_loss(c, r, X, Y, 2.0)[:2]), (codes, relt))
    Xs = np.concatenate([X[:4], X[4:8], X[8:12]])
    p = so.weights(ro.self_adversarial_loss(codes, relt, Xs, 2, 1.3, 2.0)[2], 2, 1.3)
    assert torch.autograd.gradcheck(lambda c, r: sum(ro.self_adversarial_loss(c, r, Xs, 2, 1.3, 2.0, p=p)[:2]),
                                    (codes, relt))


def test_oracle_zero_residual_subgradient():
    """u = 0 (theta = 0, s = o): the modulus contributes nothing, the L2 term alone moves the entity row, and the
    phases get exactly zero"""
    codes, relt = tables(8, 4, 2, seed=4)
    relt[0, :4] = 0.0
    codes.requires_grad_(True)
    relt.requires_grad_(True)
    X = np.array([[2, 0, 2]], np.int32)
    L, reg, e = ro.ns_loss(codes, relt, X, torch.ones(1, dtype=DT), 3.0)
    assert float(e[0].detach()) == 3.0
    (L + reg).backward()
    # dL/dE only reaches the rows through u: nothing; reg = mean(a^2) + mean(c^2) with a = c = codes[2]
    torch.testing.assert_close(codes.grad[2], 4.0 * codes[2].detach() / 8, rtol=1e-14, atol=0)
    assert float(relt.grad.abs().max()) == 0.0


def test_oracle_self_adversarial_identities():
    codes, relt = tables(8, 9, 3, seed=5)
    rng = np.random.default_rng(2)
    n = 6
    X1 = triples(rng, 9, 3, 2 * n)
    for alpha in (0.0, 1.0, 5.0):   # K = 1: the NegativeSampling loss
        L, _, e = ro.self_adversarial_loss(codes, relt, X1, 1, alpha, 4.0)
        y = torch.cat([torch.ones(n, dtype=DT), torch.zeros(n, dtype=DT)])
        assert abs(float(L - ro.ns_loss(codes, relt, X1, y, 4.0)[0])) < 1e-12
    K = 4
    X = triples(rng, 9, 3, n * (K + 1))
    L, _, e = ro.self_adversarial_loss(codes, relt, X, K, 0.0, 4.0)   # alpha = 0: p = 1/K
    b = e.reshape(K + 1, n)
    assert abs(float(L - (so.softplus(-b[0]).sum() + so.softplus(b[1:]).sum() / K) / (2 * n))) < 1e-12


def test_oracle_ranks_follow_the_counting_rules():
    codes, relt = tables(8, 12, 3, seed=6, scale=1.0)
    X = triples(np.random.default_rng(3), 12, 3, 20)
    for side in (0, 1):
        D, Dg, gold = ro.distances(codes, relt, X, side)
        known = [[int(g), (int(g) + 1) % 12] for g in gold]
        raw, filt = ro.ranks(codes, relt, X, side, known)
        np.testing.assert_array_equal(raw, (D <= Dg[:, None]).sum(1).numpy())
        assert (raw >= 1).all() and (filt >= 1).all() and (filt <= raw).all()
        # side 0 ranks the subjects by the same energy: D_gold is the triple's own distance
        np.testing.assert_allclose(Dg.numpy(), 7.0 - ro.energies(codes, relt, X, 7.0).numpy(), rtol=1e-12)


# ---- settings, factory, refusals ----
def _decoder_settings(toy, **keys):
    enc, dec = merged_settings(toy, "complex.exp", toy["V"], toy["R"], len(toy["train"]))
    d = keys.pop("d", "16")
    for s in (enc, dec):
        s.put("CodeDimension", d)
    dec.put("Name", "rotate")
    for k, v in keys.items():
        dec.put(k, v)
    return enc, dec


def test_margin_parsing():
    assert parse_margin({}) == 12.0
    assert parse_margin({'Margin': '0'}) == 0.0
    assert parse_margin({'Margin': '-3.5'}) == -3.5
    for bad in ('inf', '-inf', 'nan'):
        with pytest.raises(ValueError, match="Margin"):
            parse_margin({'Margin': bad})


def test_factory_builds_rotate(toy):
    enc, dec = _decoder_settings(toy, Margin="9")
    encoder = model_builder.build_encoder(enc, np.array(toy["train"]))
    model = model_builder.build_decoder(encoder, dec)
    assert type(model) is Rotate and model.margin == 9.0 and model.dimension == 16 and model.next_component is encoder
    assert model.training_objective == 'NegativeSampling'
    model.set_device("cpu")
    model.initialize_train()
    ws = model.get_weights()
    assert [tuple(w.shape) for w in ws] == [(toy["V"], 16), (16,), (toy["V"], 16)]   # the relation table keeps [V, d]
    _, dec = _decoder_settings(toy)
    assert model_builder.build_decoder(encoder, dec).margin == 12.0
    _, dec = _decoder_settings(toy, TrainingObjective="SelfAdversarial", AdversarialTemperature="0.5")
    m = model_builder.build_decoder(encoder, dec)
    assert m.training_objective == 'SelfAdversarial' and m.adversarial_temperature == 0.5


def test_factory_refusals(toy):
    for d in ("6", "10", "18"):
        enc, dec = _decoder_settings(toy, d=d)
        with pytest.raises(ValueError, match="CodeDimension % 4"):
            model_builder.build_decoder(None, dec)
    _, dec = _decoder_settings(toy, Margin="nan")
    with pytest.raises(ValueError, match="Margin"):
        model_builder.build_decoder(None, dec)
    _, dec = _decoder_settings(toy, TrainingObjective="1-N")
    with pytest.raises(ValueError, match=r"TrainingObjective=1-N needs the bilinear-diag or complex decoder, "
                                         r"not 'rotate'"):
        model_builder.build_decoder(None, dec)
    # the other names are untouched
    assert model_builder.build_decoder(None, {'Name': 'nonlinear-transform'}) is None
    with pytest.raises(ValueError, match="TrainingObjective=SelfAdversarial"):
        model_builder.build_decoder(None, {'Name': 'nonlinear-transform', 'TrainingObjective': 'SelfAdversarial'})


def test_ops_refusals():
    with pytest.raises(ValueError, match="gamma"):
        ops.self_adversarial_loss(None, None, None, 10, 1.0, "rotate")
    with pytest.raises(ValueError, match="gamma"):
        ops.self_adversarial_loss(None, None, None, 10, 1.0, "distmult", gamma=12.0)
    with pytest.raises(ValueError, match="gamma"):
        ops.self_adversarial_loss(None, None, None, 10, 1.0, "rotate", gamma=float("inf"))
    with pytest.raises(ValueError, match="decoder"):
        ops.self_adversarial_loss(None, None, None, 10, 1.0, "transe")
    with pytest.raises(ValueError, match="gamma"):
        ops.rotate_score(None, None, None, gamma=float("nan"))
    ranker = ops.RotateRanker.__new__(ops.RotateRanker)
    for call in (lambda: ranker.top_k(None, 1, 5), lambda: ranker.rank_relations(None),
                 lambda: ranker.top_k_relations(None, 5)):
        with pytest.raises(NotImplementedError, match="RotatE"):
            call()


# ---- the host plugin chain with the library calls replaced by the oracle ----
def oracle_rotate_score(codes, rel_table, X, Y=None, *, gamma):
    X = np.asarray(X.cpu() if torch.is_tensor(X) else X)
    if Y is None:
        e = ro.energies(codes, rel_table, X, gamma)
        return e, torch.zeros((), dtype=codes.dtype), ro.l2(codes, X)
    L, reg, e = ro.ns_loss(codes, rel_table, X, Y, gamma)
    return e, L, reg


class OracleRotateRanker(object):
    def __init__(self, codes, rel_table, relation_count=None):
        self.codes, self.rel = codes, rel_table

    def rank(self, X, side, known_mask=None):
        X = np.asarray(X.cpu())
        known = None
        if known_mask is not None:
            bits = np.asarray(known_mask.cpu()).view(np.uint32)
            known = [[v for v in range(len(self.codes)) if (bits[t, v >> 5] >> (v & 31)) & 1] for t in range(len(X))]
        raw, filt = ro.ranks(self.codes.detach(), self.rel.detach(), X, side, known)
        return torch.as_tensor(raw), None if filt is None else torch.as_tensor(filt)


@pytest.fixture
def oracle_rotate(monkeypatch, oracle_backed_ops):  # noqa: F811
    calls = []

    def fake_sa(codes, rel_table, X, K, alpha, decoder, *, gamma=None):
        calls.append((K, alpha, decoder, gamma))
        return ro.self_adversarial_loss(codes, rel_table, np.asarray(X.cpu()), K, alpha, gamma)
    monkeypatch.setattr(ops, "rotate_score", oracle_rotate_score)
    monkeypatch.setattr(ops, "self_adversarial_loss", fake_sa)
    monkeypatch.setattr(ops, "RotateRanker", OracleRotateRanker)
    return calls


@pytest.mark.parametrize("settings_file", ["complex.exp", "gcn_basis.exp"])
@pytest.mark.parametrize("objective", ["NegativeSampling", "SelfAdversarial"])
def test_host_chain(toy, oracle_rotate, settings_file, objective):
    train = np.asarray(toy["train"], np.int32)
    V, R = int(toy["V"]), int(toy["R"])
    enc, dec = merged_settings(toy, settings_file, V, R, len(train))
    for s in (enc, dec):
        s.put("CodeDimension", "16")
        s.put("InternalEncoderDimension", "16")
    dec.put("Name", "rotate")
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
        assert oracle_rotate == [(K, 1.0, "rotate", 4.0)]
        L, reg, _ = ro.self_adversarial_loss(codes, relt, X, K, 1.0, 4.0)
    else:
        L, reg, _ = ro.ns_loss(codes, relt, X, torch.as_tensor(Y), 4.0)
    param = float(dec["RegularizationParameter"])
    assert abs(total.item() - (L.item() + param * reg.item())) <= 1e-12 * abs(total.item())
    assert all(w.grad is None or torch.isfinite(w.grad).all() for w in ws)
    assert any(w.grad is not None and float(w.grad.abs().max()) > 0 for w in ws)
    # test mode: predict, the score matrices (float32 sigmoid of the energy) and the ranks
    model.preprocess(train)
    model.register_for_test(train)
    test = np.asarray(toy["test"], np.int32)
    p = np.asarray(model.score(test))
    with torch.no_grad():
        codes, relt = [t.detach() for t in model.next_component.get_all_codes(mode='test')[:2]]
        e = ro.energies(codes, relt, test, 4.0)
    np.testing.assert_allclose(p, torch.sigmoid(e).numpy(), rtol=1e-12)
    D1, _, _ = ro.distances(codes, relt, test, 1)
    D0, _, _ = ro.distances(codes, relt, test, 0)
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


def test_no_top_k_relation_prediction_or_fused_ensemble(toy, oracle_rotate):
    enc, dec = _decoder_settings(toy)
    model = model_builder.build_decoder(model_builder.build_encoder(enc, np.array(toy["train"])), dec)
    model.set_device("cpu")
    model.initialize_train()
    model.register_for_test(np.array(toy["train"]))
    tri = np.array(toy["test"])[:3]
    with pytest.raises(NotImplementedError):
        model.predict_top_k(tri, 5, 1)
    with pytest.raises(NotImplementedError):
        model.rank_all_relations(tri, [[]] * 3)
    with pytest.raises(NotImplementedError):
        model.predict_top_k_relations(tri, 5)
    ensemble = ens_mod.Ensemble(model, model, 0.5)
    assert not ensemble.supports_fused_ranking() and ensemble.rank_all_entities(tri, [[]] * 3, [[]] * 3) is None
    with pytest.raises(NotImplementedError, match="fused path"):
        ensemble.predict_top_k(tri, 5, 1)


def test_driver_trains_and_refuses_relation_metrics(toy, tmp_path, capsys, cpu_driver, oracle_rotate):  # noqa: F811
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(TOY_EXP.format(layers=1, concat="No").replace("Name=bilinear-diag", "Name=rotate\n\tMargin=6"))
    np.random.seed(0)
    torch.manual_seed(0)
    driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "40", "--device", "cpu",
                 "--no-save"])
    losses = [float(l.split(":")[-1]) for l in capsys.readouterr().out.splitlines()
              if l.startswith("Average train loss")]
    assert len(losses) == 2 and all(np.isfinite(losses))
    with pytest.raises(SystemExit, match="relation-metrics"):
        driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "40", "--device", "cpu",
                     "--no-save", "--relation-metrics"])
    assert "Initial loss" not in capsys.readouterr().out   # refused before the first iteration


# ---- C-ABI: every bad argument is refused before any device work (fake device pointers are never touched) ----
P = ctypes.c_void_p(256)


def _fwd(**kw):
    a = dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, N=33, Y=P, gamma=12.0, energies=P, loss=P)
    a.update(kw)
    return _lib.load().rgcn_rotate_forward(*a.values(), None)


def _bwd(**kw):
    a = dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, N=33, Y=P, gamma=12.0, energies=P, g_loss=1.0, g_reg=1.0,
             g_scale=None, g_energy=None, dcodes=P, drel=P, ss=None)
    a.update(kw)
    return _lib.load().rgcn_rotate_backward(*a.values(), None)


def _sa(**kw):
    a = dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, N=33, K=10, alpha=1.0, gamma=12.0, energies=P, coef=P, loss=P,
             ws=P, wsb=1 << 40)
    a.update(kw)
    return _lib.load().rgcn_rotate_self_adversarial_forward(*a.values(), None)


def _rank(**kw):
    a = dict(codes=P, rel=P, V=10, Vrel=10, d=8, X=P, n=5, side=1, known=P, raw=P, filt=P, ws=P, wsb=1 << 40)
    a.update(kw)
    return _lib.load().rgcn_rotate_rank(*a.values(), None)


SIZES = [dict(V=0), dict(Vrel=0), dict(d=0), dict(d=6), dict(d=-4), dict(d=10)]
GAMMAS = [dict(gamma=float("inf")), dict(gamma=float("-inf")), dict(gamma=float("nan"))]
INVALID = ([(_fwd, b) for b in SIZES + GAMMAS + [dict(codes=None), dict(rel=None), dict(X=None), dict(energies=None),
                                                   dict(loss=None), dict(N=-1)]] +
           [(_bwd, b) for b in SIZES + GAMMAS + [dict(codes=None), dict(rel=None), dict(X=None), dict(dcodes=None),
                                                   dict(drel=None), dict(energies=None), dict(N=-1)]] +
           [(_sa, b) for b in SIZES + GAMMAS + [dict(codes=None), dict(X=None), dict(coef=None), dict(ws=None),
                                                   dict(N=34), dict(K=0), dict(alpha=-1.0), dict(alpha=float("nan"))]] +
           [(_rank, b) for b in SIZES + [dict(codes=None), dict(rel=None), dict(X=None), dict(raw=None), dict(ws=None),
                                         dict(side=2), dict(side=-1), dict(n=-1), dict(known=None)]])


@pytest.mark.parametrize("fn,bad", INVALID, ids=lambda x: x.__name__ if callable(x) else
                         "-".join("%s=%s" % kv for kv in x.items()))
def test_cabi_rejects_bad_arguments(fn, bad):
    assert fn(**bad) == -1, _lib.load().rgcn_last_error()


def test_cabi_workspace_and_device():
    lib = _lib.load()
    need = lib.rgcn_rotate_rank_workspace_bytes(10, 8, 5)
    assert need >= 5 * 8 * 4 + 4 * 5 * 4
    for bad in ((0, 8, 5), (10, 6, 5), (10, 8, -1)):
        assert lib.rgcn_rotate_rank_workspace_bytes(*bad) == -1
    assert _rank(wsb=need - 1) == -4
    assert _sa(wsb=lib.rgcn_self_adversarial_workspace_bytes(33, 10) - 1) == -4
    if torch.cuda.is_available():
        pytest.skip("a device is present: valid arguments would run")
    assert _fwd() == -5 and _bwd() == -5 and _sa() == -5 and _rank(wsb=need) == -5
