"""CPU: self-adversarial negative sampling -- the float64 oracle and its two identities, the settings keys and every
rejection, the factory rule, the host plugin chain and the training driver with the library call replaced by the
oracle (the substitution lives in this file; the product has no CPU path), and the C-ABI argument checks, which all
return before any device work."""
import ctypes

import numpy as np
import pytest
import torch

import self_adversarial_oracle as so
from relationprediction_b200 import _lib, ops
from relationprediction_b200 import train as driver
from relationprediction_b200.common import model_builder
from relationprediction_b200.decoders.bilinear_diag import parse_adversarial_temperature, parse_training_objective
from test_gpu_train import TOY_EXP, write_toy
from test_plugin_chain_cpu import oracle_backed_ops  # noqa: F401  (fixture)
from test_plugin_host import merged_settings
from test_train_loop_cpu import cpu_driver  # noqa: F401  (fixture)

DT = torch.float64


def layout(rng, V, R, n, K):
    """n positives, then K blocks of their corruptions (subject or object replaced), as the negative sampler lays
    them out"""
    pos = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, V, n)], 1)
    neg = np.tile(pos, (K, 1))
    side = rng.integers(0, 2, n * K) * 2
    neg[np.arange(n * K), side] = rng.integers(0, V, n * K)
    return np.concatenate([pos, neg]).astype(np.int32)


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
def test_oracle_gradcheck(decoder):
    g = torch.Generator().manual_seed(3)
    codes = torch.randn(7, 8, dtype=DT, generator=g, requires_grad=True)
    rel = torch.randn(3, 8, dtype=DT, generator=g, requires_grad=True)
    X = layout(np.random.default_rng(0), 7, 3, 4, 3)
    # p is a constant of the objective: the finite differences hold it at its value at the point checked
    p = so.weights(so.loss(codes, rel, X, 3, 1.3, decoder)[2], 3, 1.3)
    f = lambda c, r: sum(so.loss(c, r, X, 3, 1.3, decoder, p=p)[:2])
    assert torch.autograd.gradcheck(f, (codes, rel))
    # alpha = 0 makes p constant everywhere: the oracle's own weights pass as they are
    assert torch.autograd.gradcheck(lambda c, r: sum(so.loss(c, r, X, 3, 0.0, decoder)[:2]), (codes, rel))


def _sigmoid_ce_mean(e, y):
    return (torch.clamp(e, min=0) - e * y + torch.log1p(torch.exp(-e.abs()))).mean()


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
@pytest.mark.parametrize("alpha", [0.0, 1.0, 5.0])
def test_oracle_k1_is_negative_sampling(decoder, alpha):
    """K = 1: p = 1, so the loss is the mean sigmoid cross-entropy over the 2n triples at any temperature"""
    g = torch.Generator().manual_seed(4)
    codes, rel = torch.randn(9, 8, dtype=DT, generator=g), torch.randn(3, 8, dtype=DT, generator=g)
    X = layout(np.random.default_rng(1), 9, 3, 6, 1)
    L, _, e = so.loss(codes, rel, X, 1, alpha, decoder)
    y = torch.cat([torch.ones(6, dtype=DT), torch.zeros(6, dtype=DT)])
    assert abs(float(L - _sigmoid_ce_mean(e, y))) < 1e-12


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
def test_oracle_alpha0_weights_uniformly(decoder):
    """alpha = 0: p = 1/K"""
    g = torch.Generator().manual_seed(5)
    codes, rel = torch.randn(9, 8, dtype=DT, generator=g), torch.randn(3, 8, dtype=DT, generator=g)
    n, K = 5, 4
    X = layout(np.random.default_rng(2), 9, 3, n, K)
    L, _, e = so.loss(codes, rel, X, K, 0.0, decoder)
    b = e.reshape(K + 1, n)
    want = (so.softplus(-b[0]).sum() + so.softplus(b[1:]).sum() / K) / (2 * n)
    assert abs(float(L - want)) < 1e-12


def test_settings_parsing_and_rejections():
    assert parse_training_objective({'TrainingObjective': 'SelfAdversarial'}) == ('SelfAdversarial', 0.0)
    assert parse_adversarial_temperature({}) == 1.0
    assert parse_adversarial_temperature({'AdversarialTemperature': '0'}) == 0.0
    assert parse_adversarial_temperature({'AdversarialTemperature': '2.5'}) == 2.5
    for alpha in ('-0.5', 'inf', 'nan'):
        with pytest.raises(ValueError, match="AdversarialTemperature"):
            parse_training_objective({'TrainingObjective': 'SelfAdversarial', 'AdversarialTemperature': alpha})
    with pytest.raises(ValueError, match="LabelSmoothing"):
        parse_training_objective({'TrainingObjective': 'SelfAdversarial', 'LabelSmoothing': '0.1'})
    with pytest.raises(ValueError, match="TrainingObjective"):
        parse_training_objective({'TrainingObjective': 'selfadversarial'})


def test_factory_rule_for_other_decoders():
    with pytest.raises(ValueError, match="TrainingObjective=SelfAdversarial"):
        model_builder.build_decoder(None, {'Name': 'nonlinear-transform', 'TrainingObjective': 'SelfAdversarial'})
    assert model_builder.build_decoder(None, {'Name': 'nonlinear-transform'}) is None   # unchanged without the key


def test_ops_rejects_bad_arguments():
    with pytest.raises(ValueError, match="decoder"):
        ops.self_adversarial_loss(None, None, None, 10, 1.0, "transe")
    with pytest.raises(ValueError, match="NegativeSampleRate"):
        ops.self_adversarial_loss(None, None, None, 0, 1.0, "distmult")
    for alpha in (-1.0, float("inf"), float("nan")):
        with pytest.raises(ValueError, match="AdversarialTemperature"):
            ops.self_adversarial_loss(None, None, None, 10, alpha, "distmult")


# ---- the host plugin chain with the library call replaced by the oracle ----
@pytest.fixture
def oracle_self_adversarial(monkeypatch, oracle_backed_ops):  # noqa: F811
    calls = []

    def fake(codes, rel, X, K, alpha, decoder):
        calls.append((np.asarray(X).copy(), K, alpha, decoder))
        return so.loss(codes, rel, np.asarray(X), K, alpha, decoder)
    monkeypatch.setattr(ops, "self_adversarial_loss", fake)
    return calls


def test_host_chain_reads_the_objective(toy, oracle_self_adversarial):
    train = np.asarray(toy["train"], np.int32)
    V, R = int(toy["V"]), int(toy["R"])
    enc, dec = merged_settings(toy, "gcn_basis.exp", V, R, len(train))
    dec.put("TrainingObjective", "SelfAdversarial")
    dec.put("AdversarialTemperature", "0.7")
    model = model_builder.build_decoder(model_builder.build_encoder(enc, train), dec)
    model.set_device("cpu")
    model.initialize_train()
    torch.manual_seed(0)
    ws = model.get_weights()
    for w in ws:
        w.data = torch.randn(w.shape, dtype=DT) * 0.3
    K = int(dec["NegativeSampleRate"])
    X = layout(np.random.default_rng(7), V, R, 9, K)
    y_garbage = np.full(len(X), 7.0, np.float32)   # Y is not read
    torch.manual_seed(1)
    total = model.train_loss(train[:20], X, y_garbage)
    total.backward()
    (fed, k, alpha, decoder), = oracle_self_adversarial
    assert k == K and alpha == 0.7 and decoder == "distmult" and np.array_equal(fed, X)
    L, reg, _ = so.loss(*[t.detach() for t in model.next_component.get_all_codes(mode='train')[:2]], X, K, 0.7,
                        "distmult")
    param = float(dec["RegularizationParameter"])
    assert abs(total.item() - (L.item() + param * reg.item())) <= 1e-12 * abs(total.item())
    assert all(w.grad is None or torch.isfinite(w.grad).all() for w in ws)
    assert any(w.grad is not None and float(w.grad.abs().max()) > 0 for w in ws)
    # test mode is unchanged: scores come from the NegativeSampling scorer (ops.distmult)
    model.preprocess(train)
    model.register_for_test(train)
    assert np.asarray(model.score(train[:5])).shape == (5,)


def test_driver_prints_the_objective(toy, tmp_path, capsys, cpu_driver, oracle_self_adversarial):  # noqa: F811
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(TOY_EXP.format(layers=1, concat="No").replace("[General]\n",
                                                                 "[General]\n\tTrainingObjective=SelfAdversarial\n"))
    np.random.seed(0)
    torch.manual_seed(0)
    driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "40", "--device", "cpu",
                 "--no-save"])
    text = capsys.readouterr().out
    assert "Training objective: SelfAdversarial, temperature 1.0" in text
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 2 and all(np.isfinite(losses))
    assert oracle_self_adversarial and all(k == 10 and a == 1.0 for _, k, a, _ in oracle_self_adversarial)
    assert all(len(x) % 11 == 0 for x, _, _, _ in oracle_self_adversarial)


# ---- C-ABI: every bad argument is refused before any device work (fake device pointers are never touched) ----
P = ctypes.c_void_p(256)


def _args(**kw):
    a = dict(decoder=0, codes=P, rel=P, V=10, Vrel=10, d=8, X=P, N=33, K=10, alpha=1.0, energies=P, coef=P, loss=P,
             ws=P, wsb=1 << 40)
    a.update(kw)
    return a


def _call(a):
    return _lib.load().rgcn_self_adversarial_forward(a["decoder"], a["codes"], a["rel"], a["V"], a["Vrel"], a["d"],
                                                     a["X"], a["N"], a["K"], a["alpha"], a["energies"], a["coef"],
                                                     a["loss"], a["ws"], a["wsb"], None)


INVALID = [
    dict(decoder=2), dict(decoder=-1), dict(codes=None), dict(rel=None), dict(X=None), dict(energies=None),
    dict(coef=None), dict(loss=None), dict(ws=None), dict(V=0), dict(Vrel=0), dict(d=0), dict(d=6), dict(d=-4),
    dict(N=-11), dict(N=34), dict(K=0), dict(K=-1), dict(N=33, K=3), dict(alpha=-0.5), dict(alpha=float("inf")),
    dict(alpha=float("nan")),
]


@pytest.mark.parametrize("decoder", [0, 1])
@pytest.mark.parametrize("bad", INVALID, ids=lambda b: "-".join("%s=%s" % kv for kv in b.items()))
def test_cabi_rejects_bad_arguments(decoder, bad):
    a = _args(decoder=decoder)
    a.update(bad)
    assert _call(a) == -1, _lib.load().rgcn_last_error()


def test_cabi_workspace_and_device():
    lib = _lib.load()
    need = lib.rgcn_self_adversarial_workspace_bytes(33, 10)
    assert need >= 2 * 3 * 4
    assert lib.rgcn_self_adversarial_workspace_bytes(34, 10) == -1
    assert lib.rgcn_self_adversarial_workspace_bytes(33, 0) == -1
    assert lib.rgcn_self_adversarial_workspace_bytes(-11, 10) == -1
    assert _call(_args(wsb=need - 1)) == -4
    if torch.cuda.is_available():
        pytest.skip("a device is present: valid arguments would run")
    assert _call(_args(wsb=need)) == -5
    assert _call(_args(decoder=1, wsb=need)) == -5
