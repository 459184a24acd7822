"""GPU: self-adversarial negative sampling (ops.self_adversarial_loss) against the float64 oracle of
tests/self_adversarial_oracle.py, at max|a - b| / max|b| < 1e-4 for the loss, the L2 term, the energies, dcodes, drel and
the relation table's IndexedSlices norm; the K = 1 identity against the NegativeSampling scorers; bitwise repeatability;
and a Toy training run of the driver."""
import numpy as np
import pytest
import torch

import self_adversarial_oracle as so
from relationprediction_b200 import ops
from relationprediction_b200 import train as driver
from test_gpu_train import TOY_EXP, write_toy

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4
REG_WEIGHT = 0.3
SCORERS = {"distmult": ops.distmult, "complex": ops.complex_score}


def rel(a, b):
    a, b = a.detach(), b.detach()
    return float((a.double() - b.double()).abs().max() / max(float(b.double().abs().max()), 1e-30))


@pytest.fixture(autouse=True)
def slice_norms():
    ops.set_slice_norms(True)
    yield
    ops.set_slice_norms(False)


def layout(rng, V, R, n, K):
    """n positives, then K blocks of their corruptions (subject or object replaced), as the negative sampler lays
    them out; a small V makes duplicate corruptions common"""
    pos = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, V, n)], 1)
    neg = np.tile(pos, (K, 1))
    side = rng.integers(0, 2, n * K) * 2
    neg[np.arange(n * K), side] = rng.integers(0, V, n * K)
    return np.concatenate([pos, neg]).astype(np.int32)


def case(d, n, K, V=300, R=7, seed=0, scale=0.5):
    g = torch.Generator().manual_seed(seed)
    codes = (torch.randn(V, d, generator=g) * scale).float()
    relt = (torch.randn(R, d, generator=g) * scale).float()
    return codes, relt, layout(np.random.default_rng(seed), V, R, n, K)


def run(codes, relt, X, K, alpha, decoder):
    c = codes.to(DEV).requires_grad_(True)
    r = relt.to(DEV).requires_grad_(True)
    loss, reg, e = ops.self_adversarial_loss(c, r, torch.as_tensor(X, device=DEV), K, alpha, decoder)
    (loss + REG_WEIGHT * reg).backward()
    return loss.detach(), reg.detach(), e.detach(), c.grad, r.grad, r._slice_sumsq


def oracle(codes, relt, X, K, alpha, decoder):
    c = codes.to(DEV).double().requires_grad_(True)
    r = relt.to(DEV).double()
    rows = torch.as_tensor(X[:, 1].astype(np.int64), device=DEV)
    b = r[rows].requires_grad_(True)   # the gathered relation rows: their gradients are the per-triple slices
    loss, reg, e = so.loss(c, r, X, K, alpha, decoder, gathered_rel=b)
    (loss + REG_WEIGHT * reg).backward()
    drel = torch.zeros_like(r).index_add_(0, rows, b.grad)
    return loss.detach(), reg.detach(), e.detach(), c.grad, drel, (b.grad ** 2).sum()


NAMES = ("loss", "reg", "energies", "dcodes", "drel", "rel_slice_sumsq")


def check(codes, relt, X, K, alpha, decoder):
    got = run(codes, relt, X, K, alpha, decoder)
    ref = oracle(codes, relt, X, K, alpha, decoder)
    for name, a, b in zip(NAMES, got, ref):
        assert torch.isfinite(a).all(), name
        assert rel(a, b) < TOL, (name, rel(a, b))
    return got


# each axis of the issue's grid against a base case, and the two corners that stress the group loop
CASES = sorted(set([(d, 33, 10, 1.0) for d in (4, 200, 500, 512, 516)] +
                   [(200, n, 10, 1.0) for n in (1, 31, 32, 33, 5000)] +
                   [(500, 33, K, 1.0) for K in (1, 2, 10, 33, 256)] +
                   [(516, 31, 33, a) for a in (0.0, 1.0, 5.0)] +
                   [(512, 32, 256, 0.0), (4, 5000, 256, 5.0), (500, 5000, 10, 5.0)]))


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
@pytest.mark.parametrize("d,n,K,alpha", CASES)
def test_matches_float64(decoder, d, n, K, alpha):
    # above 100 000 triples, FB15k-237's 237 relations: with 7 the float32 scatter of the relation gradient would add
    # some 180 000 signed terms into each row, and its rounding, not the objective, would set the error
    codes, relt, X = case(d, n, K, R=237 if n * (K + 1) > 100000 else 7)
    check(codes, relt, X, K, alpha, decoder)


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
@pytest.mark.parametrize("alpha", [0.0, 1.0, 5.0])
def test_saturated_energies_and_duplicate_corruptions(decoder, alpha):
    """groups whose energies are +-1e4 (every lane's loss and gradient stays finite), and groups whose corruptions
    are all one triple (p = 1/K at any temperature)"""
    d, V, n, K = 4, 8, 6, 5
    codes = torch.randn(V, d, generator=torch.Generator().manual_seed(1)) * 0.5
    codes[0], codes[1] = 100.0, -100.0
    relt = torch.randn(3, d, generator=torch.Generator().manual_seed(2)) * 0.5
    relt[0] = 0.25
    if decoder == "complex":   # [real | imaginary] rows: real parts only, so the energies are again +-1e4
        codes[0], codes[1], relt[0] = torch.tensor([100.0, 100.0, 0.0, 0.0]), torch.tensor([-100.0, -100.0, 0.0, 0.0]), \
            torch.tensor([0.5, 0.5, 0.0, 0.0])
    pos = np.array([[0, 0, 0], [0, 0, 1], [1, 0, 0], [2, 1, 3], [4, 2, 5], [0, 0, 0]])
    negs = []
    for j in range(K):
        neg = pos.copy()
        neg[0] = (0, 0, 1) if j % 2 else (0, 0, 0)     # +1e4 and -1e4 corruptions
        neg[1] = (1, 0, 1)                             # +1e4, the same triple K times
        neg[2] = (0, 0, j % 3)                         # +1e4 / -1e4 / small
        neg[3] = (2, 1, 6)                             # duplicates of a small-energy triple
        neg[4, 2] = j                                  # distinct corruptions
        negs.append(neg)
    X = np.concatenate([pos] + negs).astype(np.int32)
    got = check(codes, relt, X, K, alpha, decoder)
    assert abs(float(got[2].abs().max()) - 1e4) < 1.0


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
@pytest.mark.parametrize("d", [8, 500, 516])
def test_k1_is_negative_sampling(decoder, d):
    """K = 1: p = 1, so the loss, the L2 term, the energies and every gradient are those of the NegativeSampling scorer
    with Y = 1 for the positives and 0 for the corruptions, at any temperature"""
    n = 2000
    # 237 relations: a relation row then takes some 17 float32 atomic adds per element, whose order varies from call to
    # call, and that noise stays well below the 1e-6 the two objectives are held to.  Moderate energies: the
    # NegativeSampling backward forms a positive's gradient as sigmoid(s) - 1, which loses digits at large s, where this
    # objective's -sigmoid(-s) does not
    codes, relt, X = case(d, n, 1, R=237, scale=0.25)
    Y = torch.cat([torch.ones(n), torch.zeros(n)]).to(DEV)
    Xd = torch.as_tensor(X, device=DEV)
    c, r = codes.to(DEV).requires_grad_(True), relt.to(DEV).requires_grad_(True)
    e, loss, reg = SCORERS[decoder](c, r, Xd, Y)
    (loss + REG_WEIGHT * reg).backward()
    want = (loss.detach(), reg.detach(), e.detach(), c.grad, r.grad, r._slice_sumsq)
    for alpha in (0.0, 1.0, 5.0):
        got = run(codes, relt, X, 1, alpha, decoder)
        assert torch.equal(got[2], want[2])   # the same row arithmetic
        for name, a, b in zip(NAMES, got, want):
            # the slice sum is a float atomic sum over warps of squares: its order, not the objective, differs
            assert rel(a, b) < (1e-5 if name == "rel_slice_sumsq" else 1e-6), (alpha, name, rel(a, b))


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
def test_loss_is_bitwise_repeatable(decoder):
    codes, relt, X = case(500, 3000, 10)
    c, r, Xd = codes.to(DEV), relt.to(DEV), torch.as_tensor(X, device=DEV)
    a = ops.self_adversarial_loss(c, r, Xd, 10, 1.0, decoder)
    b = ops.self_adversarial_loss(c, r, Xd, 10, 1.0, decoder)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
def test_upstream_gradients_scale_the_two_terms(decoder):
    codes, relt, X = case(24, 90, 4)
    c, r = codes.to(DEV).requires_grad_(True), relt.to(DEV).requires_grad_(True)
    loss, reg, _ = ops.self_adversarial_loss(c, r, torch.as_tensor(X, device=DEV), 4, 2.0, decoder)
    c64, r64 = codes.to(DEV).double().requires_grad_(True), relt.to(DEV).double().requires_grad_(True)
    L, Rg, _ = so.loss(c64, r64, X, 4, 2.0, decoder)
    for g0, g1 in ((2.5, 0.0), (0.0, 1.7), (-0.4, 3.0)):
        got = torch.autograd.grad(g0 * loss + g1 * reg, [c, r], retain_graph=True)
        want = torch.autograd.grad(g0 * L + g1 * Rg, [c64, r64], retain_graph=True)
        for a, b in zip(got, want):
            assert rel(a, b) < TOL, (g0, g1)


SA_EXP = TOY_EXP.replace("[General]\n", "[General]\n\tTrainingObjective=SelfAdversarial\n")


@pytest.mark.parametrize("decoder", ["bilinear-diag", "complex"])
def test_toy_training_self_adversarial(toy, tmp_path, capsys, decoder):
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(SA_EXP.format(layers=1, concat="No").replace("Name=bilinear-diag", "Name=" + decoder))
    np.random.seed(0)
    torch.manual_seed(0)
    ckpt = tmp_path / "ckpt" / "Toy"
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "300",
                                 "--save-path", str(ckpt)])
    text = capsys.readouterr().out
    assert "Training objective: SelfAdversarial, temperature 1.0" in text
    assert "Initial loss" in text and "Validation filtered MRR" in text
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) >= 4 and all(np.isfinite(losses)) and losses[-1] < losses[0]
    assert list((tmp_path / "ckpt").glob("Toy-*.pt"))
    saved = [w.detach().clone() for w in model.get_weights()]
    before = scorer.compute_scores(np.array(toy["train"])[:20]).get_summary().results["Filtered"]["MRR"]
    model.save(str(tmp_path / "rt"))
    for w in model.get_weights():
        w.data.zero_()
    model.load("%s-%d.pt" % (tmp_path / "rt", model.save_iter - 1))
    assert all(torch.equal(a, w.detach()) for a, w in zip(saved, model.get_weights()))
    after = scorer.compute_scores(np.array(toy["train"])[:20]).get_summary().results["Filtered"]["MRR"]
    assert 0.0 < after <= 1.0 and abs(after - before) < 1e-3
