"""GPU: the RotatE decoder against the float64 oracle of tests/rotate_oracle.py -- the scorer and its backward
(max|a - b| / max|b| < 1e-4 for the loss, the L2 term, the energies, dcodes, drel and the relation table's
IndexedSlices norm), the self-adversarial objective, the all-entity ranks by distance, the model and Scorer end to end,
and Toy training runs of the driver under both objectives."""
import json

import numpy as np
import pytest
import torch

import rotate_oracle as ro
from relationprediction_b200 import ops
from relationprediction_b200 import train as driver
from relationprediction_b200.common import evaluation, model_builder
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag
from test_gpu_train import TOY_EXP, write_toy
from test_plugin_host import merged_settings

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4
REG_WEIGHT = 0.3
GAMMA = 12.0


def rel(a, b):
    a, b = torch.as_tensor(a).detach(), torch.as_tensor(b).detach()
    return float((a.double() - b.double().to(a.device)).abs().max() / max(float(b.double().abs().max()), 1e-30))


@pytest.fixture(autouse=True)
def slice_norms():
    ops.set_slice_norms(True)
    yield
    ops.set_slice_norms(False)


def layout(rng, V, R, n, K):
    """n positives, then K blocks of their corruptions, as the negative sampler lays them out"""
    pos = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, V, n)], 1)
    neg = np.tile(pos, (K, 1))
    side = rng.integers(0, 2, n * K) * 2
    neg[np.arange(n * K), side] = rng.integers(0, V, n * K)
    return np.concatenate([pos, neg]).astype(np.int32)


def tables(d, V, R, seed=0, scale=0.5, phase=np.pi):
    """codes N(0, scale^2) [V, d]; relation rows [R, d] with phases uniform in [-phase, phase] in the first d/2 columns
    and noise in the unread rest"""
    g = torch.Generator().manual_seed(seed)
    codes = (torch.randn(V, d, generator=g) * scale).float()
    relt = torch.randn(R, d, generator=g).float()
    relt[:, :d // 2] = ((torch.rand(R, d // 2, generator=g) * 2 - 1) * phase).float()
    return codes, relt


def run_ns(codes, relt, X, Y, gamma=GAMMA):
    c = codes.to(DEV).requires_grad_(True)
    r = relt.to(DEV).requires_grad_(True)
    e, loss, reg = ops.rotate_score(c, r, torch.as_tensor(X, device=DEV), torch.as_tensor(Y, device=DEV), gamma=gamma)
    (loss + REG_WEIGHT * reg).backward()
    return loss.detach(), reg.detach(), e.detach(), c.grad, r.grad, r._slice_sumsq


def oracle(codes, relt, X, loss_fn):
    """loss_fn(codes64, rel64, gathered_rel) -> (loss, reg, energies); the per-triple relation slices are the gradient
    of the gathered rows"""
    c = codes.to(DEV).double().requires_grad_(True)
    r = relt.to(DEV).double()
    rows = torch.as_tensor(X[:, 1].astype(np.int64), device=DEV)
    b = r[rows].requires_grad_(True)
    loss, reg, e = loss_fn(c, r, b)
    (loss + REG_WEIGHT * reg).backward()
    drel = torch.zeros_like(r).index_add_(0, rows, b.grad)
    return loss.detach(), reg.detach(), e.detach(), c.grad, drel, (b.grad ** 2).sum()


NAMES = ("loss", "reg", "energies", "dcodes", "drel", "rel_slice_sumsq")


def check(got, ref, tol=TOL):
    for name, a, b in zip(NAMES, got, ref):
        assert torch.isfinite(a).all(), name
        assert rel(a, b) < tol, (name, rel(a, b))


# each axis against a base case: d (both W paths), N, relation table height (Vrel = V or R), phase range
SCORER_CASES = sorted(set([(d, 33, "R", np.pi) for d in (4, 8, 12, 500, 512)] +
                          [(500, N, "R", np.pi) for N in (1, 31, 32, 33, 30000)] +
                          [(d, 33, "V", np.pi) for d in (12, 512)] +
                          [(d, 1000, "R", 1e3) for d in (8, 500)]))


@pytest.mark.parametrize("d,N,rows,phase", SCORER_CASES)
def test_scorer_and_backward_match_float64(d, N, rows, phase):
    V = 300
    R = V if rows == "V" else (237 if N > 10000 else 7)
    codes, relt = tables(d, V, R, seed=d + N, phase=phase)
    rng = np.random.default_rng(N)
    X = np.stack([rng.integers(0, V, N), rng.integers(0, R, N), rng.integers(0, V, N)], 1).astype(np.int32)
    Y = rng.integers(0, 2, N).astype(np.float32)
    got = run_ns(codes, relt, X, Y)
    ref = oracle(codes, relt, X, lambda c, r, b: ro.ns_loss(c, r, X, torch.as_tensor(Y), GAMMA, gathered_rel=b))
    check(got, ref)
    # the second half of every relation row is never read and gets no gradient
    assert float(got[4][:, d // 2:].abs().max()) == 0.0


def test_exact_zero_residual_takes_the_zero_subgradient():
    """theta = 0 and s = o: u = 0 in every column, E = gamma exactly, and only the L2 term moves the entity rows.
    gamma = 1 keeps sigmoid(E) - y away from the float32 cancellation of a saturated sigmoid"""
    d, V, R, gamma = 8, 5, 2, 1.0
    codes, relt = tables(d, V, R, seed=3)
    relt[0, :d // 2] = 0.0
    X = np.array([[1, 0, 1], [2, 0, 2], [3, 1, 4]], np.int32)
    Y = np.array([1.0, 0.0, 1.0], np.float32)
    got = run_ns(codes, relt, X, Y, gamma=gamma)
    ref = oracle(codes, relt, X, lambda c, r, b: ro.ns_loss(c, r, X, torch.as_tensor(Y), gamma, gathered_rel=b))
    check(got, ref)
    assert float(got[2][0]) == gamma and float(got[2][1]) == gamma
    c_reg = REG_WEIGHT * 2.0 / (3 * d)
    for v in (1, 2):   # each row appears twice (as a and as c) in one triple
        assert rel(got[3][v], 2 * c_reg * codes[v].to(DEV)) < 1e-6
    assert float(got[4][0].abs().max()) == 0.0


# ---- self-adversarial ----
def run_sa(codes, relt, X, K, alpha, gamma=GAMMA):
    c = codes.to(DEV).requires_grad_(True)
    r = relt.to(DEV).requires_grad_(True)
    loss, reg, e = ops.self_adversarial_loss(c, r, torch.as_tensor(X, device=DEV), K, alpha, "rotate", gamma=gamma)
    (loss + REG_WEIGHT * reg).backward()
    return loss.detach(), reg.detach(), e.detach(), c.grad, r.grad, r._slice_sumsq


@pytest.mark.parametrize("d,n,K,alpha", [(4, 33, 10, 1.0), (500, 33, 10, 0.7), (512, 31, 33, 5.0), (500, 3000, 10, 1.0),
                                         (12, 32, 256, 0.0)])
def test_self_adversarial_matches_float64(d, n, K, alpha):
    codes, relt = tables(d, 300, 7, seed=d + n + K)
    X = layout(np.random.default_rng(K), 300, 7, n, K)
    got = run_sa(codes, relt, X, K, alpha)
    ref = oracle(codes, relt, X, lambda c, r, b: ro.self_adversarial_loss(c, r, X, K, alpha, GAMMA, gathered_rel=b))
    check(got, ref)


def test_self_adversarial_alpha0_weights_uniformly():
    d, n, K = 500, 40, 6
    codes, relt = tables(d, 200, 7, seed=5)
    X = layout(np.random.default_rng(5), 200, 7, n, K)
    loss = run_sa(codes, relt, X, K, 0.0)[0]
    e = ro.energies(codes.to(DEV).double(), relt.to(DEV).double(), X, GAMMA).reshape(K + 1, n)
    from self_adversarial_oracle import softplus
    want = (softplus(-e[0]).sum() + softplus(e[1:]).sum() / K) / (2 * n)
    assert rel(loss, want) < TOL


@pytest.mark.parametrize("d", [8, 500, 512])
def test_self_adversarial_k1_is_negative_sampling(d):
    """K = 1: p = 1, so the loss, the L2 term, the energies and every gradient are the NegativeSampling scorer's with
    Y = 1 for the positives and 0 for the corruptions; the energies come from the same row arithmetic, bit for bit"""
    n = 2000
    codes, relt = tables(d, 300, 237, seed=d, scale=0.1)
    X = layout(np.random.default_rng(d), 300, 237, n, 1)
    Y = np.concatenate([np.ones(n), np.zeros(n)]).astype(np.float32)
    want = run_ns(codes, relt, X, Y, gamma=1.0)
    for alpha in (0.0, 1.0, 5.0):
        got = run_sa(codes, relt, X, 1, alpha, gamma=1.0)
        assert torch.equal(got[2], want[2])
        for name, a, b in zip(NAMES, got, want):
            # the slice sum (float atomics over warps) and the L2 term (the NegativeSampling forward adds its per-block
            # sums by float atomics) differ by their summation order, not by the objective
            assert rel(a, b) < (1e-5 if name in ("rel_slice_sumsq", "reg") else 1e-6), (alpha, name, rel(a, b))


# ---- all-entity ranking by distance ----
def ranker_ranks(codes, relt, X, side, known_lists=None):
    r = ops.RotateRanker(codes.to(DEV), relt.to(DEV))
    mask = None
    if known_lists is not None:
        mask = torch.as_tensor(BilinearDiag.known_bit_mask(known_lists, codes.shape[0]), device=DEV)
    raw, filt = r.rank(torch.as_tensor(X, device=DEV), side, mask)
    return raw.cpu().numpy(), None if filt is None else filt.cpu().numpy()


def queries(rng, V, R, n):
    return np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, V, n)], 1).astype(np.int32)


@pytest.mark.parametrize("V", [1, 127, 128, 129, 14541])
@pytest.mark.parametrize("d", [500, 512])
def test_ranks_match_float64(V, d):
    codes, relt = tables(d, V, 237, seed=V + d, scale=1.0)
    rng = np.random.default_rng(V)
    for n, side in ((1, 0), (129, 1), (300, 0), (300, 1)):
        X = queries(rng, V, 237, n)
        known = [sorted(set(rng.integers(0, V, 5).tolist()) | {int(x[2 if side else 0])}) for x in X]
        raw, filt = ranker_ranks(codes, relt, X, side, known)
        D, Dg, gold = ro.distances(codes.to(DEV), relt.to(DEV), X, side)
        want_raw, want_filt = ro.ranks(codes.to(DEV), relt.to(DEV), X, side, known)
        assert (raw >= 1).all() and (filt >= 1).all() and (raw <= V).all()
        same = raw == want_raw
        assert same.mean() >= 0.97
        mrr, want_mrr = np.mean(1.0 / raw), np.mean(1.0 / want_raw)
        assert abs(mrr - want_mrr) < 1e-4
        # a rank may differ only by candidates whose float64 distance agrees with the gold's to 1e-5 relative
        close = (((D - Dg[:, None]).abs() <= 1e-5 * Dg[:, None]).sum(1) - 1).cpu().numpy()
        assert (np.abs(raw - want_raw) <= close).all()
        unambiguous = close == 0
        assert (raw[unambiguous] == want_raw[unambiguous]).all()
        assert (filt[unambiguous] == want_filt[unambiguous]).all()


def test_duplicated_rows_tie_and_the_gold_counts():
    """copies of entity rows appended to the table count exactly where their originals count: for every query, the
    rank grows by the number of copied originals with D <= D_gold (read off the filtered rank with those originals as
    the known set), the gold's own copies included -- which holds only if a copy ties with the gold bit for bit"""
    d, V = 500, 1000
    codes, relt = tables(d, V, 20, seed=9, scale=1.0)
    rng = np.random.default_rng(9)
    for side in (0, 1):
        X = queries(rng, V, 20, 400)
        gold = X[:, 0] if side == 0 else X[:, 2]
        dup = np.unique(gold)[:50]
        once = [dup.tolist()] * len(X)
        twice = [dup[:10].tolist()] * len(X)
        base, f_once = ranker_ranks(codes, relt, X, side, once)
        _, f_twice = ranker_ranks(codes, relt, X, side, twice)
        counted = (base - f_once + 1) + (base - f_twice + 1)
        raw, _ = ranker_ranks(torch.cat([codes, codes[dup], codes[dup[:10]]]), relt, X, side)
        np.testing.assert_array_equal(raw - base, counted)
        assert (counted[np.isin(gold, dup)] >= 1).all()
    one, _ = ranker_ranks(codes[:1], relt, np.array([[0, 3, 0]] * 5, np.int32), 1)
    assert (one == 1).all()


def test_filtered_counts_are_exact_on_constructed_masks():
    d, V, n = 512, 700, 256
    codes, relt = tables(d, V, 9, seed=11, scale=1.0)
    X = queries(np.random.default_rng(11), V, 9, n)
    for side in (0, 1):
        raw, none = ranker_ranks(codes, relt, X, side, [[] for _ in range(n)])
        np.testing.assert_array_equal(none, raw + 1)
        _, everything = ranker_ranks(codes, relt, X, side, [list(range(V))] * n)
        assert (everything == 1).all()
        gold = X[:, 0] if side == 0 else X[:, 2]
        _, only_gold = ranker_ranks(codes, relt, X, side, [[int(g)] for g in gold])
        np.testing.assert_array_equal(only_gold, raw)


def test_ranks_need_no_margin_and_match_the_score_matrices(toy):
    """through the factory, the model and the Scorer: the fused ranks equal the float64 oracle's on codes small enough
    for the float32 sigmoid not to saturate, equal the score-matrix path's, and do not change with Margin"""
    V, R = int(toy["V"]), int(toy["R"])
    train = np.asarray(toy["train"], np.int32)
    results = []
    for margin in ("0", "12"):
        enc, dec = merged_settings(toy, "complex.exp", V, R, len(train))
        for s in (enc, dec):
            s.put("CodeDimension", "16")
        dec.put("Name", "rotate")
        dec.put("Margin", margin)
        model = model_builder.build_decoder(model_builder.build_encoder(enc, train), dec)
        model.set_device(DEV)
        model.initialize_train()
        torch.manual_seed(0)
        for w in model.get_weights():
            w.data = (torch.randn(w.shape) * 0.3).to(DEV)
        model.preprocess(train)
        model.register_for_test(train)
        sc = evaluation.Scorer({'Metric': 'MRR'})
        for part in (toy["train"], toy["valid"], toy["test"]):
            sc.register_data(np.asarray(part))
        sc.register_model(model)
        test = np.asarray(toy["test"], np.int32)
        fused = sc.compute_scores(test)
        model.supports_fused_ranking = lambda: False
        matrices = sc.compute_scores(test)
        assert fused.raw_ranks == matrices.raw_ranks and fused.filtered_ranks == matrices.filtered_ranks
        codes = model.next_component.get_all_codes(mode='test')[0].detach()
        relt = model.next_component.get_all_codes(mode='test')[1].detach()
        want = np.concatenate([ro.ranks(codes, relt, test, 0)[0], ro.ranks(codes, relt, test, 1)[0]])
        np.testing.assert_array_equal(np.asarray(fused.raw_ranks), want)
        results.append((fused.raw_ranks, fused.filtered_ranks))
    assert results[0] == results[1]


# ---- the driver on Toy ----
ROTATE_EXP = TOY_EXP.replace("Name=bilinear-diag", "Name=rotate\n\tMargin=6")


@pytest.mark.parametrize("objective", ["NegativeSampling", "SelfAdversarial"])
def test_toy_training(toy, tmp_path, capsys, objective):
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(ROTATE_EXP.format(layers=1, concat="No").replace(
        "[General]\n", "[General]\n\tTrainingObjective=%s\n" % objective))
    np.random.seed(0)
    torch.manual_seed(0)
    ckpt = tmp_path / "ckpt" / "Toy"
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "300",
                                 "--save-path", str(ckpt), "--final-eval", "0"])
    text = capsys.readouterr().out
    assert "Initial loss" in text and "Validation filtered MRR" in text
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) >= 4 and all(np.isfinite(losses)) and losses[-1] < losses[0]
    line = json.loads(text.strip().splitlines()[-1])
    assert line["test_triples"] == len(toy["test"]) and 0.0 < line["filtered"]["MRR"] <= 1.0
    assert list((tmp_path / "ckpt").glob("Toy-*.pt"))
    saved = [w.detach().clone() for w in model.get_weights()]
    before = scorer.compute_scores(np.array(toy["train"])[:20]).get_summary().results["Filtered"]["MRR"]
    model.save(str(tmp_path / "rt"))
    for w in model.get_weights():
        w.data.zero_()
    model.load("%s-%d.pt" % (tmp_path / "rt", model.save_iter - 1))
    assert all(torch.equal(a, w.detach()) for a, w in zip(saved, model.get_weights()))
    after = scorer.compute_scores(np.array(toy["train"])[:20]).get_summary().results["Filtered"]["MRR"]
    assert after == before
