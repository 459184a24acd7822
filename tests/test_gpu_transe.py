"""GPU: the TransE decoder against the float64 oracle of tests/transe_oracle.py -- the scorer and its backward
(max|a - b| / max|b| < 1e-4 for the loss, the L2 term, the energies, dcodes, drel and the relation table's
IndexedSlices norm), the self-adversarial objective, entity and relation ranks and top-k by L1 distance (exact on
small-integer tables, where every distance is exact), chunked calls, and Toy runs of the driver, the predict command
and a CompGCN + TransE chain."""
import json

import numpy as np
import pytest
import torch

import transe_oracle as to
from relationprediction_b200 import ops
from relationprediction_b200 import predict as predict_cmd
from relationprediction_b200 import train as driver
from relationprediction_b200.common import evaluation, model_builder
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag
from test_gpu_train import TOY_EXP, write_toy

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4
REG_WEIGHT = 0.3
GAMMA = 12.0
mask_of = BilinearDiag.known_bit_mask


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


def tables(d, V, R, seed=0, scale=0.5):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(V, d, generator=g) * scale).float(), (torch.randn(R, d, generator=g) * scale).float()


def int_tables(d, V, R, seed=0, lo=-3, hi=4):
    """small-integer tables: every sum of the distance is exact in float32"""
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(lo, hi, (V, d), generator=g).float(), torch.randint(lo, hi, (R, d), generator=g).float())


def with_zero_residuals(codes, relt, X):
    """relation row 0 is zero and every triple of relation 0 has s == o; integer columns 0..d/4-1 of the other rows
    are translations of each other, so many residual columns are exactly 0"""
    codes, relt = codes.clone(), relt.clone()
    relt[0] = 0.0
    q = codes.shape[1] // 4
    codes[:, :q] = codes[:, :q].round()
    relt[:, :q] = relt[:, :q].round()
    for s, r, o in X[::3]:
        codes[o, :q] = codes[s, :q] + relt[r, :q]
    X = X.copy()
    X[X[:, 1] == 0, 2] = X[X[:, 1] == 0, 0]
    return codes, relt, X


def float64_grads(codes, relt, X, loss_fn):
    c = codes.double().requires_grad_(True)
    r = relt.double().requires_grad_(True)
    rg = r[torch.as_tensor(X[:, 1].astype(np.int64))].detach().requires_grad_(True)
    L, reg, e = loss_fn(c, r, rg)
    (L + REG_WEIGHT * reg).backward()
    drel = torch.zeros_like(r).index_add_(0, torch.as_tensor(X[:, 1].astype(np.int64)), rg.grad)
    return L, reg, e, c.grad, drel, float((rg.grad ** 2).sum())


def check_step(codes, relt, X, gpu_fn, loss_fn):
    c = codes.to(DEV).requires_grad_(True)
    r = relt.to(DEV).requires_grad_(True)
    L, reg, e = gpu_fn(c, r, torch.as_tensor(X, device=DEV))
    (L + REG_WEIGHT * reg).backward()
    L64, reg64, e64, dc64, dr64, ss64 = float64_grads(codes, relt, X, loss_fn)
    assert rel(L, L64) < TOL and rel(reg, reg64) < TOL and rel(e, e64) < TOL
    assert rel(c.grad, dc64) < TOL and rel(r.grad, dr64) < TOL
    assert rel(r._slice_sumsq, torch.tensor(ss64)) < TOL
    del r._slice_sumsq


@pytest.mark.parametrize("d", [4, 8, 500, 512])
@pytest.mark.parametrize("N,rows", [(333, 50), (5000, 7)])
def test_scorer_and_backward_match_float64(d, N, rows):
    rng = np.random.default_rng(d + N)
    codes, relt = tables(d, rows, 5, seed=d)
    X = layout(rng, rows, 5, N, 0)
    codes, relt, X = with_zero_residuals(codes, relt, X)
    Y = rng.integers(0, 2, N).astype(np.float32)

    def gpu(c, r, Xd):
        e, L, reg = ops.transe_score(c, r, Xd, torch.as_tensor(Y, device=DEV), gamma=GAMMA)
        return L, reg, e
    check_step(codes, relt, X, gpu, lambda c, r, rg: to.ns_loss(c, r, X, torch.as_tensor(Y), GAMMA, rg))


def test_exact_zero_residual_takes_the_zero_subgradient():
    codes, relt = int_tables(8, 6, 2, seed=1)
    relt[0] = 0.0
    X = np.array([[3, 0, 3]], np.int32)
    c = codes.to(DEV).requires_grad_(True)
    r = relt.to(DEV).requires_grad_(True)
    e, L, reg = ops.transe_score(c, r, torch.as_tensor(X, device=DEV), torch.ones(1, device=DEV), gamma=5.0)
    assert float(e[0]) == 5.0
    L.backward()   # the loss alone: nothing reaches the rows through u = 0
    assert float(c.grad.abs().max()) == 0.0 and float(r.grad.abs().max()) == 0.0


@pytest.mark.parametrize("d,n,K,alpha", [(8, 64, 1, 1.0), (500, 300, 10, 1.0), (512, 100, 33, 0.5), (4, 7, 256, 2.0)])
def test_self_adversarial_matches_float64(d, n, K, alpha):
    rng = np.random.default_rng(K)
    codes, relt = tables(d, 40, 6, seed=K)
    X = layout(rng, 40, 6, n, K)

    def gpu(c, r, Xd):
        return ops.self_adversarial_loss(c, r, Xd, K, alpha, "transe", gamma=GAMMA)
    check_step(codes, relt, X, gpu, lambda c, r, rg: to.self_adversarial_loss(c, r, X, K, alpha, GAMMA, rg))


@pytest.mark.parametrize("d", [8, 500])
def test_self_adversarial_k1_is_negative_sampling(d):
    rng = np.random.default_rng(3)
    codes, relt = tables(d, 30, 4, seed=3)
    X = layout(rng, 30, 4, 50, 1)
    c, r, Xd = codes.to(DEV), relt.to(DEV), torch.as_tensor(X, device=DEV)
    L, reg, e = ops.self_adversarial_loss(c, r, Xd, 1, 1.0, "transe", gamma=GAMMA)
    Y = torch.cat([torch.ones(50), torch.zeros(50)]).to(DEV)
    e_ns, L_ns, reg_ns = ops.transe_score(c, r, Xd, Y, gamma=GAMMA)
    assert torch.equal(e, e_ns)
    assert rel(L, L_ns) < 1e-6 and rel(reg, reg_ns) < 1e-6


# ---- entity ranks ----
def _known(rng, X, side, C, extra=3):
    gold = X[:, 0] if side == 0 else X[:, 2]
    return [sorted({int(g)} | set(rng.integers(0, C, extra).tolist())) for g in gold]


@pytest.mark.parametrize("V", [1, 127, 128, 129, 14541])
def test_entity_ranks_match_float64(V):
    d = 500 if V == 14541 else 64
    rng = np.random.default_rng(V)
    codes, relt = tables(d, V, 11, seed=V)
    X = layout(rng, V, 11, 300, 0)
    ranker = ops.TransERanker(codes.to(DEV), relt.to(DEV), gamma=GAMMA)
    for side in (0, 1):
        known = _known(rng, X, side, V)
        raw, filt = ranker.rank(torch.as_tensor(X, device=DEV), side,
                                torch.as_tensor(mask_of(known, V), device=DEV))
        ref_raw, ref_filt = to.ranks(codes.to(DEV), relt.to(DEV), X, side, known)
        for got, ref in ((raw, ref_raw), (filt, ref_filt)):
            got = got.cpu().numpy()
            assert (got == ref).mean() >= 0.97
            assert abs(np.mean(1.0 / got) - np.mean(1.0 / ref)) < 1e-4


@pytest.mark.parametrize("V", [1, 127, 128, 129, 300])
def test_entity_ranks_are_exact_on_integer_tables(V):
    rng = np.random.default_rng(V + 1)
    codes, relt = int_tables(24, V, 7, seed=V)
    if V > 10:
        codes[V // 2] = codes[3]            # duplicated rows tie exactly
    X = layout(rng, V, 7, 200, 0)
    if V > 10:
        X[:20, 2] = 3
        X[20:40, 0] = V // 2
    ranker = ops.TransERanker(codes.to(DEV), relt.to(DEV))
    for side in (0, 1):
        known = _known(rng, X, side, V)
        raw, filt = ranker.rank(torch.as_tensor(X, device=DEV), side,
                                torch.as_tensor(mask_of(known, V), device=DEV))
        ref_raw, ref_filt = to.ranks(codes, relt, X, side, known)
        np.testing.assert_array_equal(raw.cpu().numpy(), ref_raw)
        np.testing.assert_array_equal(filt.cpu().numpy(), ref_filt)
        assert (raw.cpu().numpy() >= 1).all()    # the gold counts itself


# ---- top-k ----
def _excl(rng, n, C, dense_rows=3):
    """random exclusions, plus rows that leave fewer than k (or no) eligible candidates"""
    lists = [sorted(set(rng.integers(0, C, rng.integers(0, 6)).tolist())) for _ in range(n)]
    for t in range(min(dense_rows, n)):
        keep = set(rng.integers(0, C, t).tolist())
        lists[t] = [v for v in range(C) if v not in keep]
    return lists


def check_top_k(ids, en, D, k, gamma, excl, exact):
    ids, en = ids.cpu().numpy(), en.cpu().numpy()
    ref_ids, ref_en = to.top_k(D, k, gamma, excl)
    if exact:
        np.testing.assert_array_equal(ids, ref_ids)
        np.testing.assert_array_equal(en, ref_en.astype(np.float32))
        return
    assert ((ids < 0) == (ref_ids < 0)).all()
    ok = ref_ids >= 0
    np.testing.assert_allclose(en[ok], ref_en[ok], rtol=1e-4, atol=1e-4 * np.abs(ref_en[ok]).max())
    D = np.asarray(D.cpu(), np.float64)
    rows = np.nonzero(ok)[0]
    got_D, ref_D = D[rows, ids[ok]], D[rows, ref_ids[ok]]
    swapped = ids[ok] != ref_ids[ok]
    assert (np.abs(got_D - ref_D)[swapped] <= 1e-5 * np.abs(ref_D[swapped])).all()
    for t in range(len(ids)):
        assert not set(ids[t][ids[t] >= 0].tolist()) & set(excl[t])


@pytest.mark.parametrize("V", [127, 128, 129, 257])
@pytest.mark.parametrize("k", [1, 10, 128])
@pytest.mark.parametrize("integer", [True, False])
def test_entity_top_k(V, k, integer):
    rng = np.random.default_rng(V * k)
    codes, relt = int_tables(16, V, 5, seed=V) if integer else tables(64, V, 5, seed=V)
    if integer:
        codes[V - 1] = codes[0]             # ties across tile boundaries go to the smaller id
        codes[128 % V] = codes[1]
    X = layout(rng, V, 5, 70, 0)
    ranker = ops.TransERanker(codes.to(DEV), relt.to(DEV), gamma=GAMMA)
    for side in (0, 1):
        excl = _excl(rng, len(X), V)
        ids, en = ranker.top_k(torch.as_tensor(X, device=DEV), side, k, torch.as_tensor(mask_of(excl, V), device=DEV))
        D = to.distances(codes, relt, X, side)[0]
        check_top_k(ids, en, D, k, GAMMA, excl, integer)
        ids, en = ranker.top_k(torch.as_tensor(X, device=DEV), side, k)   # no mask
        check_top_k(ids, en, D, k, GAMMA, [[]] * len(X), integer)


# ---- relation queries ----
@pytest.mark.parametrize("R", [1, 31, 32, 33, 237])
def test_relation_ranks_and_top_k(R):
    rng = np.random.default_rng(R)
    V = 300
    for integer in (True, False):
        codes, relt = int_tables(24, V, V, seed=R) if integer else tables(64, V, V, seed=R)
        if integer and R > 2:
            relt[R - 1] = relt[0]
        X = layout(rng, V, R, 150, 0)
        ranker = ops.TransERanker(codes.to(DEV), relt.to(DEV), R, gamma=GAMMA)   # the [V, d] relation table
        Xd = torch.as_tensor(X, device=DEV)
        known = [sorted({int(r)} | set(rng.integers(0, R, 2).tolist())) for r in X[:, 1]]
        raw, filt = ranker.rank_relations(Xd, torch.as_tensor(mask_of(known, R), device=DEV))
        ref_raw, ref_filt = to.ranks(codes, relt, X, "relation", known, R)
        for got, ref in ((raw, ref_raw), (filt, ref_filt)):
            got = got.cpu().numpy()
            if integer:
                np.testing.assert_array_equal(got, ref)
            else:
                assert (got == ref).mean() >= 0.97 and abs(np.mean(1.0 / got) - np.mean(1.0 / ref)) < 1e-4
        D = to.distances(codes, relt, X, "relation", R)[0]
        for k in (1, 10, 128):
            excl = _excl(rng, len(X), R)
            ids, en = ranker.top_k_relations(Xd, k, torch.as_tensor(mask_of(excl, R), device=DEV))
            check_top_k(ids, en, D, k, GAMMA, excl, integer)


def test_chunked_calls_equal_one_call(monkeypatch):
    rng = np.random.default_rng(5)
    V, R = 400, 40
    codes, relt = tables(64, V, V, seed=5)
    X = torch.as_tensor(layout(rng, V, R, 500, 0), device=DEV)
    em = torch.as_tensor(mask_of(_excl(rng, 500, V), V), device=DEV)
    rm = torch.as_tensor(mask_of(_excl(rng, 500, R), R), device=DEV)

    def run():
        ranker = ops.TransERanker(codes.to(DEV), relt.to(DEV), R, gamma=GAMMA)
        return [t for r in (ranker.rank(X, 0, em), ranker.top_k(X, 1, 10, em), ranker.rank_relations(X, rm),
                            ranker.top_k_relations(X, 7, rm)) for t in r]
    whole = run()
    monkeypatch.setattr(ops.TransERanker, "TOPK_CHUNK_BYTES", 64 * 1024)
    chunked = run()
    assert all(torch.equal(a, b) for a, b in zip(whole, chunked))


# ---- end to end on Toy ----
def _toy_exp(toy, tmp_path, objective="NegativeSampling", encoder=None):
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    text = TOY_EXP.format(layers=1, concat="No").replace(
        "Name=bilinear-diag", "Name=transe\n\tMargin=6\n\tTrainingObjective=%s" % objective)
    if encoder:
        text = text.replace("Name=gcn_basis", encoder)
    exp.write_text(text)
    return exp


@pytest.mark.parametrize("objective", ["NegativeSampling", "SelfAdversarial"])
def test_toy_training_with_relation_metrics(toy, tmp_path, capsys, objective):
    exp = _toy_exp(toy, tmp_path, objective)
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--no-save", "--no-early-stopping", "--final-eval", "0", "--relation-metrics"])
    out = capsys.readouterr().out
    losses = [float(l.split(":")[-1]) for l in out.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and all(np.isfinite(losses))
    assert "Relation prediction:" in out
    table = out.split("Relation prediction:")[1].strip().splitlines()[:5]
    assert table[0].split() == ["Raw", "Filtered"]
    line = json.loads([l for l in out.splitlines() if l.startswith("{")][-1])
    assert 0.0 < line["relation"]["filtered"]["MRR"] <= 1.0 and 0.0 < line["filtered"]["MRR"] <= 1.0
    # the Scorer's fused ranks against float64 ranks of the test codes
    test = np.array(toy["test"])
    fused = scorer.compute_scores(test)
    model._feed_test(getattr(model, "test_graph", None), test[:1])
    with torch.no_grad():
        codes, relt = [t.detach() for t in model.next_component.get_all_codes(mode='test')[:2]]
    raw = [to.ranks(codes, relt, test, side)[0] for side in (0, 1)]
    got = np.array(fused.raw_ranks)
    assert (got == np.concatenate(raw)).mean() >= 0.97


def test_predict_command_answers_entity_and_relation_queries(toy, tmp_path, capsys):
    exp = _toy_exp(toy, tmp_path)
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "40",
                                 "--no-save", "--no-early-stopping"])
    model.save(str(tmp_path / "Toy"))
    ckpt = sorted(tmp_path.glob("Toy-*.pt"))[-1]
    ent = {int(k): v for k, v in toy["entities"].items()}
    rl = {int(k): v for k, v in toy["relations"].items()}
    tri = np.array(toy["test"])[:8]
    lines = []
    for s_, r_, o_ in tri.tolist():
        lines += ["%s\t?\t%s" % (ent[s_], ent[o_]), "%s\t%s\t?" % (ent[s_], rl[r_]), "?\t%s\t%s" % (rl[r_], ent[o_])]
    (tmp_path / "queries.tsv").write_text("\n".join(lines) + "\n")
    out = tmp_path / "answers.tsv"
    R = int(model.relation_count)
    k = min(4, R)
    predict_cmd.main(["--settings", str(exp), "--dataset", str(tmp_path), "--checkpoint", str(ckpt),
                      "--queries", str(tmp_path / "queries.tsv"), "--k", str(k), "--out", str(out)])
    rows = [l.split("\t") for l in out.read_text().splitlines()]
    assert {int(r[0]) for r in rows} == set(range(len(lines)))
    for q in range(len(lines)):
        got = [r for r in rows if int(r[0]) == q]
        assert [int(r[1]) for r in got] == list(range(1, len(got) + 1)) and 0 < len(got) <= k
        scores = [float(r[3]) for r in got]
        assert scores == sorted(scores, reverse=True) and all(0.0 <= s <= 1.0 for s in scores)
    # the object queries agree with the Scorer's fused top-k
    ids, _, _ = scorer.predict_top_k(tri, k, 1, filtered=True)
    obj = [(int(a), int(b), c) for a, b, c, _ in rows if int(a) % 3 == 1]
    assert obj == [(3 * j + 1, p + 1, ent[int(ids[j, p])]) for j in range(len(tri)) for p in range(k) if ids[j, p] >= 0]


def test_compgcn_transe_chain_trains_and_evaluates(toy, tmp_path, capsys):
    exp = _toy_exp(toy, tmp_path, "SelfAdversarial", "Name=compgcn\n\tComposition=sub")
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--no-save", "--no-early-stopping", "--final-eval", "0", "--relation-metrics"])
    out = capsys.readouterr().out
    losses = [float(l.split(":")[-1]) for l in out.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and all(np.isfinite(losses))
    line = json.loads([l for l in out.splitlines() if l.startswith("{")][-1])
    assert 0.0 < line["filtered"]["MRR"] <= 1.0 and 0.0 < line["relation"]["filtered"]["MRR"] <= 1.0
    assert type(model).__name__ == "TransE"
