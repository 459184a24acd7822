"""GPU: the QuatE decoder against the float64 oracle of tests/quate_oracle.py -- the scorer and its backward
(max|a - b| / max|b| < 1e-4 for the loss, the L2 term, the energies, dcodes, drel and the relation table's
IndexedSlices norm), a zero relation quaternion, the self-adversarial and 1-N objectives, entity and relation ranks and
top-k (exact on tables whose relation quaternions have power-of-two norms, where every normalised row, query row and
energy is exact in float32), chunked calls, and Toy runs of the driver under each objective, the predict command and
a CompGCN + QuatE chain."""
import json

import numpy as np
import pytest
import torch

import one_to_n_oracle as oo
import quate_oracle as qo
from relationprediction_b200 import ops
from relationprediction_b200 import predict as predict_cmd
from relationprediction_b200 import train as driver
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag
from test_gpu_train import TOY_EXP, write_toy

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4
REG_WEIGHT = 0.3
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


def exact_tables(d, V, R, seed=0, Vrel=None):
    """entity rows with three +-1 entries among the first 8 columns; relation quaternions (+-1, +-1, +-1, +-1) or a
    permutation of (+-2, 0, 0, 0): norm 2, so rh is exact, and so is every query row and energy (|E| <= 6).  Rows
    R..Vrel-1 of the relation table are 2 rel[0]: they would tie with relation 0 if they were ever scored."""
    rng = np.random.default_rng(seed)
    codes = np.zeros((V, d), np.float32)
    cols = np.arange(min(d, 8))
    for v in range(V):
        pick = rng.choice(cols, min(3, len(cols)), replace=False)
        codes[v, pick] = rng.choice([-1.0, 1.0], len(pick))
    relt = np.zeros((Vrel or R, d), np.float32)
    for r in range(R):
        for k in range(d // 4):
            if rng.random() < 0.5:
                relt[r, 4 * k:4 * k + 4] = rng.choice([-1.0, 1.0], 4)
            else:
                relt[r, 4 * k + rng.integers(0, 4)] = rng.choice([-2.0, 2.0])
    relt[R:] = 2 * relt[0]
    return torch.as_tensor(codes), torch.as_tensor(relt)


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
    errs = {"loss": rel(L, L64), "reg": rel(reg, reg64), "energies": rel(e, e64), "dcodes": rel(c.grad, dc64),
            "drel": rel(r.grad, dr64), "slice_norm": rel(r._slice_sumsq, torch.tensor(ss64))}
    del r._slice_sumsq
    assert all(v < TOL for v in errs.values()), errs


@pytest.mark.parametrize("d", [4, 8, 12, 500, 512])
@pytest.mark.parametrize("N,rows", [(333, 50), (5001, 7)])
def test_scorer_and_backward_match_float64(d, N, rows):
    rng = np.random.default_rng(d + N)
    codes, relt = tables(d, rows, 5, seed=d)
    X = layout(rng, rows, 5, N, 0)
    Y = rng.integers(0, 2, N).astype(np.float32)

    def gpu(c, r, Xd):
        e, L, reg = ops.quate_score(c, r, Xd, torch.as_tensor(Y, device=DEV))
        return L, reg, e
    check_step(codes, relt, X, gpu, lambda c, r, rg: qo.ns_loss(c, r, X, torch.as_tensor(Y), rg))


def test_zero_relation_quaternion_has_a_finite_gradient():
    """a zero (and a below-eps) relation quaternion: rh = r / eps, the gradient g / eps, no NaN"""
    codes, relt = tables(8, 6, 2, seed=1)
    relt[0, :4] = 0.0
    relt[1, 4:] = torch.tensor([2e-13, 0.0, -1e-13, 0.0])
    X = np.array([[3, 0, 4], [2, 1, 5]], np.int32)
    Y = np.array([1.0, 0.0], np.float32)

    def gpu(c, r, Xd):
        e, L, reg = ops.quate_score(c, r, Xd, torch.as_tensor(Y, device=DEV))
        return L, reg, e
    c = codes.to(DEV).requires_grad_(True)
    r = relt.to(DEV).requires_grad_(True)
    L, reg, e = gpu(c, r, torch.as_tensor(X, device=DEV))
    (L + REG_WEIGHT * reg).backward()
    assert torch.isfinite(c.grad).all() and torch.isfinite(r.grad).all()
    del r._slice_sumsq
    check_step(codes, relt, X, gpu, lambda c, r, rg: qo.ns_loss(c, r, X, torch.as_tensor(Y), rg))


@pytest.mark.parametrize("d,n,K,alpha", [(8, 64, 1, 1.0), (500, 300, 10, 1.0), (512, 101, 33, 0.5), (4, 7, 256, 2.0)])
def test_self_adversarial_matches_float64(d, n, K, alpha):
    rng = np.random.default_rng(K)
    codes, relt = tables(d, 40, 6, seed=K)
    X = layout(rng, 40, 6, n, K)

    def gpu(c, r, Xd):
        return ops.self_adversarial_loss(c, r, Xd, K, alpha, "quate")
    check_step(codes, relt, X, gpu, lambda c, r, rg: qo.self_adversarial_loss(c, r, X, K, alpha, rg))


@pytest.mark.parametrize("d", [8, 500])
def test_self_adversarial_k1_is_negative_sampling(d):
    rng = np.random.default_rng(3)
    codes, relt = tables(d, 30, 4, seed=3)
    X = layout(rng, 30, 4, 50, 1)
    c, r, Xd = codes.to(DEV), relt.to(DEV), torch.as_tensor(X, device=DEV)
    L, reg, e = ops.self_adversarial_loss(c, r, Xd, 1, 1.0, "quate")
    Y = torch.cat([torch.ones(50), torch.zeros(50)]).to(DEV)
    e_ns, L_ns, reg_ns = ops.quate_score(c, r, Xd, Y)
    assert torch.equal(e, e_ns)
    assert rel(L, L_ns) < 1e-6 and rel(reg, reg_ns) < 1e-6


# ---- 1-N ----
def one_to_n_case(V, d, n, R=5, seed=0):
    g = torch.Generator().manual_seed(seed)
    codes = (torch.randn(V, d, generator=g) * 0.5).float()
    relt = (torch.randn(R + 2, d, generator=g) * 0.5).float()   # rows R.. are never queried
    rng = np.random.default_rng(seed)
    qs = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, 2, n)], 1).astype(np.int32)
    qs = qs[np.lexsort((qs[:, 0], qs[:, 1], qs[:, 2]))]
    y = (rng.random((n, V)) < 0.05).astype(np.float64)
    return codes, relt, qs, y


def run_one_to_n(codes, relt, qs, y, eps, R=5):
    c = codes.to(DEV).requires_grad_(True)
    r = relt.to(DEV).requires_grad_(True)
    loss, reg = ops.one_to_n_loss(c, r, qs, torch.as_tensor(oo.bits(y), device=DEV), eps, "quate", R)
    (loss + REG_WEIGHT * reg).backward()
    return loss.detach(), reg.detach(), c.grad, r.grad


@pytest.mark.parametrize("V,d,n", [(129, 4, 65), (129, 12, 65), (700, 24, 300), (1000, 500, 1000)])
@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_one_to_n_matches_float64(V, d, n, eps, monkeypatch):
    codes, relt, qs, y = one_to_n_case(V, d, n, seed=V + d)
    c = codes.to(DEV).double().requires_grad_(True)
    r = relt.to(DEV).double().requires_grad_(True)
    L, reg = qo.one_to_n_loss(c, r, qs, torch.as_tensor(y, device=DEV), eps)
    (L + REG_WEIGHT * reg).backward()
    whole = run_one_to_n(codes, relt, qs, y, eps)
    for name, a, b in zip(("loss", "reg", "dcodes", "drel"), whole, (L, reg, c.grad, r.grad)):
        assert torch.isfinite(a).all() and rel(a, b) < TOL, (name, rel(a, b))
    monkeypatch.setattr(ops, "ONE_TO_N_CHUNK_BYTES", (V + 4 * d) * 4 * 37)   # 37 queries per pass
    chunked = run_one_to_n(codes, relt, qs, y, eps)
    for a, b in zip(chunked, whole):
        assert rel(a, b) < 1e-5


# ---- entity ranks and top-k ----
def _known(rng, gold, C, extra=3):
    return [sorted({int(g)} | set(rng.integers(0, C, extra).tolist())) for g in gold]


def _excl(rng, n, C, dense_rows=3):
    """random exclusions, plus rows that leave fewer than k (or no) eligible candidates"""
    lists = [sorted(set(rng.integers(0, C, rng.integers(0, 6)).tolist())) for _ in range(n)]
    for t in range(min(dense_rows, n)):
        keep = set(rng.integers(0, C, t).tolist())
        lists[t] = [v for v in range(C) if v not in keep]
    return lists


def test_query_rows_match_float64():
    codes, relt = tables(500, 100, 9, seed=2)
    X = layout(np.random.default_rng(2), 100, 9, 77, 0)
    for side in (0, 1):
        Q = ops.quate_query_rows(codes.to(DEV), relt.to(DEV), torch.as_tensor(X, device=DEV), side)
        assert rel(Q, qo.queries(codes.double(), relt.double(), X, side)[0]) < 1e-6


@pytest.mark.parametrize("V", [1, 127, 128, 129, 300])
@pytest.mark.parametrize("d", [8, 12, 500])
def test_entity_ranks_and_top_k_are_exact(V, d):
    rng = np.random.default_rng(V * d)
    codes, relt = exact_tables(d, V, 7, seed=V + d)
    if V > 10:
        codes[V - 1] = codes[3]            # duplicated rows tie exactly, across tile boundaries
    X = layout(rng, V, 7, 200, 0)
    ranker = ops.QuatERanker(codes.to(DEV), relt.to(DEV))
    Xd = torch.as_tensor(X, device=DEV)
    for side in (0, 1):
        S, Sg, gold = qo.scores(codes, relt, X, side)
        assert float(S.abs().max()) <= 6 and torch.equal(S, S.float().double())
        known = _known(rng, gold.numpy(), V)
        raw, filt = ranker.rank(Xd, side, torch.as_tensor(mask_of(known, V), device=DEV))
        ref_raw, ref_filt = qo.ranks(S, gold, known)
        np.testing.assert_array_equal(raw.cpu().numpy(), ref_raw)
        np.testing.assert_array_equal(filt.cpu().numpy(), ref_filt)
        for k in (1, 10, 128):
            excl = _excl(rng, len(X), V)
            ids, en = ranker.top_k(Xd, side, k, torch.as_tensor(mask_of(excl, V), device=DEV))
            ref_ids, ref_en = qo.top_k(S, k, excl)
            np.testing.assert_array_equal(ids.cpu().numpy(), ref_ids)
            np.testing.assert_array_equal(en.cpu().numpy(), ref_en.astype(np.float32))


@pytest.mark.parametrize("V", [127, 14541])
def test_entity_ranks_match_float64(V):
    d = 500 if V > 1000 else 64
    rng = np.random.default_rng(V)
    codes, relt = tables(d, V, 11, seed=V)
    X = layout(rng, V, 11, 300, 0)
    ranker = ops.QuatERanker(codes.to(DEV), relt.to(DEV))
    for side in (0, 1):
        S, _, gold = qo.scores(codes.to(DEV), relt.to(DEV), X, side)
        known = _known(rng, gold.cpu().numpy(), V)
        raw, filt = ranker.rank(torch.as_tensor(X, device=DEV), side, torch.as_tensor(mask_of(known, V), device=DEV))
        ref_raw, ref_filt = qo.ranks(S, gold, known)
        for got, ref in ((raw, ref_raw), (filt, ref_filt)):
            got = got.cpu().numpy()
            # the gold's score is a float32 dot product, the candidates' the 3xTF32 GEMM's: near-ties may flip
            off = np.abs(got - ref)
            assert (off == 0).mean() >= 0.9 and (off <= 3).mean() >= 0.99, (off.max(), (off > 0).sum())
            assert abs(np.mean(1.0 / got) - np.mean(1.0 / ref)) < 1e-3


# ---- relation queries ----
@pytest.mark.parametrize("R", [1, 31, 32, 33, 237])
def test_relation_ranks_and_top_k_are_exact(R):
    rng = np.random.default_rng(R)
    V, d = 300, 12
    codes, relt = exact_tables(d, V, R, seed=R, Vrel=V)    # the [V, d] relation table of the R-GCN encoders
    if R > 2:
        relt[R - 1] = relt[0]
    X = layout(rng, V, R, 150, 0)
    ranker = ops.QuatERanker(codes.to(DEV), relt.to(DEV), R)
    Xd = torch.as_tensor(X, device=DEV)
    S, Sg, gold = qo.scores(codes, relt, X, "relation", R)
    assert float(S.abs().max()) <= 6 and torch.equal(S, S.float().double())
    known = _known(rng, gold.numpy(), R, 2)
    raw, filt = ranker.rank_relations(Xd, torch.as_tensor(mask_of(known, R), device=DEV))
    ref_raw, ref_filt = qo.ranks(S, gold, known)
    np.testing.assert_array_equal(raw.cpu().numpy(), ref_raw)
    np.testing.assert_array_equal(filt.cpu().numpy(), ref_filt)
    for k in (1, 10, 128):
        for excl in (None, _excl(rng, len(X), R)):
            ids, en = ranker.top_k_relations(Xd, k, None if excl is None else torch.as_tensor(mask_of(excl, R),
                                                                                             device=DEV))
            ref_ids, ref_en = qo.top_k(S, k, excl)
            np.testing.assert_array_equal(ids.cpu().numpy(), ref_ids)
            np.testing.assert_array_equal(en.cpu().numpy(), ref_en.astype(np.float32))


def test_relation_ranks_match_float64():
    rng = np.random.default_rng(9)
    V, R = 400, 237
    codes, relt = tables(500, V, V, seed=9)
    X = layout(rng, V, R, 300, 0)
    ranker = ops.QuatERanker(codes.to(DEV), relt.to(DEV), R)
    S, _, gold = qo.scores(codes.to(DEV), relt.to(DEV), X, "relation", R)
    raw, _ = ranker.rank_relations(torch.as_tensor(X, device=DEV))
    ref_raw, _ = qo.ranks(S, gold)
    got = raw.cpu().numpy()
    assert (got == ref_raw).mean() >= 0.97 and abs(np.mean(1.0 / got) - np.mean(1.0 / ref_raw)) < 1e-3


def test_chunked_calls_equal_one_call(monkeypatch):
    rng = np.random.default_rng(5)
    V, R = 400, 40
    codes, relt = tables(64, V, V, seed=5)
    X = torch.as_tensor(layout(rng, V, R, 500, 0), device=DEV)
    em = torch.as_tensor(mask_of(_excl(rng, 500, V), V), device=DEV)
    rm = torch.as_tensor(mask_of(_excl(rng, 500, R), R), device=DEV)

    def run():
        ranker = ops.QuatERanker(codes.to(DEV), relt.to(DEV), R)
        out = [ranker.top_k(X, 1, 10, em), ranker.rank_relations(X, rm), ranker.top_k_relations(X, 7, rm),
               ranker.rank_relations(X, rm)]
        return [t for r in out for t in r]
    whole = run()
    monkeypatch.setattr(ops.QuatERanker, "TOPK_CHUNK_BYTES", 64 * 1024)
    chunked = run()
    assert all(torch.equal(a, b) for a, b in zip(whole, chunked))


# ---- end to end on Toy ----
def _toy_exp(toy, tmp_path, objective="NegativeSampling", encoder=None):
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    text = TOY_EXP.format(layers=1, concat="No").replace(
        "Name=bilinear-diag", "Name=quate\n\tTrainingObjective=%s" % objective)
    if encoder:
        text = text.replace("Name=gcn_basis", encoder)
    exp.write_text(text)
    return exp


@pytest.mark.parametrize("objective", ["NegativeSampling", "SelfAdversarial", "1-N"])
def test_toy_training_with_relation_metrics(toy, tmp_path, capsys, objective):
    exp = _toy_exp(toy, tmp_path, objective)
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--no-save", "--no-early-stopping", "--final-eval", "0", "--relation-metrics"])
    out = capsys.readouterr().out
    losses = [float(l.split(":")[-1]) for l in out.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and all(np.isfinite(losses)) and losses[-1] < losses[0]
    assert "Relation prediction:" in out
    line = json.loads([l for l in out.splitlines() if l.startswith("{")][-1])
    assert 0.0 < line["relation"]["filtered"]["MRR"] <= 1.0 and 0.0 < line["filtered"]["MRR"] <= 1.0
    # the Scorer's fused ranks against float64 ranks of the test codes
    test = np.array(toy["test"])
    fused = scorer.compute_scores(test)
    model._feed_test(getattr(model, "test_graph", None), test[:1])
    with torch.no_grad():
        codes, relt = [t.detach() for t in model.next_component.get_all_codes(mode='test')[:2]]
    raw = [qo.ranks(*qo.scores(codes, relt, test, side)[::2])[0] for side in (0, 1)]
    assert (np.array(fused.raw_ranks) == np.concatenate(raw)).mean() >= 0.97


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
    # the relation queries answer with relation names, the object queries agree with the Scorer's fused top-k
    assert all(r[2] in rl.values() for r in rows if int(r[0]) % 3 == 0)
    ids, _, _ = scorer.predict_top_k(tri, k, 1, filtered=True)
    obj = [(int(a), int(b), c) for a, b, c, _ in rows if int(a) % 3 == 1]
    assert obj == [(3 * j + 1, p + 1, ent[int(ids[j, p])]) for j in range(len(tri)) for p in range(k) if ids[j, p] >= 0]


def test_compgcn_quate_chain_trains_and_evaluates(toy, tmp_path, capsys):
    exp = _toy_exp(toy, tmp_path, "1-N", "Name=compgcn\n\tComposition=mult")
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--no-save", "--no-early-stopping", "--final-eval", "0", "--relation-metrics"])
    out = capsys.readouterr().out
    losses = [float(l.split(":")[-1]) for l in out.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and all(np.isfinite(losses))
    line = json.loads([l for l in out.splitlines() if l.startswith("{")][-1])
    assert 0.0 < line["filtered"]["MRR"] <= 1.0 and 0.0 < line["relation"]["filtered"]["MRR"] <= 1.0
    assert type(model).__name__ == "QuatE"
