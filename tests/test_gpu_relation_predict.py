"""GPU: fused relation prediction (distmult_relation_rank / _topk and the ComplEx twins: the pair-query prepare
kernels, the entity-side scoring GEMM run over the first R relation rows with its rank or top-k epilogue) against a
float64 restatement -- ranks raw and filtered, top-k ids and energies with the smaller id first on ties, rows
R..Vrel-1 never counted or returned -- and the whole chain up to Scorer, the predict command and train.py."""
import json

import numpy as np
import pytest
import torch

from relationprediction_b200 import _lib, ops
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag
from test_gpu_topk import reference_topk

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RANKERS = {"distmult": ops.DistMultRanker, "complex": ops.ComplexRanker}
HUGE = 1.0e6


def pair_queries64(codes, X, decoder):
    """float64 query rows of (h, ?, t): DistMult codes[h] * codes[t]; ComplEx [hr tr + hi ti, hr ti - hi tr]."""
    c = codes.astype(np.float64)
    a, b = c[X[:, 0]], c[X[:, 2]]
    if decoder == "distmult":
        return a * b
    h = c.shape[1] // 2
    ar, ai, br, bi = a[:, :h], a[:, h:], b[:, :h], b[:, h:]
    return np.concatenate([ar * br + ai * bi, ar * bi - ai * br], 1)


def energies64(codes, rel, R, X, decoder):
    return pair_queries64(codes, X, decoder) @ rel[:R].astype(np.float64).T


def reference_ranks(e, gold, known):
    """raw = #{r : e_r >= e_gold}, filtered = raw - #{known r : e_r >= e_gold} + 1 (energy order; the callers keep
    |e| <= 16, where the float32 sigmoid is strictly increasing on the integers)."""
    g = e[np.arange(len(e)), gold][:, None]
    ge = e >= g
    raw = ge.sum(1)
    kn = np.array([int(ge[i, np.asarray(l, dtype=np.int64)].sum()) for i, l in enumerate(known)])
    return raw, raw - kn + 1


def integer_problem(rng, V, R, d, n):
    """Entity codes with three +-1 entries among six shared columns (|energy| <= 9 for both decoders, exact in fp32
    and in the 3xTF32 GEMM, many exact ties), +-1/0 relation rows with two duplicated rows, and HUGE rows R..R+6
    that must never be counted or returned."""
    cols = rng.choice(d, min(d, 6), replace=False)
    codes = np.zeros((V, d), np.float32)
    for v in range(V):
        pick = rng.choice(cols, min(3, len(cols)), replace=False)
        codes[v, pick] = rng.choice([-1.0, 1.0], len(pick))
    rel = rng.randint(-1, 2, (R + 7, d)).astype(np.float32)
    if R >= 3:
        rel[R - 1] = rel[0]
        rel[R // 2] = rel[1]
    rel[R:] = HUGE
    X = np.stack([rng.randint(0, V, n), rng.randint(0, R, n), rng.randint(0, V, n)], 1).astype(np.int32)
    return codes, rel, X


def random_known(rng, X, R):
    return [sorted(set(rng.randint(0, R, rng.randint(0, R // 3 + 2)).tolist()) | {int(g)}) for g in X[:, 1]]


def mask_of(lists, R):
    return torch.as_tensor(BilinearDiag.known_bit_mask(lists, R), device=DEV)


def chunk_bytes(R, d, k, rows):
    """TOPK_CHUNK_BYTES that puts about `rows` queries in one library call of either relation path"""
    lib = _lib.load()
    rank = lib.rgcn_relation_rank_workspace_bytes(R, d, 1) - lib.rgcn_relation_rank_workspace_bytes(R, d, 0)
    topk = lib.rgcn_relation_topk_workspace_bytes(R, d, 1, k) - lib.rgcn_relation_topk_workspace_bytes(R, d, 0, k)
    return rows * max(rank, topk)


def run_rank(ranker, X, known):
    raw, filt = ranker.rank_relations(torch.as_tensor(X, device=DEV), None if known is None else mask_of(
        known, ranker.relation_count))
    return raw.cpu().numpy(), None if filt is None else filt.cpu().numpy()


def run_topk(ranker, X, k, excl):
    ids, en = ranker.top_k_relations(torch.as_tensor(X, device=DEV), k, None if excl is None else mask_of(
        excl, ranker.relation_count))
    return ids.cpu().numpy().astype(np.int64), en.cpu().numpy()


@pytest.mark.parametrize("decoder", sorted(RANKERS))
@pytest.mark.parametrize("d", [8, 12, 500])
@pytest.mark.parametrize("R", [1, 31, 33, 129, 237, 1345])
def test_integer_codes_give_exact_ranks_and_order_with_ties(decoder, R, d):
    """Every energy is exact, so ties are real: raw ranks count every tied relation, top-k puts the smaller id first.
    n = 300 spans three 128-row M tiles; the chunked ranker makes several library calls per path."""
    rng = np.random.RandomState(R * 7 + d)
    V, n = 300, 300
    codes, rel, X = integer_problem(rng, V, R, d, n)
    e = energies64(codes, rel, R, X, decoder)
    assert np.abs(e).max() <= 16
    if R >= 3:
        np.testing.assert_array_equal(e[:, 0], e[:, R - 1])           # duplicated rows score alike
    ct, rt = torch.as_tensor(codes, device=DEV), torch.as_tensor(rel, device=DEV)
    ranker = RANKERS[decoder](ct, rt, R)
    chunked = RANKERS[decoder](ct, rt, R)
    chunked.TOPK_CHUNK_BYTES = chunk_bytes(R, d, 128, 100)
    known = random_known(rng, X, R)
    ref_raw, ref_filt = reference_ranks(e, X[:, 1], known)
    for rk in (ranker, chunked):
        raw, filt = run_rank(rk, X, known)
        np.testing.assert_array_equal(raw, ref_raw)
        np.testing.assert_array_equal(filt, ref_filt)
        raw_only, none = run_rank(rk, X, None)
        assert none is None
        np.testing.assert_array_equal(raw_only, ref_raw)
    for k in (1, 10, 128):
        for excl in (None, known):
            ref_ids, ref_en = reference_topk(e, k, excl)
            for rk in (ranker, chunked):
                ids, en = run_topk(rk, X, k, excl)
                np.testing.assert_array_equal(ids, ref_ids)
                np.testing.assert_array_equal(en, ref_en)
                assert ids.max() < R


@pytest.mark.parametrize("decoder", sorted(RANKERS))
@pytest.mark.parametrize("R,d", [(237, 500), (1345, 200), (33, 12)])
def test_float_codes_match_float64_up_to_near_ties(decoder, R, d):
    rng = np.random.RandomState(R + d)
    V, n, k = 2000, 1500, 10
    codes = rng.normal(0, 0.3, (V, d)).astype(np.float32)
    rel = rng.normal(0, 1, (R + 50, d)).astype(np.float32)
    rel[R:] = HUGE
    X = np.stack([rng.randint(0, V, n), rng.randint(0, R, n), rng.randint(0, V, n)], 1).astype(np.int32)
    ranker = RANKERS[decoder](torch.as_tensor(codes, device=DEV), torch.as_tensor(rel, device=DEV), R)
    e = energies64(codes, rel, R, X, decoder)
    known = random_known(rng, X, R)
    s = 1.0 / (1.0 + np.exp(-e))
    ref_raw, ref_filt = reference_ranks(s, X[:, 1], known)
    raw, filt = run_rank(ranker, X, known)
    for got, ref in ((raw, ref_raw), (filt, ref_filt)):
        diff = np.abs(got - ref)
        # fp32 rounding may swap relations whose scores agree to ~1e-7 or saturate together; nothing else may move
        assert (diff == 0).mean() > 0.97 and diff.max() <= max(3, 0.002 * R), (diff.mean(), diff.max())
        assert abs(np.mean(1.0 / got) - np.mean(1.0 / ref)) < 1e-3
    for excl in (None, known):
        ids, en = run_topk(ranker, X, k, excl)
        ref_ids, ref_en = reference_topk(e, k, excl)
        valid = ref_ids >= 0
        np.testing.assert_array_equal(ids >= 0, valid)
        got64 = np.take_along_axis(e, np.maximum(ids, 0), 1)
        assert (np.abs(en - got64) <= 1e-4 * np.abs(got64) + 1e-6)[valid].all()
        swapped = (ids != ref_ids) & valid
        scale = np.abs(ref_en).astype(np.float64) + 1e-30
        assert (np.abs(got64 - ref_en.astype(np.float64))[swapped] <= 1e-5 * scale[swapped]).all()
        assert swapped.mean() < 0.01


@pytest.mark.parametrize("decoder", sorted(RANKERS))
def test_exclusion_pads_and_an_all_excluded_row_returns_only_padding(decoder):
    rng = np.random.RandomState(3)
    R, d, n = 40, 16, 60
    codes, rel, X = integer_problem(rng, 100, R, d, n)
    ranker = RANKERS[decoder](torch.as_tensor(codes, device=DEV), torch.as_tensor(rel, device=DEV), R)
    keep = [sorted(rng.choice(R, i % 6, replace=False).tolist()) for i in range(n)]   # 0..5 eligible, row 0 none
    excl = [sorted(set(range(R)) - set(kp)) for kp in keep]
    e = energies64(codes, rel, R, X, decoder)
    for k in (10, 128):
        ids, en = run_topk(ranker, X, k, excl)
        ref_ids, ref_en = reference_topk(e, k, excl)
        np.testing.assert_array_equal(ids, ref_ids)
        np.testing.assert_array_equal(en, ref_en)
        for t, kp in enumerate(keep):
            assert sorted(ids[t, :len(kp)].tolist()) == kp
            assert (ids[t, len(kp):] == -1).all() and np.isneginf(en[t, len(kp):]).all()
    # k larger than R: the tail past the R relations is padding
    ids, en = run_topk(ranker, X, 100, None)
    assert (ids[:, :R] >= 0).all() and (ids[:, R:] == -1).all() and np.isneginf(en[:, R:]).all()


@pytest.mark.parametrize("decoder", sorted(RANKERS))
def test_entity_and_relation_splits_never_mix(decoder):
    """One ranker serves entity and relation queries from two workspaces: alternating the four paths (in both
    orders, with the relation workspace regrown in between) gives what fresh rankers give."""
    rng = np.random.RandomState(11)
    V, R, d, n, k = 700, 237, 64, 500, 10
    codes = rng.normal(0, 0.3, (V, d)).astype(np.float32)
    rel = rng.normal(0, 1, (V, d)).astype(np.float32)                  # an R-GCN style [V, d] relation table
    X = np.stack([rng.randint(0, V, n), rng.randint(0, R, n), rng.randint(0, V, n)], 1).astype(np.int32)
    Xt = torch.as_tensor(X, device=DEV)
    ct, rt = torch.as_tensor(codes, device=DEV), torch.as_tensor(rel, device=DEV)
    ent_known = [[int(o)] for o in X[:, 2]]
    rel_known = random_known(rng, X, R)
    make = lambda: RANKERS[decoder](ct, rt, R)
    paths = {
        "rank": lambda rk: rk.rank(Xt, 1, torch.as_tensor(BilinearDiag.known_bit_mask(ent_known, V), device=DEV)),
        "rank_relations": lambda rk: rk.rank_relations(Xt, mask_of(rel_known, R)),
        "top_k": lambda rk: rk.top_k(Xt, 0, k, None),
        "top_k_relations": lambda rk: rk.top_k_relations(Xt, k, mask_of(rel_known, R)),
        "top_k_relations_128": lambda rk: rk.top_k_relations(Xt, 128, None),
    }
    fresh = {name: [t.cpu().numpy() for t in fn(make())] for name, fn in paths.items()}
    shared = make()
    for order in (list(paths), list(reversed(list(paths))), ["rank_relations", "top_k", "top_k_relations_128",
                                                             "rank", "top_k_relations", "rank_relations"]):
        for name in order:
            got = [t.cpu().numpy() for t in paths[name](shared)]
            for a, b in zip(got, fresh[name]):
                assert a.tobytes() == b.tobytes(), name


@pytest.mark.parametrize("decoder", sorted(RANKERS))
@pytest.mark.parametrize("d", [500, 16])
def test_pair_query_energy_equals_the_decoders_own_energy(decoder, d):
    """Q . rel[r] (the energies top_k_relations returns for k >= R) equals the decoder's scorer energy of (h, r, t)
    for every r: the ComplEx query formula follows the code's real / imaginary layout and sign convention."""
    rng = np.random.RandomState(d)
    V, R, n = 300, 100, 50
    codes = rng.normal(0, 0.3, (V, d)).astype(np.float32)
    rel = rng.normal(0, 1, (V, d)).astype(np.float32)
    X = np.stack([rng.randint(0, V, n), np.zeros(n, np.int64), rng.randint(0, V, n)], 1).astype(np.int32)
    ct, rt = torch.as_tensor(codes, device=DEV), torch.as_tensor(rel, device=DEV)
    ids, en = run_topk(RANKERS[decoder](ct, rt, R), X, 128, None)
    assert (ids[:, :R] >= 0).all() and (ids[:, R:] == -1).all()
    fused = np.zeros((n, R), np.float64)
    np.put_along_axis(fused, ids[:, :R], en[:, :R].astype(np.float64), 1)
    full = np.repeat(X, R, 0)
    full[:, 1] = np.tile(np.arange(R), n)
    score_op = ops.distmult if decoder == "distmult" else ops.complex_score
    own = score_op(ct, rt, torch.as_tensor(full, device=DEV), None)[0].cpu().numpy().reshape(n, R)
    assert np.abs(fused - own).max() <= 1e-5 * max(1.0, np.abs(own).max())


def _trained(toy, tmp_path, decoder):
    from test_gpu_topk import _trained_toy
    return _trained_toy(toy, tmp_path, decoder)


def _all_relation_scores(model, pairs, R):
    full = np.repeat(pairs, R, 0)
    full[:, 1] = np.tile(np.arange(R), len(pairs))
    return model.score(full).astype(np.float64).reshape(len(pairs), R)


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
def test_predict_command_and_relation_metrics_on_toy(toy, tmp_path, decoder):
    from relationprediction_b200 import predict as predict_cmd
    exp, model, scorer = _trained(toy, tmp_path, decoder)
    R = int(model.relation_count)
    test = np.array(toy["test"])
    # Scorer.compute_relation_mrr_scores against ranks recomputed in float64 from Model.score over all r
    score = scorer.compute_relation_mrr_scores(test)
    s = _all_relation_scores(model, test, R)
    known = [scorer.known_relation_triples[(t[0], t[2])] for t in test.tolist()]
    ref_raw, ref_filt = reference_ranks(s, test[:, 1], known)
    for got, ref in ((np.array(score.raw_ranks), ref_raw), (np.array(score.filtered_ranks), ref_filt)):
        assert len(got) == len(test)
        diff = np.abs(got - ref)
        assert (diff == 0).mean() > 0.95 and diff.max() <= 2, (diff.mean(), diff.max())
        assert abs(np.mean(1.0 / got) - np.mean(1.0 / ref)) < 1e-2
    # the predict command on relation queries (with entity queries between them) against the argsort of Model.score
    model.save(str(tmp_path / "Toy"))
    ckpt = sorted(tmp_path.glob("Toy-*.pt"))[-1]
    ent = {int(k): v for k, v in toy["entities"].items()}
    rel = {int(k): v for k, v in toy["relations"].items()}
    tri = test[:10]
    lines = []
    for s_, r_, o_ in tri.tolist():
        lines += ["%s\t?\t%s" % (ent[s_], ent[o_]), "%s\t%s\t?" % (ent[s_], rel[r_])]
    (tmp_path / "queries.tsv").write_text("\n".join(lines) + "\n")
    out = tmp_path / "answers.tsv"
    k = min(5, R)
    predict_cmd.main(["--settings", str(exp), "--dataset", str(tmp_path), "--checkpoint", str(ckpt),
                      "--queries", str(tmp_path / "queries.tsv"), "--k", str(k), "--out", str(out)])
    rows = [l.split("\t") for l in out.read_text().splitlines()]
    pair_scores = _all_relation_scores(model, tri, R)
    name_to_rel = {v: i for i, v in rel.items()}
    for j, (s_, r_, o_) in enumerate(tri.tolist()):
        got = [r for r in rows if int(r[0]) == 2 * j]
        excl = scorer.known_relation_triples.get((s_, o_), [])
        ok = np.ones(R, bool)
        ok[excl] = False
        cand = np.nonzero(ok)[0]
        ref = cand[np.lexsort((cand, -pair_scores[j, cand]))][:k]
        assert [int(r[1]) for r in got] == list(range(1, len(ref) + 1))
        got_ids = np.array([name_to_rel[r[2]] for r in got], np.int64)
        assert not set(got_ids.tolist()) & set(excl)
        # the model's scores are float32 sigmoids: relations may swap only where those agree to 1e-5
        assert (np.abs(pair_scores[j, got_ids] - pair_scores[j, ref]) <= 1e-5).all()
        np.testing.assert_allclose([float(r[3]) for r in got], pair_scores[j, got_ids], rtol=1e-5, atol=1e-6)
    # entity queries in the same file give the rows the entity path gives on its own
    ent_rows = [r for r in rows if int(r[0]) % 2 == 1]
    ids, _, scores = scorer.predict_top_k(tri, k, 1, filtered=True)
    expect = [(2 * j + 1, p + 1, ent[int(ids[j, p])]) for j in range(len(tri)) for p in range(k) if ids[j, p] >= 0]
    assert [(int(a), int(b), c) for a, b, c, _ in ent_rows] == expect


def test_train_relation_metrics_flag_prints_the_relation_table(toy, tmp_path, capsys):
    from relationprediction_b200 import train as driver
    from test_gpu_train import TOY_EXP, write_toy
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(TOY_EXP.format(layers=2, concat="Yes"))
    args = ["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "40", "--no-save",
            "--no-early-stopping", "--final-eval", "0"]
    texts = []
    for extra in ([], ["--relation-metrics"]):
        np.random.seed(0)
        torch.manual_seed(0)
        model, scorer = driver.main(args + extra)
        texts.append(capsys.readouterr().out)
    plain, rel = texts
    assert "Validation filtered MRR at iteration 40" in plain and "Relation prediction" not in plain
    assert '"relation"' not in plain
    assert "Relation prediction:" in rel
    table = rel.split("Relation prediction:")[1].strip().splitlines()[:5]
    assert table[0].split() == ["Raw", "Filtered"]
    assert [row.split("\t")[0] for row in table[1:]] == ["MRR", "H@1", "H@3", "H@10"]
    line = json.loads([l for l in rel.splitlines() if l.startswith("{")][-1])
    res = scorer.compute_relation_mrr_scores(np.array(toy["test"])).get_summary().results
    for kind, key in (("Raw", "raw"), ("Filtered", "filtered")):
        for m in ("MRR", "H@1", "H@3", "H@10"):
            assert abs(line["relation"][key][m] - res[kind][m]) < 1e-12
            assert 0.0 < line["relation"]["filtered"]["MRR"] <= 1.0
