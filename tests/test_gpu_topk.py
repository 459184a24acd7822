"""GPU: fused top-k entity prediction (distmult_topk / rgcn_complex_topk: the scoring GEMM with a top-k epilogue and a
merge) against a float64 restatement of the order -- energy descending, the smaller entity id first on ties, excluded
entities never returned, the tail padded (-1, -inf) -- for DistMult and ComplEx on both sides, and the whole chain up
to Scorer.predict_top_k and the predict command."""
import numpy as np
import pytest
import torch

from relationprediction_b200 import ops
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RANKERS = {"distmult": ops.DistMultRanker, "complex": ops.ComplexRanker}


def queries64(codes, rel, X, side, decoder):
    """float64 query rows: DistMult rel[r] * codes[o] / codes[s] * rel[r]; ComplEx the complex products."""
    c, r = codes.astype(np.float64), rel.astype(np.float64)
    kept = c[X[:, 2]] if side == 0 else c[X[:, 0]]
    b = r[X[:, 1]]
    if decoder == "distmult":
        return b * kept
    h = c.shape[1] // 2
    kr, ki, br, bi = kept[:, :h], kept[:, h:], b[:, :h], b[:, h:]
    if side == 0:
        return np.concatenate([br * kr + bi * ki, br * ki - bi * kr], 1)
    return np.concatenate([kr * br - ki * bi, ki * br + kr * bi], 1)


def energies64(codes, rel, X, side, decoder):
    return queries64(codes, rel, X, side, decoder) @ codes.astype(np.float64).T


def reference_topk(e, k, exclude_lists=None):
    """ids / energies of the k best per row of the float64 energies e [n, V], energy descending, smaller id first."""
    n, V = e.shape
    ok = np.ones((n, V), bool)
    if exclude_lists is not None:
        for i, l in enumerate(exclude_lists):
            ok[i, np.asarray(l, dtype=np.int64)] = False
    key = np.where(ok, -e, np.inf)
    order = np.lexsort((np.broadcast_to(np.arange(V), (n, V)), key), axis=-1)[:, :k]
    ids = order.astype(np.int64)
    en = np.take_along_axis(e, order, 1).astype(np.float32)
    valid = np.take_along_axis(ok, order, 1)
    ids = np.where(valid, ids, -1)
    en = np.where(valid, en, -np.inf).astype(np.float32)
    if k > V:
        ids = np.concatenate([ids, -np.ones((n, k - V), np.int64)], 1)
        en = np.concatenate([en, np.full((n, k - V), -np.inf, np.float32)], 1)
    return ids, en


def integer_problem(rng, V, d, n, density=0.05):
    codes = (rng.randint(-1, 2, (V, d)) * (rng.uniform(size=(V, d)) < density)).astype(np.float32)
    rel = rng.randint(-1, 2, (V, d)).astype(np.float32)
    X = np.stack([rng.randint(0, V, n), rng.randint(0, V, n), rng.randint(0, V, n)], 1).astype(np.int32)
    return codes, rel, X


def random_exclusion(rng, n, V):
    return [sorted(set(rng.randint(0, V, rng.randint(0, V // 3 + 2)).tolist())) for _ in range(n)]


def run(ranker, X, side, k, lists, V):
    mask = None if lists is None else torch.as_tensor(BilinearDiag.known_bit_mask(lists, V), device=DEV)
    ids, en = ranker.top_k(torch.as_tensor(X, device=DEV), side, k, mask)
    return ids.cpu().numpy().astype(np.int64), en.cpu().numpy()


@pytest.mark.parametrize("decoder", sorted(RANKERS))
@pytest.mark.parametrize("k", [1, 10, 128])
@pytest.mark.parametrize("V,n", [(129, 5), (1000, 300), (4133, 777)])
def test_integer_codes_give_the_exact_order_with_ties(decoder, k, V, n):
    """Integer codes: every energy is exact in the 3xTF32 GEMM, so ties are real and the tie order is checked."""
    rng = np.random.RandomState(V + k)
    codes, rel, X = integer_problem(rng, V, 64, n)
    ranker = RANKERS[decoder](torch.as_tensor(codes, device=DEV), torch.as_tensor(rel, device=DEV))
    for side in (0, 1):
        e = energies64(codes, rel, X, side, decoder)
        for lists in (None, random_exclusion(rng, n, V)):
            ids, en = run(ranker, X, side, k, lists, V)
            ref_ids, ref_en = reference_topk(e, k, lists)
            np.testing.assert_array_equal(ids, ref_ids)
            np.testing.assert_array_equal(en, ref_en)


@pytest.mark.parametrize("decoder", sorted(RANKERS))
def test_float_codes_match_float64_up_to_near_ties(decoder):
    rng = np.random.RandomState(1)
    V, d, n, k = 14541, 500, 1000, 10           # FB15k-237 entities, complex.exp width
    codes = rng.normal(0, 0.3, (V, d)).astype(np.float32)
    rel = rng.normal(0, 1, (V, d)).astype(np.float32)
    X = np.stack([rng.randint(0, V, n), rng.randint(0, 237, n), rng.randint(0, V, n)], 1).astype(np.int32)
    ranker = RANKERS[decoder](torch.as_tensor(codes, device=DEV), torch.as_tensor(rel, device=DEV))
    for side in (0, 1):
        e = energies64(codes, rel, X, side, decoder)
        ids, en = run(ranker, X, side, k, None, V)
        ref_ids, ref_en = reference_topk(e, k)
        assert (ids >= 0).all()
        got64 = np.take_along_axis(e, ids, 1)
        scale = np.abs(ref_en).astype(np.float64) + 1e-30
        assert (np.abs(en - got64) <= 1e-4 * np.abs(got64) + 1e-6).all()
        swapped = ids != ref_ids
        # a different entity at a position is allowed only where the two float64 energies agree to 1e-5
        assert (np.abs(got64 - ref_en.astype(np.float64))[swapped] <= 1e-5 * scale[swapped]).all()
        assert swapped.mean() < 0.01


@pytest.mark.parametrize("decoder", sorted(RANKERS))
def test_positions_agree_with_the_fused_ranker(decoder):
    """Energies within +-16 (fp32 sigmoid strictly increasing), exclusion = known minus gold: a gold entity with
    filtered rank <= k sits at that rank minus the eligible entities that tie with it and have a larger id (the rank
    counts ties against the gold entity; the top-k list puts the smaller id first)."""
    rng = np.random.RandomState(7)
    V, n, k = 600, 400, 128
    codes, rel, X = integer_problem(rng, V, 8, n, density=0.5)            # |energy| <= 2 d = 16
    ranker = RANKERS[decoder](torch.as_tensor(codes, device=DEV), torch.as_tensor(rel, device=DEV))
    checked = 0
    for side in (0, 1):
        e = energies64(codes, rel, X, side, decoder)
        assert np.abs(e).max() <= 16
        gold = X[:, 0] if side == 0 else X[:, 2]
        known = [sorted(set(rng.randint(0, V, rng.randint(0, 60)).tolist()) | {int(g)}) for g in gold]
        mask = torch.as_tensor(BilinearDiag.known_bit_mask(known, V), device=DEV)
        _, filt = ranker.rank(torch.as_tensor(X, device=DEV), side, mask)
        filt = filt.cpu().numpy()
        excl = [[v for v in l if v != g] for l, g in zip(known, gold)]
        ids, _ = run(ranker, X, side, k, excl, V)
        for t in range(n):
            if filt[t] > k:
                continue
            g = int(gold[t])
            eligible = np.ones(V, bool)
            eligible[excl[t]] = False
            later_ties = int(((e[t] == e[t, g]) & eligible & (np.arange(V) > g)).sum())
            pos = int(np.nonzero(ids[t] == g)[0][0]) + 1
            assert pos == filt[t] - later_ties, (t, pos, filt[t], later_ties)
            checked += 1
    assert checked > 50


@pytest.mark.parametrize("decoder", sorted(RANKERS))
def test_rows_with_fewer_than_k_eligible_entities_are_padded(decoder):
    rng = np.random.RandomState(3)
    V, n = 700, 40
    codes, rel, X = integer_problem(rng, V, 32, n, density=0.3)
    ranker = RANKERS[decoder](torch.as_tensor(codes, device=DEV), torch.as_tensor(rel, device=DEV))
    keep = [sorted(rng.choice(V, i % 6, replace=False).tolist()) for i in range(n)]   # 0..5 eligible entities
    lists = [sorted(set(range(V)) - set(kp)) for kp in keep]
    for side in (0, 1):
        e = energies64(codes, rel, X, side, decoder)
        ids, en = run(ranker, X, side, 10, lists, V)
        ref_ids, ref_en = reference_topk(e, 10, lists)
        np.testing.assert_array_equal(ids, ref_ids)
        np.testing.assert_array_equal(en, ref_en)
        for t, kp in enumerate(keep):
            assert sorted(ids[t, :len(kp)].tolist()) == kp
            assert (ids[t, len(kp):] == -1).all() and np.isneginf(en[t, len(kp):]).all()
    # fewer entities than k
    small_codes, small_rel, Xs = integer_problem(rng, 50, 32, 9, density=0.3)
    ranker = RANKERS[decoder](torch.as_tensor(small_codes, device=DEV), torch.as_tensor(small_rel, device=DEV))
    ids, en = run(ranker, Xs, 1, 100, None, 50)
    ref_ids, ref_en = reference_topk(energies64(small_codes, small_rel, Xs, 1, decoder), 100)
    np.testing.assert_array_equal(ids, ref_ids)
    np.testing.assert_array_equal(en, ref_en)
    assert (ids[:, 50:] == -1).all() and np.isneginf(en[:, 50:]).all()


@pytest.mark.parametrize("decoder", sorted(RANKERS))
def test_output_is_repeatable_and_split_reuse_across_chunks_changes_nothing(decoder):
    rng = np.random.RandomState(5)
    V, d, n, k = 5000, 200, 900, 10
    codes = rng.normal(0, 0.3, (V, d)).astype(np.float32)
    rel = rng.normal(0, 1, (V, d)).astype(np.float32)
    X = np.stack([rng.randint(0, V, n), rng.randint(0, 50, n), rng.randint(0, V, n)], 1).astype(np.int32)
    lists = random_exclusion(rng, n, V)
    ct, rt = torch.as_tensor(codes, device=DEV), torch.as_tensor(rel, device=DEV)
    ranker = RANKERS[decoder](ct, rt)
    a = run(ranker, X, 1, k, lists, V)
    b = run(ranker, X, 1, k, lists, V)                  # split reused
    c = run(RANKERS[decoder](ct, rt), X, 1, k, lists, V)  # fresh split
    chunked = RANKERS[decoder](ct, rt)
    chunked.TOPK_CHUNK_BYTES = 100 * (4 * d + 8 * k * ((V + 127) // 128))   # about 100 queries per library call
    c2 = run(chunked, X, 1, k, lists, V)
    for other in (b, c, c2):
        np.testing.assert_array_equal(a[0], other[0])
        assert a[1].tobytes() == other[1].tobytes()
    # rank and top_k share one workspace and its split
    ranker.rank(torch.as_tensor(X, device=DEV), 1, None)
    np.testing.assert_array_equal(run(ranker, X, 1, k, lists, V)[0], a[0])


def _trained_toy(toy, tmp_path, decoder):
    from relationprediction_b200 import train as driver
    from test_gpu_train import TOY_EXP, write_toy
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    if decoder == "distmult":
        exp.write_text(TOY_EXP.format(layers=2, concat="Yes"))
    else:
        exp.write_text(toy["settings_text"]["complex.exp"].replace("CodeDimension=500", "CodeDimension=32"))
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "30",
                                 "--no-periodic-eval", "--no-save"])
    return exp, model, scorer


def host_topk(scores, k, exclude):
    """ids of the k best scores per row after removing `exclude`, scores descending, smaller id first."""
    out = []
    for i, row in enumerate(scores):
        ok = np.ones(len(row), bool)
        ok[np.asarray(exclude[i], dtype=np.int64)] = False
        cand = np.nonzero(ok)[0]
        cand = cand[np.lexsort((cand, -row[cand].astype(np.float64)))][:k]
        out.append(np.concatenate([cand, -np.ones(k - len(cand), np.int64)]))
    return np.array(out)


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
def test_scorer_predict_top_k_agrees_with_the_score_matrices(toy, tmp_path, decoder):
    _, model, scorer = _trained_toy(toy, tmp_path, decoder)
    triples = np.array(toy["test"])
    k = 10
    for side in (0, 1):
        mat = model.score_all_subjects(triples) if side == 0 else model.score_all_objects(triples)
        for filtered in (True, False):
            ids, energies, scores = scorer.predict_top_k(triples, k, side, filtered=filtered)
            if filtered:
                known = (scorer.known_subject_triples if side == 0 else scorer.known_object_triples)
                excl = [known.get((t[2], t[1]) if side == 0 else (t[0], t[1]), []) for t in triples.tolist()]
            else:
                excl = [[] for _ in triples]
            ref = host_topk(mat, k, excl)
            assert ids.shape == (len(triples), k) and scores.dtype == np.float32
            valid = ids >= 0
            np.testing.assert_array_equal(valid, ref >= 0)
            got_s = np.where(valid, np.take_along_axis(mat, np.maximum(ids, 0), 1), 0)
            ref_s = np.where(valid, np.take_along_axis(mat, np.maximum(ref, 0), 1), 0)
            # the matrix path is a torch fp32 matmul: entities may swap only where their scores agree to 1e-5
            assert (np.abs(got_s - ref_s) <= 1e-5).all()
            np.testing.assert_allclose(scores[valid], got_s[valid], rtol=1e-5, atol=1e-6)
            for i, l in enumerate(excl):
                assert not set(ids[i][valid[i]].tolist()) & set(l)


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
def test_predict_command_on_toy(toy, tmp_path, decoder):
    from relationprediction_b200 import predict as predict_cmd
    exp, model, scorer = _trained_toy(toy, tmp_path, decoder)
    model.save(str(tmp_path / "Toy"))
    ckpts = list(tmp_path.glob("Toy-*.pt"))
    assert len(ckpts) == 1
    ent = {int(k): v for k, v in toy["entities"].items()}
    rel = {int(k): v for k, v in toy["relations"].items()}
    tri = np.array(toy["test"])[:12]
    lines = ["%s\t%s\t?" % (ent[s], rel[r]) if i % 2 else "?\t%s\t%s" % (rel[r], ent[o])
             for i, (s, r, o) in enumerate(tri.tolist())]
    (tmp_path / "queries.tsv").write_text("\n".join(lines) + "\n")
    out = tmp_path / "answers.tsv"
    for raw in (False, True):
        predict_cmd.main(["--settings", str(exp), "--dataset", str(tmp_path), "--checkpoint", str(ckpts[-1]),
                          "--queries", str(tmp_path / "queries.tsv"), "--k", "5", "--out", str(out)]
                         + (["--raw"] if raw else []))
        rows = [l.split("\t") for l in out.read_text().splitlines()]
        expect = []
        for i, t in enumerate(tri):
            side = 1 if i % 2 else 0
            ids, _, scores = scorer.predict_top_k(t[None], 5, side, filtered=not raw)
            expect += [(i, p + 1, ent[int(ids[0, p])], float(scores[0, p])) for p in range(5) if ids[0, p] >= 0]
        assert [(int(a), int(b), c) for a, b, c, _ in rows] == [e[:3] for e in expect]
        np.testing.assert_allclose([float(r[3]) for r in rows], [e[3] for e in expect], rtol=1e-6)
