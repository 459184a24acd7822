"""GPU: the R-GCN+ ensemble's fused top-k entity and relation prediction and relation ranks (rgcn_ensemble_topk,
rgcn_ensemble_relation_rank, rgcn_ensemble_relation_topk; ops.EnsembleRanker; ensemble.Ensemble) against the float64
restatement of tests/ensemble_topk_oracle.py, exact identities with the single-model paths, split reuse, chunking,
repeatability, and the ensemble command's query mode and relation metrics end to end on Toy."""
import json

import numpy as np
import pytest
import torch

import ensemble_oracle as oracle
import ensemble_topk_oracle as tko
from relationprediction_b200 import ops
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RANKERS = {oracle.DISTMULT: ops.DistMultRanker, oracle.COMPLEX: ops.ComplexRanker}
V237, R237 = 14541, 237


def _ranker(decoder, codes, rel, R=None):
    return RANKERS[decoder](torch.as_tensor(codes, device=DEV), torch.as_tensor(rel, device=DEV), R)


def _mask(lists, count):
    return None if lists is None else torch.as_tensor(BilinearDiag.known_bit_mask(lists, count), device=DEV)


def _np(res):
    return tuple(x.cpu().numpy() for x in res)


def _member(rng, decoder, V, Vrel, d, scale=0.3):
    return (decoder, rng.normal(0, scale, (V, d)).astype(np.float32), rng.normal(0, 1, (Vrel, d)).astype(np.float32))


def _exclusions(rng, n, count, k):
    """Random exclusion lists, with row 0 fully excluded and row 1 left with fewer than k candidates."""
    lists = [sorted(set(rng.randint(0, count, rng.randint(0, 20)).tolist())) for _ in range(n)]
    lists[0] = list(range(count))
    lists[1] = list(range(k - 1, count))    # k - 1 left
    return lists


MIXES = {"dm500+dm512": ((oracle.DISTMULT, 500), (oracle.DISTMULT, 512)),
         "dm500+cx512": ((oracle.DISTMULT, 500), (oracle.COMPLEX, 512)),
         "cx500+dm200": ((oracle.COMPLEX, 500), (oracle.DISTMULT, 200))}


@pytest.mark.parametrize("mix", sorted(MIXES))
@pytest.mark.parametrize("k", [1, 10, 128])
def test_top_k_against_float64_at_fb15k237_size(mix, k):
    rng = np.random.RandomState(11 + k)
    (da_kind, d_a), (db_kind, d_b) = MIXES[mix]
    Vrel = V237 + 13   # a longer relation table than R: rows R.. are never candidates
    ma, mb = _member(rng, da_kind, V237, Vrel, d_a), _member(rng, db_kind, V237, Vrel, d_b)
    w = 0.35
    ranker = ops.EnsembleRanker(_ranker(*ma, R237), _ranker(*mb, R237), w)
    n = 150
    X = np.stack([rng.randint(0, V237, n), rng.randint(0, R237, n), rng.randint(0, V237, n)], 1).astype(np.int32)
    Xd = torch.as_tensor(X, device=DEV)
    for side in (0, 1):
        excl = _exclusions(rng, n, V237, k)
        u_ref = tko.u_of(w, oracle.energies(ma[0], ma[1], ma[2], X, side), oracle.energies(mb[0], mb[1], mb[2], X, side))
        ids, u, sc = _np(ranker.top_k(Xd, side, k, _mask(excl, V237)))
        tko.check_top_k(ids, u, sc, u_ref, k, excl)
        ids, u, sc = _np(ranker.top_k(Xd, side, k))
        tko.check_top_k(ids, u, sc, u_ref, k)
    excl = _exclusions(rng, n, R237, k)
    u_ref = tko.u_of(w, tko.relation_energies(ma[0], ma[1], ma[2], X, R237),
                     tko.relation_energies(mb[0], mb[1], mb[2], X, R237))
    ids, u, sc = _np(ranker.top_k_relations(Xd, k, _mask(excl, R237)))
    tko.check_top_k(ids, u, sc, u_ref, k, excl)
    ids, u, sc = _np(ranker.top_k_relations(Xd, k))
    tko.check_top_k(ids, u, sc, u_ref, k)


@pytest.mark.parametrize("N", [1, 63, 65, 200])
def test_candidate_counts_not_multiples_of_64(N):
    rng = np.random.RandomState(N)
    ma, mb = _member(rng, oracle.DISTMULT, N, N, 12), _member(rng, oracle.COMPLEX, N, N, 8)
    ranker = ops.EnsembleRanker(_ranker(*ma), _ranker(*mb), 0.5)
    X = np.stack([rng.randint(0, N, 70), rng.randint(0, N, 70), rng.randint(0, N, 70)], 1).astype(np.int32)
    Xd = torch.as_tensor(X, device=DEV)
    for k in (1, 10, 128):
        u_ref = tko.u_of(0.5, oracle.energies(ma[0], ma[1], ma[2], X, 1), oracle.energies(mb[0], mb[1], mb[2], X, 1))
        tko.check_top_k(*_np(ranker.top_k(Xd, 1, k)), u_ref, k)
        u_ref = tko.u_of(0.5, tko.relation_energies(ma[0], ma[1], ma[2], X, N),
                         tko.relation_energies(mb[0], mb[1], mb[2], X, N))
        tko.check_top_k(*_np(ranker.top_k_relations(Xd, k)), u_ref, k)


def test_saturated_energies_keep_their_order():
    """Energies far past the float32 sigmoid's saturation (20 .. 600) still order by u: one-hot codes make the
    energy of entity v exactly scale_v."""
    V, d = 40, 4
    scales = np.array([20, 40, 200, 600, 25, 19, 41, 201] + [1] * (V - 8), np.float32)
    codes = np.zeros((V, d), np.float32)
    codes[:, 0] = scales
    codes[0, 0] = 1.0                       # the query's anchor: q = codes[0] * rel[0] = e_0
    rel = np.zeros((3, d), np.float32)
    rel[:, 0] = 1.0
    m = (oracle.DISTMULT, codes, rel)
    ranker = ops.EnsembleRanker(_ranker(*m), _ranker(*m), 0.5)
    X = torch.as_tensor(np.array([[0, 0, 0]], np.int32), device=DEV)
    ids, u, sc = _np(ranker.top_k(X, 1, 8))
    assert ids[0].tolist() == [3, 7, 2, 6, 1, 4, 5, 0]      # energy 600, 201, 200, 41, 40, 25, 19, then 1 (id 0)
    assert np.all(np.diff(u[0]) > 0) and u[0][0] > 0        # e^-600 is a normal double
    tko.check_top_k(ids, u, sc, tko.u_of(0.5, codes[:, 0][None], codes[:, 0][None]), 8)


def test_members_with_different_relation_counts_rank_entities_but_refuse_relation_queries():
    """An R-GCN member's relation table has V rows; paired with a plain member of R rows and no relation_count, the
    ensemble still ranks and predicts entities, and only its relation queries refuse the mismatch."""
    rng = np.random.RandomState(2)
    V, n = 300, 40
    ma, mb = _member(rng, oracle.DISTMULT, V, V, 8), _member(rng, oracle.DISTMULT, V, 9, 12)
    ranker = ops.EnsembleRanker(_ranker(*ma), _ranker(*mb), 0.5)
    X = torch.as_tensor(np.stack([rng.randint(0, V, n), rng.randint(0, 9, n), rng.randint(0, V, n)], 1)
                        .astype(np.int32), device=DEV)
    assert ranker.rank(X, 1)[0].shape == (n,) and ranker.top_k(X, 1, 5)[0].shape == (n, 5)
    for call in (lambda: ranker.rank_relations(X), lambda: ranker.top_k_relations(X, 5)):
        with pytest.raises(ValueError, match="relation sets"):
            call()
    fixed = ops.EnsembleRanker(_ranker(*ma, 9), _ranker(*mb), 0.5)
    assert fixed.top_k_relations(X, 5)[0].shape == (n, 5)


# ---- identities: exact on integer codes ---------------------------------------------------------------------------
def _int_member(rng, decoder, V, Vrel, d):
    return (decoder, rng.randint(-1, 2, (V, d)).astype(np.float32), rng.randint(-1, 2, (Vrel, d)).astype(np.float32))


@pytest.mark.parametrize("decoder", [oracle.DISTMULT, oracle.COMPLEX])
def test_identities_on_integer_codes(decoder):
    """Ensemble(M, M, w) predicts as M, (A, B, 1) as A and (A, B, 0) as B: top-k ids of entities (both sides) and
    relations, and the relation ranks, bit for bit.  Integer energies stay far from the double sigmoid's saturation,
    so u orders exactly as the energy does, ties by id included."""
    rng = np.random.RandomState(7)
    V, R, n, k = 3000, 237, 400, 10
    ma, mb = _int_member(rng, decoder, V, R, 8), _int_member(rng, 1 - decoder, V, R, 12)
    single_a, single_b = _ranker(*ma), _ranker(*mb)
    X = np.stack([rng.randint(0, V, n), rng.randint(0, R, n), rng.randint(0, V, n)], 1).astype(np.int32)
    Xd = torch.as_tensor(X, device=DEV)
    known = [sorted(set(rng.randint(0, R, 5).tolist()) | {int(t[1])}) for t in X]
    for ens, single in ((ops.EnsembleRanker(single_a, _ranker(*ma), 0.3), single_a),
                        (ops.EnsembleRanker(single_a, single_b, 1.0), single_a),
                        (ops.EnsembleRanker(single_a, single_b, 0.0), single_b)):
        for side in (0, 1):
            np.testing.assert_array_equal(ens.top_k(Xd, side, k)[0].cpu().numpy(),
                                          single.top_k(Xd, side, k)[0].cpu().numpy())
        np.testing.assert_array_equal(ens.top_k_relations(Xd, k)[0].cpu().numpy(),
                                      single.top_k_relations(Xd, k)[0].cpu().numpy())
        got, want = _np(ens.rank_relations(Xd, _mask(known, R))), _np(single.rank_relations(Xd, _mask(known, R)))
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[1], want[1])


def test_relation_ranks_against_the_oracle():
    rng = np.random.RandomState(5)
    V, R, n, w = 2000, 97, 300, 0.4
    ma, mb = _member(rng, oracle.DISTMULT, V, R, 16, 1.0), _member(rng, oracle.COMPLEX, V, R, 24, 1.0)
    ranker = ops.EnsembleRanker(_ranker(*ma), _ranker(*mb), w)
    X = np.stack([rng.randint(0, V, n), rng.randint(0, R, n), rng.randint(0, V, n)], 1).astype(np.int32)
    known = [sorted(set(rng.randint(0, R, 6).tolist()) | {int(t[1])}) for t in X]
    raw, filt = _np(ranker.rank_relations(torch.as_tensor(X, device=DEV), _mask(known, R)))
    ea = tko.relation_energies(ma[0], ma[1], ma[2], X, R)
    eb = tko.relation_energies(mb[0], mb[1], mb[2], X, R)
    rraw, rfilt = oracle.ranks(oracle.combine(w, oracle.sigmoid32(ea), oracle.sigmoid32(eb)), X[:, 1], known)
    flagged = oracle.near_tie_rows(ea, eb, w, X[:, 1], 2.0 ** -22)   # two float32 ulps of a score near 1
    ok = ~flagged
    assert flagged.mean() < 0.12
    np.testing.assert_array_equal(raw[ok], rraw[ok])
    np.testing.assert_array_equal(filt[ok], rfilt[ok])


def test_split_reuse_chunking_and_repeatability(monkeypatch):
    """Entity, relation and entity calls interleaved on one ranker keep their splits apart; many small chunks give
    the answer of one call; repeated calls are bitwise equal."""
    rng = np.random.RandomState(9)
    V, R, n, k = 5000, 150, 600, 10
    ma, mb = _member(rng, oracle.COMPLEX, V, R, 16), _member(rng, oracle.DISTMULT, V, R, 20)
    X = np.stack([rng.randint(0, V, n), rng.randint(0, R, n), rng.randint(0, V, n)], 1).astype(np.int32)
    Xd = torch.as_tensor(X, device=DEV)
    known = [[int(t[1])] for t in X]
    fresh = lambda: ops.EnsembleRanker(_ranker(*ma), _ranker(*mb), 0.5)
    ref_e = _np(fresh().top_k(Xd, 1, k))
    ref_r = _np(fresh().top_k_relations(Xd, k))
    ref_rank = _np(fresh().rank_relations(Xd, _mask(known, R)))
    ref_rank_e = _np(fresh().rank(Xd, 0, _mask(known, V)))
    r = fresh()
    for _ in range(2):
        for got, ref in ((r.top_k(Xd, 1, k), ref_e), (r.top_k_relations(Xd, k), ref_r),
                         (r.rank_relations(Xd, _mask(known, R)), ref_rank), (r.rank(Xd, 0, _mask(known, V)), ref_rank_e),
                         (r.top_k(Xd, 1, k), ref_e)):
            for g, f in zip(_np(got), ref):
                np.testing.assert_array_equal(g, f)
    monkeypatch.setattr(ops.DistMultRanker, "TOPK_CHUNK_BYTES", 1 << 16)
    small = fresh()
    for got, ref in ((small.top_k(Xd, 1, k), ref_e), (small.top_k_relations(Xd, k), ref_r),
                     (small.rank_relations(Xd, _mask(known, R)), ref_rank)):
        for g, f in zip(_np(got), ref):
            np.testing.assert_array_equal(g, f)


# ---- end to end on Toy ----------------------------------------------------------------------------------------
def test_query_mode_and_relation_metrics_on_toy(toy, tmp_path, capsys):
    from relationprediction_b200 import ensemble as ens_mod
    from relationprediction_b200 import predict
    from relationprediction_b200 import train as driver
    from test_gpu_train import TOY_EXP, write_toy
    write_toy(toy, tmp_path)
    gcn_exp, dm_exp = tmp_path / "gcn.exp", tmp_path / "distmult.exp"
    gcn_exp.write_text(TOY_EXP.format(layers=2, concat="Yes"))
    dm_exp.write_text(toy["settings_text"]["distmult.exp"].replace("CodeDimension=500", "CodeDimension=24"))
    models = []
    for exp, name in ((gcn_exp, "gcn"), (dm_exp, "dm")):
        np.random.seed(0)
        torch.manual_seed(0)
        model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "30",
                                     "--no-periodic-eval", "--no-save"])
        model.save(str(tmp_path / name))
        models.append(model)
    members = ["--member", str(gcn_exp), str(tmp_path / "gcn-0.pt"), "--member", str(dm_exp), str(tmp_path / "dm-0.pt")]
    capsys.readouterr()
    results = ens_mod.main(["--dataset", str(tmp_path)] + members + ["--relation-metrics"])
    out = capsys.readouterr().out
    assert out.count("\tRaw\tFiltered") == 6 and "relation prediction" in out
    line = json.loads(out.strip().splitlines()[-1])
    ensemble = ens_mod.Ensemble(models[0], models[1], 0.5)
    scorer.register_model(ensemble)
    test = np.array(toy["test"])
    rel = scorer.compute_relation_mrr_scores(test).get_summary().results
    assert line["relations"]["ensemble"] == rel == results["relations"]["ensemble"]
    # the query mode answers as Scorer.predict_top_k* on the Ensemble
    entities, relations = driver.load_dataset(str(tmp_path))[1:]
    en, rn = list(entities.values()), list(relations.values())
    t = toy["test"][:3]
    lines = ["%s\t%s\t?" % (entities[t[0][0]], relations[t[0][1]]), "?\t%s\t%s" % (relations[t[1][1]], entities[t[1][2]]),
             "%s\t?\t%s" % (entities[t[2][0]], entities[t[2][2]]), "%s\t%s\t?" % (en[0], rn[0])]
    qfile, ofile = tmp_path / "q.txt", tmp_path / "a.txt"
    qfile.write_text("\n".join(lines) + "\n")
    for raw in (False, True):
        ens_mod.main(["--dataset", str(tmp_path)] + members + ["--queries", str(qfile), "--k", "5", "--out", str(ofile)]
                     + (["--raw"] if raw else []))
        queries = predict.parse_queries(lines, {v: i for i, v in entities.items()}, {v: i for i, v in relations.items()})
        want = predict.answer(scorer, queries, 5, filtered=not raw)
        # the command's models are rebuilt from the checkpoints: the same answers, scores to the encoder's
        # float32 run-to-run spread (its aggregation adds in a run-dependent order)
        got = [line.split("\t") for line in ofile.read_text().splitlines()]
        assert len(got) == len(want) > 0
        for g, (qi, pos, a, sc) in zip(got, want):
            assert g[:3] == [str(qi), str(pos), relations[a] if queries[qi][3] == 2 else entities[a]]
            assert abs(float(g[3]) - sc) <= 1e-6
