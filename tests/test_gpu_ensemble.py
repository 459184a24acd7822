"""GPU: the fused R-GCN+ ensemble ranker (rgcn_ensemble_rank, ops.EnsembleRanker, ensemble.Ensemble) against the
single-model fused rankers (exact identities), the numpy oracle of tests/ensemble_oracle.py, and end to end on Toy
against the Ensemble's score-matrix path."""
import json

import numpy as np
import pytest
import torch

import ensemble_oracle as oracle
from relationprediction_b200 import ops
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RANKERS = {oracle.DISTMULT: ops.DistMultRanker, oracle.COMPLEX: ops.ComplexRanker}


def make_known(rng, X, V, side, include_gold=True):
    lists = []
    for t in X:
        k = set(rng.randint(0, V, rng.randint(0, 12)).tolist())
        gold = int(t[0] if side == 0 else t[2])
        if include_gold:
            k.add(gold)
        else:
            k.discard(gold)
        lists.append(sorted(k))
    return lists


def _mask(lists, V):
    return torch.as_tensor(BilinearDiag.known_bit_mask(lists, V), device=DEV)


def _np(pair):
    raw, filt = pair
    return raw.cpu().numpy(), None if filt is None else filt.cpu().numpy()


def _ranker(decoder, codes, rel):
    return RANKERS[decoder](torch.as_tensor(codes, device=DEV), torch.as_tensor(rel, device=DEV))


def _triples(rng, V, Vrel, n):
    return np.stack([rng.randint(0, V, n), rng.randint(0, Vrel, n), rng.randint(0, V, n)], 1).astype(np.int32)


# ---- identities: exact ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("decoder", [oracle.DISTMULT, oracle.COMPLEX])
def test_identities_are_exact_at_fb15k237_size(decoder):
    """Ensemble(M, M, w) ranks as M for any w, (A, B, 1) as A and (A, B, 0) as B: each output element sees its
    member's K steps in the single-model kernel's order, and the float64 combination of one float32 value is strictly
    monotone, so no tie appears or disappears."""
    rng = np.random.RandomState(3)
    V, n = 14541, 1000
    ra = _ranker(decoder, rng.normal(0, 0.3, (V, 500)).astype(np.float32),
                 rng.normal(0, 1, (237, 500)).astype(np.float32))
    rb = _ranker(1 - decoder, rng.normal(0, 0.3, (V, 200)).astype(np.float32),
                 rng.normal(0, 1, (237, 200)).astype(np.float32))
    X = torch.as_tensor(_triples(rng, V, 237, n), device=DEV)
    for side in (0, 1):
        mask = _mask(make_known(rng, X.cpu().numpy(), V, side), V)
        for single, other in ((ra, rb), (rb, ra)):
            ref = _np(single.rank(X, side, mask))
            for w in (0.0, 0.3, 0.5, 1.0):
                got = _np(ops.EnsembleRanker(single, single, w).rank(X, side, mask))
                np.testing.assert_array_equal(got[0], ref[0], err_msg="self raw w=%g side %d" % (w, side))
                np.testing.assert_array_equal(got[1], ref[1], err_msg="self filtered w=%g side %d" % (w, side))
            for w, ens in ((1.0, ops.EnsembleRanker(single, other, 1.0)), (0.0, ops.EnsembleRanker(other, single, 0.0))):
                got = _np(ens.rank(X, side, mask))
                np.testing.assert_array_equal(got[0], ref[0], err_msg="w=%g raw side %d" % (w, side))
                np.testing.assert_array_equal(got[1], ref[1], err_msg="w=%g filtered side %d" % (w, side))
            raw_only = _np(ops.EnsembleRanker(single, other, 1.0).rank(X, side, None))
            assert raw_only[1] is None
            np.testing.assert_array_equal(raw_only[0], ref[0])


# ---- against the numpy oracle ---------------------------------------------------------------------------------
# (decoder A, d_A, decoder B, d_B, V, n, w)
ORACLE_CASES = [
    (oracle.DISTMULT, 500, oracle.DISTMULT, 500, 14541, 777, 0.5),
    (oracle.COMPLEX, 500, oracle.COMPLEX, 500, 14541, 129, 0.25),
    (oracle.DISTMULT, 500, oracle.COMPLEX, 200, 129, 777, 0.25),
    (oracle.COMPLEX, 200, oracle.DISTMULT, 500, 65, 128, 0.5),
    (oracle.DISTMULT, 8, oracle.COMPLEX, 12, 1, 127, 0.5),
    (oracle.COMPLEX, 8, oracle.DISTMULT, 12, 63, 129, 0.25),
    (oracle.DISTMULT, 12, oracle.DISTMULT, 8, 64, 1, 0.5),
    (oracle.COMPLEX, 12, oracle.COMPLEX, 8, 14541, 128, 0.5),
]


def _codes(rng, kind, shape):
    """Integer codes, or float codes in multiples of 1/16: either way every product and partial sum of the GEMM is
    exact in float32, so the energies equal the float64 oracle's and only the float32 sigmoid can differ (expf
    against a correctly rounded exp, an ulp or two).  Non-negative and sparse, so that few energies saturate."""
    if kind == "int":
        return (rng.randint(0, 3, shape) * (rng.uniform(size=shape) < 0.15)).astype(np.float32)
    return (np.abs(np.round(rng.normal(0, 0.6, shape) * 16)) / 16 * (rng.uniform(size=shape) < 0.3)).astype(np.float32)


ORACLE_TOL = 2 * 2.0 ** -24   # two float32 ulps of a score in [0.5, 1)


@pytest.mark.parametrize("kind", ["int", "float"])
@pytest.mark.parametrize("case", ORACLE_CASES, ids=lambda c: "%d.%d-%d.%d-V%d-n%d-w%g" % c)
def test_ranks_match_the_oracle_except_on_flagged_near_ties(kind, case):
    dec_a, d_a, dec_b, d_b, V, n, w = case
    rng = np.random.RandomState(V + n + d_a)
    R = 7
    ca, rla = _codes(rng, kind, (V, d_a)), _codes(rng, kind, (R, d_a))
    cb, rlb = _codes(rng, kind, (V, d_b)), _codes(rng, kind, (R, d_b))
    X = _triples(rng, V, R, n)
    ens = ops.EnsembleRanker(_ranker(dec_a, ca, rla), _ranker(dec_b, cb, rlb), w)
    Xt = torch.as_tensor(X, device=DEV)
    tol = ORACLE_TOL
    for side in (0, 1):
        gold = X[:, 0] if side == 0 else X[:, 2]
        known = make_known(rng, X, V, side)
        raw, filt = _np(ens.rank(Xt, side, _mask(known, V)))
        ea, eb = oracle.energies(dec_a, ca, rla, X, side), oracle.energies(dec_b, cb, rlb, X, side)
        c = oracle.combine(w, oracle.sigmoid32(ea), oracle.sigmoid32(eb))
        ref_raw, ref_filt = oracle.ranks(c, gold, known)
        flagged = oracle.near_tie_rows(ea, eb, w, gold, tol)
        # at w = 0.5 sums like s(a) + s(-a) = s(b) + s(-b) = 1 tie to within an ulp; a few small cases flag ~11%
        assert flagged.mean() <= 0.12, (flagged.mean(), flagged.sum())
        ok = ~flagged
        np.testing.assert_array_equal(raw[ok], ref_raw[ok], err_msg="raw side %d" % side)
        np.testing.assert_array_equal(filt[ok], ref_filt[ok], err_msg="filtered side %d" % side)
        assert np.all(raw >= 1) and np.all(filt >= 1) and np.all(raw <= V)


# ---- edge cases -----------------------------------------------------------------------------------------------
def _edge_setup(seed=5, V=1000, n=300):
    rng = np.random.RandomState(seed)
    ca, rla = _codes(rng, "int", (V, 16)), _codes(rng, "int", (9, 16))
    cb, rlb = _codes(rng, "int", (V, 24)), _codes(rng, "int", (9, 24))
    X = _triples(rng, V, 9, n)
    return rng, V, X, (oracle.DISTMULT, ca, rla), (oracle.COMPLEX, cb, rlb)


def test_known_masks_empty_full_and_without_gold():
    rng, V, X, A, B = _edge_setup()
    ens = ops.EnsembleRanker(_ranker(*A), _ranker(*B), 0.25)
    Xt = torch.as_tensor(X, device=DEV)
    for side in (0, 1):
        gold = X[:, 0] if side == 0 else X[:, 2]
        c = oracle.combine(0.25, oracle.sigmoid32(oracle.energies(A[0], A[1], A[2], X, side)),
                           oracle.sigmoid32(oracle.energies(B[0], B[1], B[2], X, side)))
        raw_ref = oracle.ranks(c, gold)[0]
        raw, filt = _np(ens.rank(Xt, side, _mask([[] for _ in X], V)))
        np.testing.assert_array_equal(filt, raw + 1)                      # nothing known: raw + 1
        raw_full, filt_full = _np(ens.rank(Xt, side, _mask([list(range(V))] * len(X), V)))
        np.testing.assert_array_equal(filt_full, np.ones(len(X)))         # everything known: 1
        np.testing.assert_array_equal(raw_full, raw)
        known = make_known(rng, X, V, side, include_gold=False)
        raw_ng, filt_ng = _np(ens.rank(Xt, side, _mask(known, V)))
        np.testing.assert_array_equal(filt_ng, oracle.ranks(c, gold, known)[1])
        for got in (raw, raw_ng):
            np.testing.assert_array_equal(got, raw_ref)


def test_split_reuse_across_small_chunks_and_repeatability():
    rng, V, X, A, B = _edge_setup(seed=6, V=2000, n=700)
    ra, rb = _ranker(*A), _ranker(*B)
    Xt = torch.as_tensor(X, device=DEV)
    known = make_known(rng, X, V, 1)
    mask = _mask(known, V)
    whole = _np(ops.EnsembleRanker(ra, rb, 0.5).rank(Xt, 1, mask))
    again = _np(ops.EnsembleRanker(ra, rb, 0.5).rank(Xt, 1, mask))
    for g, r in zip(whole, again):
        assert np.array_equal(g, r)                                       # bitwise repeatable
    ens = ops.EnsembleRanker(ra, rb, 0.5)
    parts = [[], []]
    for c0 in range(0, len(X), 64):                                       # the split is made by the first chunk only
        raw, filt = _np(ens.rank(Xt[c0:c0 + 64], 1, mask[c0:c0 + 64]))
        parts[0].append(raw)
        parts[1].append(filt)
        assert ens._split_ready
    np.testing.assert_array_equal(np.concatenate(parts[0]), whole[0])
    np.testing.assert_array_equal(np.concatenate(parts[1]), whole[1])
    # Ensemble.rank_all_entities with chunks forced small, through the models' hooks
    from relationprediction_b200 import ensemble as ens_mod

    class Member(object):
        def __init__(self, ranker):
            self.ranker, self.entity_count = ranker, V

        def supports_fused_ranking(self):
            return True

        def test_ranker(self):
            return self.ranker

        def entity_ranker(self, triplets):
            return self.ranker

        def get_device(self):
            return torch.device(DEV)

    model = ens_mod.Ensemble(Member(ra), Member(rb), 0.5)
    ks = make_known(rng, X, V, 0)
    res = model.rank_all_entities(X, ks, known, chunk=100)
    np.testing.assert_array_equal(res[2], whole[0])
    np.testing.assert_array_equal(res[3], whole[1])
    ref0 = _np(ops.EnsembleRanker(ra, rb, 0.5).rank(Xt, 0, _mask(ks, V)))
    np.testing.assert_array_equal(res[0], ref0[0])
    np.testing.assert_array_equal(res[1], ref0[1])


# ---- end to end on Toy ----------------------------------------------------------------------------------------
def test_command_and_fused_scorer_on_toy(toy, tmp_path, capsys):
    from relationprediction_b200 import ensemble as ens_mod
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
    capsys.readouterr()
    results = ens_mod.main(["--dataset", str(tmp_path), "--member", str(gcn_exp), str(tmp_path / "gcn-0.pt"),
                            "--member", str(dm_exp), str(tmp_path / "dm-0.pt")])
    out = capsys.readouterr().out
    assert out.count("\tRaw\tFiltered") == 3 and "Member A" in out and "Member B" in out and "Ensemble" in out
    line = json.loads(out.strip().splitlines()[-1])
    assert line["weight"] == 0.5 and line["triples"] == len(toy["test"])
    for key in ("a", "b", "ensemble"):
        assert 0.0 < line[key]["Filtered"]["MRR"] <= 1.0
        assert line[key] == results[key]
    # the fused Scorer path with an Ensemble against the score-matrix path
    ensemble = ens_mod.Ensemble(models[0], models[1], 0.5)
    assert ensemble.supports_fused_ranking()
    scorer.register_model(ensemble)
    test = np.array(toy["test"])
    fused = scorer.compute_scores(test).get_summary().results
    ensemble.supports_fused_ranking = lambda: False
    matrix = scorer.compute_scores(test).get_summary().results
    for kind in ("Raw", "Filtered"):
        for k in ("MRR", "H@1", "H@3", "H@10"):
            assert abs(fused[kind][k] - matrix[kind][k]) < 2e-2, (kind, k, fused[kind][k], matrix[kind][k])
