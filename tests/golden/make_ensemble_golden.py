"""Golden ranks of the R-GCN+ ensemble produced by RUNNING THE REFERENCE'S OWN TOOLS (needs a checkout of the
reference; run HERE):

  python tests/golden/make_ensemble_golden.py REFERENCE_DIR   ->  tests/golden/reference_ensemble_golden.npz

The reference forms R-GCN+ offline: common/evaluation.py's Scorer.dump_all_scores writes, for every test triple and
both sides, the gold score and every non-known entity's score as text, and code/tools/ensemble.py --method
weighted_sum (WeightEnsemble) reads two such dumps and ranks  c = w s_1 + (1 - w) s_2  as  #{others >= target} + 1.

Here a small synthetic dataset (V = 40, 3 relations, 380 triples: under the Scorer's 1000-triple chunk) is registered
split by split with the reference's own Scorer (it imports only numpy), two stub models return stored float32 score
matrices, dump_all_scores writes each model's files into a temporary directory, and the tool runs through runpy with
a patched sys.argv; its four printed numbers (MRR, H@1, H@3, H@10 at its built-in w = 0.5) and its ranks are kept.
The module's WeightEnsemble is then re-instantiated at w = 0.3 and 0.8.

The scores include ties on purpose: saturated 1.0, exact 0.5, a small pool of repeated values, and pairs of entities
whose A and B scores are swapped (equal combinations at w = 0.5 only), some of them with the gold entity.  The tool
reads the scores back from their shortest float32 decimal text, which differs from the float32 value by less than
half a float32 ulp; that can only change a comparison between two combined scores within ~1e-8 of each other, and
the generator checks that every comparison with the gold score comes out the same from the float32 values."""
import contextlib
import io
import os
import runpy
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
V, R = 40, 3
N_SPLIT = {"train": 300, "valid": 40, "test": 40}
WEIGHTS = (0.5, 0.3, 0.8)


class StubModel(object):
    """score_all_subjects / score_all_objects of the stored [n_test, V] float32 matrices, rows by test triple."""

    def __init__(self, test, subj, obj):
        self.row = {tuple(t): i for i, t in enumerate(np.asarray(test).tolist())}
        self.subj, self.obj = subj, obj

    def _rows(self, triples):
        return [self.row[tuple(t)] for t in np.asarray(triples).tolist()]

    def score_all_subjects(self, triples):
        return self.subj[self._rows(triples)]

    def score_all_objects(self, triples):
        return self.obj[self._rows(triples)]


def make_data(rng):
    seen, splits = set(), {}
    for name, n in N_SPLIT.items():
        rows = []
        while len(rows) < n:
            t = (int(rng.randint(V)), int(rng.randint(R)), int(rng.randint(V)))
            if name != "test" or t not in seen:   # test triples unique: the stubs find their rows by triple
                rows.append(t)
                seen.add(t)
        splits[name] = np.array(rows, dtype=np.int64)
    return splits


def make_scores(rng, test, side):
    """(s_A, s_B) [n, V] float32 with ties; side 0 = subject scores (gold column 0), 1 = object scores (column 2)."""
    n = len(test)
    gold = test[:, 0] if side == 0 else test[:, 2]
    pool = np.array([0.25, 0.75, 0.125, 0.5, 1.0], np.float32)
    out = []
    for _ in range(2):
        s = rng.uniform(0.0, 1.0, (n, V)).astype(np.float32)
        u = rng.uniform(size=(n, V))
        s[u < 0.10] = 1.0                                    # saturated
        s[(u >= 0.10) & (u < 0.18)] = 0.5                    # exact one half
        m = (u >= 0.18) & (u < 0.30)
        s[m] = pool[rng.randint(len(pool), size=int(m.sum()))]
        out.append(s)
    sa, sb = out
    for i in range(n):                                       # swapped pairs: (x, y) at j, (y, x) at k
        for _ in range(3):
            j, k = rng.choice(V, 2, replace=False)
            if rng.uniform() < 0.4:
                j = gold[i] if gold[i] != k else j
            sa[i, k], sb[i, k] = sb[i, j], sa[i, j]
    return sa, sb


def combined(w, sa, sb):
    return w * sa.astype(np.float64) + (1.0 - w) * sb.astype(np.float64)


def check_text_round_trip(w, sa, sb, gold):
    """Every comparison c(t, v) >= c(t, gold) comes out the same from the float32 values and from the decimal text
    the tool reads back."""
    text = np.vectorize(lambda x: float(str(x)), otypes=[np.float64])
    rows = np.arange(len(gold))
    c, ct = combined(w, sa, sb), combined(w, text(sa), text(sb))
    assert np.array_equal(c >= c[rows, gold][:, None], ct >= ct[rows, gold][:, None]), \
        "a comparison depends on the decimal text: pick another seed"


def main(ref):
    sys.path.insert(0, os.path.join(ref, "code"))
    from common import evaluation as ref_eval   # reference module, numpy only
    rng = np.random.RandomState(20261016)
    splits = make_data(rng)
    test = splits["test"]
    sa_s, sb_s = make_scores(rng, test, 0)
    sa_o, sb_o = make_scores(rng, test, 1)
    for w in WEIGHTS:
        check_text_round_trip(w, sa_s, sb_s, test[:, 0])
        check_text_round_trip(w, sa_o, sb_o, test[:, 2])
    scorer = ref_eval.Scorer({})
    for name in ("train", "valid", "test"):
        scorer.register_data(splits[name].tolist())
    tool = os.path.join(ref, "code", "tools", "ensemble.py")
    with tempfile.TemporaryDirectory() as tmp:
        dirs = []
        for tag, subj, obj in (("a", sa_s, sa_o), ("b", sb_s, sb_o)):
            d = os.path.join(tmp, tag)
            os.makedirs(d)
            scorer.register_model(StubModel(test, subj, obj))
            scorer.dump_all_scores(test.tolist(), os.path.join(d, "subjects.test"), os.path.join(d, "objects.test"))
            dirs.append(d)
        argv = sys.argv
        sys.argv = [tool, "--p1", dirs[0], "--p2", dirs[1], "--method", "weighted_sum"]
        buf = io.StringIO()
        try:
            with contextlib.redirect_stdout(buf):
                mod = runpy.run_path(tool, run_name="__main__")
        finally:
            sys.argv = argv
        printed = np.array([float(x) for x in buf.getvalue().split()], np.float64)
        ranks, metrics = [], []
        for w in WEIGHTS:
            ens = mod["model"] if w == 0.5 else mod["WeightEnsemble"](w, dirs[0], dirs[1])
            if w != 0.5:
                ens.compute_ranks()
            ranks.append(np.asarray(ens.ranks, np.int64))
            metrics.append([ens.combined_mrr(), ens.hits_at(1), ens.hits_at(3), ens.hits_at(10)])
    assert printed.shape == (4,) and np.allclose(printed, metrics[0], rtol=0, atol=0), (printed, metrics[0])
    out = os.path.join(HERE, "reference_ensemble_golden.npz")
    np.savez_compressed(out, V=V, R=R, train=splits["train"], valid=splits["valid"], test=test,
                        sa_subjects=sa_s, sb_subjects=sb_s, sa_objects=sa_o, sb_objects=sb_o,
                        weights=np.array(WEIGHTS), ranks=np.stack(ranks), metrics=np.array(metrics, np.float64),
                        printed=printed)
    print("wrote", out, "ranks", np.stack(ranks).shape, "printed", printed.tolist())


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: make_ensemble_golden.py REFERENCE_DIR")
    main(sys.argv[1])
