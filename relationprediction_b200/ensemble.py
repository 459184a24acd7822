"""R-GCN+: two trained models ranked under the weighted sum of their scores.

The paper's R-GCN+ is an R-GCN plus a separately trained DistMult model, combined by a weighted sum of their sigmoid
scores.  The reference produces it offline: Scorer.dump_all_scores (common/evaluation.py:391-408) writes every test
triple's scores as text, and tools/ensemble.py --method weighted_sum (WeightEnsemble, :43-83) reads two such dumps
and ranks  c = w s_A + (1 - w) s_B  with w = 0.5.  Here `Ensemble` is a model the Scorer can evaluate directly:

  c(t, v) = w s_A(t, v) + (1 - w) s_B(t, v)     float64, separately rounded products and sum (the tool's Python
                                                 floats), s_X the member's float32 sigmoid score

ranked by the Scorer's raw / filtered rules.  With every split registered the gold entity is in the known set, and
the filtered rank equals the tool's  #{others >= target} + 1.  When both members have a fused ranker on the same CUDA
device (DistMult or ComplEx decoders) the ranks come from one fused kernel (ops.EnsembleRanker, rgcn_ensemble_rank)
without any [n, V] score matrix; otherwise score_all_subjects / score_all_objects combine the members' matrices.

  python -m relationprediction_b200.ensemble --dataset DIR | --dataset-npz F
                                             --member SETTINGS CHECKPOINT --member SETTINGS CHECKPOINT
                                             [--weight W] [--split test|valid] [--limit N] [--device DEV]

builds each member as the training driver does (train.build_chain), loads its Model.save checkpoint, and prints the
Raw / Filtered table of member A, of member B and of the ensemble (weight W on A, default 0.5 as in the reference
tool), then one JSON line with all three."""
import argparse
import json
import math

import numpy as np
import torch

from . import ops


def _check_weight(weight):
    weight = float(weight)
    if not (math.isfinite(weight) and 0.0 <= weight <= 1.0):
        raise ValueError("the ensemble weight must be in [0, 1], got %r" % weight)
    return weight


class Ensemble(object):
    """Two trained models over the same entities, scored by  w s_A + (1 - w) s_B  (weight w on model_a)."""

    def __init__(self, model_a, model_b, weight=0.5):
        ea, eb = int(model_a.entity_count), int(model_b.entity_count)
        if ea != eb:
            raise ValueError("the ensemble members must share one entity set, got %d and %d entities" % (ea, eb))
        self.a, self.b = model_a, model_b
        self.weight = _check_weight(weight)
        self.entity_count = ea

    # ---- fused path (Scorer.compute_mrr_scores prefers it) ----
    def supports_fused_ranking(self):
        """Both members have a fused ranker (DistMult or ComplEx decoder) and live on the same CUDA device."""
        for m in (self.a, self.b):
            if not (hasattr(m, 'test_ranker') and m.supports_fused_ranking()):
                return False
        return self.a.get_device() == self.b.get_device()

    def rank_all_entities(self, triplets, known_subject_lists, known_object_lists, chunk=4096):
        """Raw and filtered ranks of every triple under subject and object corruption, as Model.rank_all_entities:
        one encoder pass per member, both members' codes split once, chunks of `chunk` triples.  Returns four int64
        arrays (raw_subjects, filtered_subjects, raw_objects, filtered_objects), or None when a member has no fused
        ranker."""
        from .decoders.bilinear_diag import BilinearDiag
        if not self.supports_fused_ranking():
            return None
        tri = np.ascontiguousarray(np.asarray(triplets, dtype=np.int32).reshape(-1, 3))
        ranker_a, ranker_b = self.a.entity_ranker(tri), self.b.entity_ranker(tri)
        ranker = ops.EnsembleRanker(ranker_a, ranker_b, self.weight)
        dev, V = ranker_a.codes.device, self.entity_count
        out = [[], [], [], []]
        with torch.no_grad():
            for c0 in range(0, len(tri), chunk):
                X = torch.as_tensor(tri[c0:c0 + chunk], device=dev)
                for side, lists in ((0, known_subject_lists), (1, known_object_lists)):
                    mask = torch.as_tensor(BilinearDiag.known_bit_mask(lists[c0:c0 + chunk], V), device=dev)
                    raw, filt = ranker.rank(X, side, mask)
                    out[2 * side].append(raw)
                    out[2 * side + 1].append(filt)
        return tuple(torch.cat(o).cpu().numpy().astype(np.int64) if o else np.zeros(0, np.int64) for o in out)

    # ---- score matrices (the fallback path, and the oracle of the fused one) ----
    def _combine(self, sa, sb):
        sa, sb = np.asarray(sa, dtype=np.float64), np.asarray(sb, dtype=np.float64)
        return self.weight * sa + (1.0 - self.weight) * sb   # numpy never fuses these into an FMA

    def score_all_subjects(self, triplets):
        """[n, V] float64 combined scores of every entity as the subject of each triple."""
        return self._combine(self.a.score_all_subjects(triplets), self.b.score_all_subjects(triplets))

    def score_all_objects(self, triplets):
        """[n, V] float64 combined scores of every entity as the object of each triple."""
        return self._combine(self.a.score_all_objects(triplets), self.b.score_all_objects(triplets))


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Evaluate the R-GCN+ ensemble of two trained models: filtered and raw "
                                             "MRR and Hits@1/3/10 of each member and of their weighted score sum.")
    ap.add_argument("--dataset", default=None, help="directory with train/valid/test.txt + the two .dict files")
    ap.add_argument("--dataset-npz", default=None, help="the same data packed by scripts/pack_dataset.py")
    ap.add_argument("--member", nargs=2, action="append", default=[], metavar=("SETTINGS", "CHECKPOINT"),
                    help="a member's settings file and Model.save checkpoint; given exactly twice, A first")
    ap.add_argument("--weight", type=float, default=0.5, help="weight of member A in [0, 1] (B gets 1 - W); the "
                                                              "reference tool's value 0.5 by default")
    ap.add_argument("--split", choices=("test", "valid"), default="test")
    ap.add_argument("--limit", type=int, default=None, metavar="N", help="evaluate the first N triples of the split")
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args(argv)
    if (args.dataset is None) == (args.dataset_npz is None):
        ap.error("give exactly one of --dataset / --dataset-npz")
    if len(args.member) != 2:
        ap.error("give --member SETTINGS CHECKPOINT exactly twice (member A, then member B), got %d"
                 % len(args.member))
    try:
        args.weight = _check_weight(args.weight)
    except ValueError as e:
        ap.error(str(e))
    if args.limit is not None and args.limit < 1:
        ap.error("--limit must be positive, got %d" % args.limit)
    return args


def main(argv=None):
    from . import train as driver
    from .common import settings_reader
    args = parse_args(argv)
    if args.dataset_npz is not None:
        splits, entities, relations = driver.load_dataset_npz(args.dataset_npz)
    else:
        splits, entities, relations = driver.load_dataset(args.dataset)
    models, scorer = [], None
    for settings_path, checkpoint in args.member:
        _, model, member_scorer = driver.build_chain(settings_reader.read(settings_path), splits, len(entities),
                                                     len(relations), args.device)
        model.load(checkpoint)
        models.append(model)
        scorer = scorer or member_scorer   # every member registers the same splits
    triples = splits[args.split]
    if args.limit is not None:
        triples = triples[:args.limit]
    results = {}
    for key, title, model in (("a", "Member A", models[0]), ("b", "Member B", models[1]),
                              ("ensemble", "Ensemble (weight %g on A)" % args.weight,
                               Ensemble(models[0], models[1], args.weight))):
        scorer.register_model(model)
        summary = scorer.compute_scores(triples).get_summary()
        print(title)
        summary.pretty_print()
        results[key] = summary.results
    print(json.dumps({"weight": args.weight, "split": args.split, "triples": int(len(triples)), **results}))
    return results


if __name__ == "__main__":
    main()
