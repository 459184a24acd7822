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
                                             [--relation-metrics]
                                             [--queries FILE --k K [--raw] --out FILE]

builds each member as the training driver does (train.build_chain), loads its Model.save checkpoint, and prints the
Raw / Filtered table of member A, of member B and of the ensemble (weight W on A, default 0.5 as in the reference
tool), then one JSON line with all three.  --relation-metrics adds the relation prediction tables (each triple's
relation ranked among all relations for its (head, tail) pair) of A, B and the ensemble, and their results under
"relations" in the JSON line.  With --queries the command evaluates nothing (so it refuses --split, --limit and
--relation-metrics): it answers the query file of
`python -m relationprediction_b200.predict` with the ensemble (same query format, --k, --raw and output lines; the
score is the combined score c = 1 - u of Ensemble.predict_top_k)."""
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
        # RelationCount: the relation candidates of relation prediction (members without one only rank entities)
        ra, rb = getattr(model_a, 'relation_count', None), getattr(model_b, 'relation_count', None)
        if ra is not None and rb is not None and int(ra) != int(rb):
            raise ValueError("the ensemble members must share one relation set, got %d and %d relations"
                             % (int(ra), int(rb)))
        self.a, self.b = model_a, model_b
        self.weight = _check_weight(weight)
        self.entity_count = ea
        self.relation_count = None if ra is None else int(ra)

    # ---- fused path (Scorer.compute_mrr_scores prefers it) ----
    def supports_fused_ranking(self):
        """Both members have a fused ranker (DistMult or ComplEx decoder) and live on the same CUDA device.  A RotatE
        member ranks by distance, which the ensemble's scoring GEMM cannot combine: its ranks come from the score
        matrices."""
        for m in (self.a, self.b):
            if not (hasattr(m, 'test_ranker') and getattr(m, 'ensemble_fused', True) and m.supports_fused_ranking()):
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

    # ---- top-k and relation prediction (fused only: Scorer.predict_top_k*, compute_relation_mrr_scores) ----
    def _fused_ranker(self, what, triplets):
        """ops.EnsembleRanker over both members' test codes (one encoder pass each), fed with `triplets`."""
        if not self.supports_fused_ranking():
            raise NotImplementedError("the ensemble has %s only through the fused path: both members need a DistMult "
                                      "or ComplEx decoder on the same CUDA device" % what)
        tri = triplets[:1]
        return ops.EnsembleRanker(self.a.entity_ranker(tri), self.b.entity_ranker(tri), self.weight)

    def _check_ids(self, triplets, relations):
        """Entity ids (columns 0 and 2) in [0, EntityCount), and relation ids (column 1) in [0, RelationCount) when
        `relations` is set."""
        if len(triplets):
            ent = triplets[:, [0, 2]]
            if ent.min() < 0 or ent.max() >= self.entity_count:
                raise ValueError("entity ids must be in [0, %d)" % self.entity_count)
            if relations and self.relation_count is not None and (triplets[:, 1].min() < 0 or
                                                                   triplets[:, 1].max() >= self.relation_count):
                raise ValueError("relation ids must be in [0, %d)" % self.relation_count)

    @staticmethod
    def _check_k(k):
        k = int(k)
        if not 1 <= k <= 128:
            raise ValueError("k must be in [1, 128], got %d" % k)
        return k

    @staticmethod
    def _chunked(ranker_fn, tri, lists, count, dev, chunk=4096):
        """ranker_fn(X, mask) over chunks of `chunk` triples, the mask built from lists[c0:c1] (or None), the
        results concatenated and copied to numpy."""
        from .decoders.bilinear_diag import BilinearDiag
        parts = []
        for c0 in range(0, len(tri), chunk):
            X = torch.as_tensor(tri[c0:c0 + chunk], device=dev)
            mask = None
            if lists is not None:
                mask = torch.as_tensor(BilinearDiag.known_bit_mask(lists[c0:c0 + chunk], count), device=dev)
            parts.append(ranker_fn(X, mask))
        return [torch.cat(p).cpu().numpy() for p in zip(*parts)] if parts else None

    @staticmethod
    def _top_k_out(res, k):
        if res is None:
            return np.zeros((0, k), np.int64), np.zeros((0, k)), np.zeros((0, k))
        ids, u, scores = res
        return ids.astype(np.int64), u, scores

    def predict_top_k(self, triplets, k, side, exclude_lists=None):
        """The k entities of best combined score for every triple (side 0 predicts subjects, 1 objects; the
        predicted column is not read but must hold an entity id), ordered by
          u = w sigma(-E_A) + (1 - w) sigma(-E_B)   ascending (double, sigma(-E) = 1 / (1 + exp(E))),
        the smaller id first on ties: the c-descending order without the saturation of the float32 sigmoid, so in
        saturated cases an entity's position here can differ from its rank.  exclude_lists[t] (optional) lists the
        entities row t may not return.  Returns numpy (ids int64 [n, k], u float64 [n, k], scores = 1 - u float64
        [n, k]); rows with fewer than k eligible entities end in id -1, u +inf, score 0."""
        k, side = self._check_k(k), int(side)
        if side not in (0, 1):
            raise ValueError("side must be 0 (predict subjects) or 1 (predict objects), got %r" % (side,))
        tri = np.ascontiguousarray(np.asarray(triplets, dtype=np.int32).reshape(-1, 3))
        self._check_ids(tri, relations=True)
        ranker = self._fused_ranker("top-k prediction", tri)
        with torch.no_grad():
            res = self._chunked(lambda X, m: ranker.top_k(X, side, k, m), tri, exclude_lists, self.entity_count,
                                ranker.a.codes.device)
        return self._top_k_out(res, k)

    def predict_top_k_relations(self, triplets, k, exclude_lists=None):
        """The k relations of best combined score for every (head, ?, tail) pair of `triplets` (the relation column
        is not read), in predict_top_k's order.  exclude_lists[t] (optional) lists the relations row t may not
        return.  Returns numpy (ids int64 [n, k], u float64 [n, k], scores = 1 - u float64 [n, k]); rows with fewer
        than k eligible relations end in id -1, u +inf, score 0."""
        k = self._check_k(k)
        tri = np.ascontiguousarray(np.asarray(triplets, dtype=np.int32).reshape(-1, 3))
        self._check_ids(tri, relations=False)
        ranker = self._fused_ranker("relation prediction", tri)
        with torch.no_grad():
            res = self._chunked(lambda X, m: ranker.top_k_relations(X, k, m), tri, exclude_lists,
                                self.relation_count, ranker.a.codes.device)
        return self._top_k_out(res, k)

    def rank_all_relations(self, triplets, known_relation_lists):
        """Ranks of every triple's relation among the RelationCount relations for its (head, tail) pair under the
        combined score, raw and filtered by known_relation_lists[t] with the entity ranks' rules.  Returns numpy
        (raw, filtered) int64 [n]."""
        tri = np.ascontiguousarray(np.asarray(triplets, dtype=np.int32).reshape(-1, 3))
        self._check_ids(tri, relations=True)
        ranker = self._fused_ranker("relation prediction", tri)
        with torch.no_grad():
            res = self._chunked(lambda X, m: ranker.rank_relations(X, m), tri, known_relation_lists,
                                self.relation_count, ranker.a.codes.device)
        if res is None:
            return np.zeros(0, np.int64), np.zeros(0, np.int64)
        return res[0].astype(np.int64), res[1].astype(np.int64)

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
    ap.add_argument("--split", choices=("test", "valid"), default=None, help="the split to evaluate (default test)")
    ap.add_argument("--limit", type=int, default=None, metavar="N", help="evaluate the first N triples of the split")
    ap.add_argument("--device", default="cuda:0")
    ap.add_argument("--relation-metrics", action="store_true",
                    help="also rank every triple's relation among all relations for its (head, tail) pair")
    ap.add_argument("--queries", default=None, help="answer this query file instead of evaluating: one query per "
                                                    "line, head<TAB>relation<TAB>?, ?<TAB>relation<TAB>tail or "
                                                    "head<TAB>?<TAB>tail (the predict command's format)")
    ap.add_argument("--k", type=int, default=None, help="answers per query, 1 <= K <= 128 (with --queries)")
    ap.add_argument("--raw", action="store_true", help="keep entities (relations) that complete a known triple "
                                                       "(with --queries)")
    ap.add_argument("--out", default=None, help="output file of --queries: query_index<TAB>position<TAB>answer"
                                                "<TAB>score")
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
    if args.queries is None:
        for flag, value in (("--k", args.k), ("--out", args.out)):
            if value is not None:
                ap.error("%s goes with --queries" % flag)
        if args.raw:
            ap.error("--raw goes with --queries")
    else:
        if args.k is None or args.out is None:
            ap.error("--queries needs --k K and --out FILE")
        if not 1 <= args.k <= 128:
            ap.error("--k must be in [1, 128], got %d" % args.k)
        for flag, given in (("--relation-metrics", args.relation_metrics), ("--split", args.split is not None),
                            ("--limit", args.limit is not None)):
            if given:
                ap.error("%s evaluates a split; --queries answers queries: give one of them" % flag)
    if args.split is None:
        args.split = "test"
    return args


def _names(args, entities, relations):
    """(entity name -> id, relation name -> id, entity name of id, relation name of id) as the predict command
    makes them: numeric ids for --dataset-npz."""
    if args.dataset_npz is not None:
        return {str(i): i for i in entities}, {str(i): i for i in relations}, str, str
    return ({v: i for i, v in entities.items()}, {v: i for i, v in relations.items()}, entities.__getitem__,
            relations.__getitem__)


def main(argv=None):
    from . import predict
    from . import train as driver
    from .common import settings_reader
    args = parse_args(argv)
    if args.dataset_npz is not None:
        splits, entities, relations = driver.load_dataset_npz(args.dataset_npz)
    else:
        splits, entities, relations = driver.load_dataset(args.dataset)
    queries = None
    if args.queries is not None:   # read before the models are built: a bad file fails fast
        ent_names, rel_names, name_of, rel_name_of = _names(args, entities, relations)
        with open(args.queries) as fh:
            try:
                queries = predict.parse_queries(fh, ent_names, rel_names)
            except predict.QueryError as e:
                raise SystemExit("%s: %s" % (args.queries, e))
    models, scorer = [], None
    for settings_path, checkpoint in args.member:
        _, model, member_scorer = driver.build_chain(settings_reader.read(settings_path), splits, len(entities),
                                                     len(relations), args.device)
        model.load(checkpoint)
        models.append(model)
        scorer = scorer or member_scorer   # every member registers the same splits
    ensemble = Ensemble(models[0], models[1], args.weight)
    if queries is not None:
        scorer.register_model(ensemble)
        rows = predict.answer(scorer, queries, args.k, filtered=not args.raw)
        with open(args.out, "w") as fh:
            for qi, pos, ans, score in rows:
                name = rel_name_of(ans) if queries[qi][3] == 2 else name_of(ans)
                fh.write("%d\t%d\t%s\t%.9g\n" % (qi, pos, name, score))
        return rows
    triples = splits[args.split]
    if args.limit is not None:
        triples = triples[:args.limit]
    results, relation_results = {}, {}
    members = (("a", "Member A", models[0]), ("b", "Member B", models[1]),
               ("ensemble", "Ensemble (weight %g on A)" % args.weight, ensemble))
    for key, title, model in members:
        scorer.register_model(model)
        summary = scorer.compute_scores(triples).get_summary()
        print(title)
        summary.pretty_print()
        results[key] = summary.results
    if args.relation_metrics:
        for key, title, model in members:
            scorer.register_model(model)
            summary = scorer.compute_relation_mrr_scores(triples).get_summary()
            print(title + ", relation prediction")
            summary.pretty_print()
            relation_results[key] = summary.results
    line = {"weight": args.weight, "split": args.split, "triples": int(len(triples)), **results}
    if args.relation_metrics:
        line["relations"] = relation_results
        results["relations"] = relation_results
    print(json.dumps(line))
    return results


if __name__ == "__main__":
    main()
