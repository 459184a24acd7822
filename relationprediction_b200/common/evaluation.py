"""Link-prediction evaluation: raw and filtered MRR, Hits@1/3/10 (next-row N3, SURVEY.md 8f).

Ranking rules restated from the reference (common/evaluation.py:148-152, :334-386):
  raw rank      = #{entities whose score >= score of the gold entity}
  filtered rank = raw rank - #{KNOWN true entities whose score >= gold score} + 1
with the known sets built from every registered split (train.py:103-105), both corruption directions
(subjects then objects) per triple, in chunks of 1000 triples.  Per-degree / per-frequency breakdowns
of the reference are not reproduced."""
import math

import numpy as np


class MrrSummary(object):
    def __init__(self, raw_ranks, filtered_ranks):
        self.results = {'Raw': self._stats(np.asarray(raw_ranks, dtype=np.float64)),
                        'Filtered': self._stats(np.asarray(filtered_ranks, dtype=np.float64))}

    @staticmethod
    def _stats(ranks):
        return {'MRR': float(np.mean(1.0 / ranks)) if len(ranks) else 0.0,
                'H@1': float(np.mean(ranks <= 1)) if len(ranks) else 0.0,
                'H@3': float(np.mean(ranks <= 3)) if len(ranks) else 0.0,
                'H@10': float(np.mean(ranks <= 10)) if len(ranks) else 0.0}

    def mrr_string(self):
        return 'MRR'

    def pretty_print(self):
        print('\tRaw\tFiltered')   # same table as the reference (common/evaluation.py:74-84)
        for item in ('MRR', 'H@1', 'H@3', 'H@10'):
            print("%s\t%s\t%s" % (item, round(self.results['Raw'][item], 3), round(self.results['Filtered'][item], 3)))


class MrrScore(object):
    def __init__(self):
        self.raw_ranks, self.filtered_ranks = [], []

    def append_rows(self, scores, gold_idx, known_lists):
        gold = scores[np.arange(scores.shape[0]), gold_idx]
        raw = (scores >= gold[:, None]).sum(1)
        known_ge = np.array([int((scores[i, k] >= gold[i]).sum()) for i, k in enumerate(known_lists)])
        self.raw_ranks.extend(raw.tolist())
        self.filtered_ranks.extend((raw - known_ge + 1).tolist())

    def get_summary(self):
        return MrrSummary(self.raw_ranks, self.filtered_ranks)


class Scorer(object):
    def __init__(self, settings=None):
        self.settings = settings
        self.known_object_triples = {}
        self.known_subject_triples = {}
        self.known_relation_triples = {}
        self.model = None

    def register_data(self, triples):
        # de-duplicated lists, like extend_triple_dict (common/evaluation.py:232-245); known_relation_triples[(s, o)]
        # lists the relations linking s to o, for the relation queries (s, ?, o)
        for s, r, o in np.asarray(triples).reshape(-1, 3).tolist():
            lo = self.known_object_triples.setdefault((s, r), [])
            if o not in lo:
                lo.append(o)
            ls = self.known_subject_triples.setdefault((o, r), [])
            if s not in ls:
                ls.append(s)
            lr = self.known_relation_triples.setdefault((s, o), [])
            if r not in lr:
                lr.append(r)

    def register_degrees(self, triples):  # kept for call compatibility (train.py:106); unused here
        pass

    def finalize_frequency_computation(self, triples):
        pass

    def register_model(self, model):
        self.model = model

    def predict_top_k(self, triples, k, side, filtered=True):
        """The k most likely entities for each triple through the model's fused top-k path (Model.predict_top_k):
        side 0 predicts subjects, 1 objects.  filtered=True leaves out every entity that completes a triple of any
        registered split -- the known_subject_triples / known_object_triples lists the filtered ranks use -- so only
        new answers come back; filtered=False excludes nothing.  Returns numpy (ids, energies, scores), each [n, k]."""
        triples = np.asarray(triples).reshape(-1, 3)
        exclude = None
        if filtered:
            tl = triples.tolist()
            if int(side) == 0:
                exclude = [self.known_subject_triples.get((t[2], t[1]), []) for t in tl]
            else:
                exclude = [self.known_object_triples.get((t[0], t[1]), []) for t in tl]
        return self.model.predict_top_k(triples, k, side, exclude)

    def predict_top_k_relations(self, triples, k, filtered=True):
        """The k most likely relations for each (s, ?, o) pair of `triples` through the model's fused path
        (Model.predict_top_k_relations; the relation column is not read).  filtered=True leaves out every relation
        r with (s, r, o) in a registered split (known_relation_triples); filtered=False excludes nothing.  Returns
        numpy (ids, energies, scores), each [n, k]."""
        triples = np.asarray(triples).reshape(-1, 3)
        exclude = None
        if filtered:
            exclude = [self.known_relation_triples.get((t[0], t[2]), []) for t in triples.tolist()]
        return self.model.predict_top_k_relations(triples, k, exclude)

    def compute_relation_mrr_scores(self, triples):
        """Relation prediction metrics: each triple's relation ranked among all relations for its (s, o) pair by
        the model's fused relation ranker, raw and filtered by known_relation_triples with the entity ranks' rules.
        Returns an MrrScore (one rank per triple) whose summary prints the same Raw / Filtered table."""
        triples = np.asarray(triples).reshape(-1, 3)
        score = MrrScore()
        known = [self.known_relation_triples.get((t[0], t[2]), []) for t in triples.tolist()]
        raw, filt = self.model.rank_all_relations(triples, known)
        score.raw_ranks.extend(np.asarray(raw).tolist())
        score.filtered_ranks.extend(np.asarray(filt).tolist())
        return score

    def compute_scores(self, triples, verbose=False):
        return self.compute_mrr_scores(triples, verbose)

    def compute_mrr_scores(self, triples, verbose=False):
        triples = np.asarray(triples).reshape(-1, 3)
        score = MrrScore()
        # GPU models rank inside the scoring GEMM (distmult_rank): same counting rules, no [chunk, V] matrices, one
        # encoder pass.  The interleaving of the reference (subjects then objects per triple chunk) only orders the
        # rank lists; every summary statistic is a mean over them.
        fused = getattr(self.model, 'rank_all_entities', None)
        if fused is not None and getattr(self.model, 'supports_fused_ranking', lambda: False)():
            tl = triples.tolist()
            ks = [self.known_subject_triples.get((t[2], t[1]), []) for t in tl]
            ko = [self.known_object_triples.get((t[0], t[1]), []) for t in tl]
            res = fused(triples, ks, ko)
            if res is not None:
                raw_s, filt_s, raw_o, filt_o = res
                score.raw_ranks.extend(raw_s.tolist() + raw_o.tolist())
                score.filtered_ranks.extend(filt_s.tolist() + filt_o.tolist())
                return score
        chunk = 1000
        for c in range(math.ceil(len(triples) / chunk)):
            part = triples[c * chunk:(c + 1) * chunk]
            pred_s = self.model.score_all_subjects(part)
            score.append_rows(pred_s, part[:, 0],
                              [np.asarray(self.known_subject_triples.get((t[2], t[1]), []), dtype=np.int64) for t in part.tolist()])
            pred_o = self.model.score_all_objects(part)
            score.append_rows(pred_o, part[:, 2],
                              [np.asarray(self.known_object_triples.get((t[0], t[1]), []), dtype=np.int64) for t in part.tolist()])
        return score
