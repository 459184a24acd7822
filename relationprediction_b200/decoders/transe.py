"""TransE decoder (Bordes et al., NIPS 2013) with the L1 distance (DESIGN.md section 1).

Entity and relation rows are plain real vectors of CodeDimension columns; a relation translates the subject: the
energy of (s, r, o) is  E = gamma - sum_k |h_k + r_k - t_k|  with h = codes[s], r = rel[r], t = codes[o] and gamma the
`Margin` key of [Decoder] (default 12).  Same plugin protocol, placeholders, caches and objectives (NegativeSampling,
SelfAdversarial) as BilinearDiag; the scorer is ops.transe_score, and every query -- subjects, objects or relations,
ranks or top-k -- is ops.TransERanker, by distance.  The score matrices are float32 sigmoid(E).  There is no 1-N
training or fused ensemble membership for TransE."""
import torch

from .. import ops
from .bilinear_diag import BilinearDiag
from .rotate import parse_margin


class TransE(BilinearDiag):
    ONE_TO_N = "transe"   # the decoder kind of ops.self_adversarial_loss (TransE has no 1-N objective)
    # ranks by distance: the ensemble's fused kernel combines scoring-GEMM members only
    ensemble_fused = False

    def __init__(self, dimension, settings, next_component=None):
        if dimension % 4:
            raise ValueError("the TransE decoder needs CodeDimension %% 4 == 0, got %d" % dimension)
        self.dimension = dimension
        BilinearDiag.__init__(self, next_component, settings)

    def parse_settings(self):
        BilinearDiag.parse_settings(self)
        self.margin = parse_margin(self.settings)

    def _score_op(self):
        return lambda codes, rel, X, Y: ops.transe_score(codes, rel, X, Y, gamma=self.margin)

    def _self_adversarial_args(self):
        return {'gamma': self.margin}

    def _ranker(self, codes, rel):
        return ops.TransERanker(codes, rel, self.relation_count, gamma=self.margin)

    def _all_scores(self, queries, candidates):
        """float32 sigmoid(gamma - D) [n, V] of the query rows q [n, d] against every candidate row, D = sum_k |q - v|
        summed over k."""
        D = torch.zeros((queries.shape[0], candidates.shape[0]), dtype=queries.dtype, device=queries.device)
        for k in range(self.dimension):
            D += (queries[:, k, None] - candidates[None, :, k]).abs()
        return torch.sigmoid(self.margin - D)

    def predict_all_subject_scores(self):
        """[n, V]: every entity as the subject, q = t - r (|v + r - t| = |v - (t - r)|)."""
        e1s, rs, e2s = self.compute_codes(mode='test')
        all_subject_codes = self.next_component.get_all_subject_codes(mode='test')
        return self._all_scores(e2s - rs, all_subject_codes)

    def predict_all_object_scores(self):
        """[n, V]: every entity as the object, q = h + r."""
        e1s, rs, e2s = self.compute_codes(mode='test')
        all_object_codes = self.next_component.get_all_object_codes(mode='test')
        return self._all_scores(e1s + rs, all_object_codes)
