"""QuatE decoder (Zhang, Tay, Yao, Liu; NeurIPS 2019; DESIGN.md section 1).

Entity and relation rows are CodeDimension / 4 quaternions, interleaved: quaternion k of a row x is (x[4k], x[4k+1],
x[4k+2], x[4k+3]) = a + b i + c j + d k.  A relation quaternion is normalised, rh_k = r_k / max(|r_k|, 1e-12), and
rotates the subject: the energy of (s, r, o) is  E = sum_k <h_k (x) rh_k, t_k>  with h = codes[s], r = rel[r],
t = codes[o] and (x) the Hamilton product.  E is linear in each row, so QuatE has the whole surface of BilinearDiag on
the same scoring GEMMs: the NegativeSampling, SelfAdversarial and 1-N objectives with DistMult's L2 term on the raw
rows, filtered ranks, top-k and relation prediction (ops.QuatERanker).  The score matrices are float32 sigmoid(E).
There is no fused ensemble membership for QuatE; the decoder has no weights of its own."""
import torch

from .. import ops
from .bilinear_diag import BilinearDiag


class QuatE(BilinearDiag):
    ONE_TO_N = "quate"   # the decoder kind of ops.one_to_n_loss and ops.self_adversarial_loss
    # the ensemble's fused kernels score DistMult and ComplEx rows only
    ensemble_fused = False

    def __init__(self, dimension, settings, next_component=None):
        if dimension % 4:
            raise ValueError("the QuatE decoder needs CodeDimension %% 4 == 0, got %d" % dimension)
        self.dimension = dimension
        BilinearDiag.__init__(self, next_component, settings)

    def _score_op(self):
        return ops.quate_score

    def _ranker(self, codes, rel):
        return ops.QuatERanker(codes, rel, self.relation_count)

    def _relation_ranker(self):
        """ops.QuatERanker over the test-mode codes: its relation queries score the normalised rel[0:R]."""
        return self.test_ranker()

    def _all_scores(self, side):
        """float32 sigmoid(Q @ codes^T) [n, V] of the fed triples' query rows (ops.quate_query_rows)."""
        subject_codes, relation_codes, object_codes = self.next_component.get_all_codes(mode='test')
        assert subject_codes is object_codes, "QuatE scoring expects one shared entity code matrix"
        codes = subject_codes.contiguous()
        Q = ops.quate_query_rows(codes, relation_codes.contiguous(), self._x_device(), side)
        return torch.sigmoid(Q @ codes.T)

    def predict_all_subject_scores(self):
        """[n, V]: every entity as the subject, Q = t (x) conj(rh)."""
        return self._all_scores(0)

    def predict_all_object_scores(self):
        """[n, V]: every entity as the object, Q = h (x) rh."""
        return self._all_scores(1)
