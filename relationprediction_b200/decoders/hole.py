"""HolE decoder (Nickel, Rosasco, Poggio; AAAI 2016; DESIGN.md section 1).

Entity and relation rows are real vectors of CodeDimension d (d % 4 == 0).  The energy of (s, r, o) is the circular
correlation of the subject and object rows read by the relation row:  E = sum_k r_k [h * t]_k  with
[h * t]_k = sum_i h_i t_{(i + k) mod d}, h = codes[s], r = rel[r], t = codes[o].  Written out that is O(d^2) per triple;
the decoder instead moves both tables once per mode into the orthonormal real Fourier basis (ops.hole_transform, one
GEMM each), where the energy is a ComplEx-type product that costs O(d) per triple and query.  E is linear in each row,
so HolE has the whole surface of BilinearDiag on the same scoring GEMMs: the NegativeSampling, SelfAdversarial and 1-N
objectives with DistMult's L2 term (the basis is orthogonal, so it is the raw rows' term), filtered ranks, top-k and
relation prediction (ops.HolERanker).  The score matrices are float32 sigmoid(E).

Not built: the paper's pairwise margin loss and its unit-norm constraint on entity rows, and fused ensemble
membership.  The decoder has no weights of its own."""
import torch

from .. import ops
from .bilinear_diag import BilinearDiag


class HolE(BilinearDiag):
    ONE_TO_N = "hole"   # the decoder kind of ops.one_to_n_loss and ops.self_adversarial_loss
    # the ensemble's fused kernels score DistMult and ComplEx rows only
    ensemble_fused = False

    def __init__(self, dimension, settings, next_component=None):
        if dimension % 4:
            raise ValueError("the HolE decoder needs CodeDimension %% 4 == 0, got %d" % dimension)
        self.dimension = dimension
        self._transformed = {'train': None, 'test': None}
        BilinearDiag.__init__(self, next_component, settings)

    def local_clear_cache(self):
        BilinearDiag.local_clear_cache(self)
        self._transformed = {'train': None, 'test': None}

    def _all_codes(self, mode):
        """The encoder's entity table and its first RelationCount relation rows in the HolE basis, transformed once per
        mode and feed.  The other rows of the relation table (the R-GCN encoders keep EntityCount of them) are never
        scored, so they are not transformed."""
        if self._transformed[mode] is None:
            subject_codes, relation_codes, object_codes = self.next_component.get_all_codes(mode=mode)
            assert subject_codes is object_codes, "HolE scoring expects one shared entity code matrix"
            codes = ops.hole_transform(subject_codes.contiguous())
            rel = ops.hole_transform(relation_codes[:self.relation_count].contiguous())
            self._transformed[mode] = (codes, rel, codes)
        return self._transformed[mode]

    def _score_op(self):
        return ops.hole_score

    def _ranker(self, codes, rel):
        return ops.HolERanker(codes, rel, self.relation_count)

    def _all_scores(self, side):
        """float32 sigmoid(Q @ codes~^T) [n, V] of the fed triples' query rows (ops.hole_query_rows)."""
        codes, relation_codes, _ = self._all_codes('test')
        Q = ops.hole_query_rows(codes, relation_codes, self._x_device(), side)
        return torch.sigmoid(Q @ codes.T)

    def predict_all_subject_scores(self):
        """[n, V]: every entity as the subject, Q = w conj(r~) t~."""
        return self._all_scores(0)

    def predict_all_object_scores(self):
        """[n, V]: every entity as the object, Q = w (h~ r~)."""
        return self._all_scores(1)
