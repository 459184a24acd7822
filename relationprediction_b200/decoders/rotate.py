"""RotatE decoder (Sun et al., ICLR 2019; DESIGN.md section 1).

Entity rows are complex vectors [re | im] of h = CodeDimension / 2 columns each, as for ComplEx; a relation rotates
them: the first h columns of its row are the phases theta (radians), the other h are never read.  The energy of
(s, r, o) is  E = gamma - sum_k |a_k e^{i theta_k} - c_k|  with a = codes[s], c = codes[o] and gamma the `Margin` key
of [Decoder] (default 12).  Same plugin protocol, placeholders, caches and objectives (NegativeSampling,
SelfAdversarial) as BilinearDiag; the scorer is ops.rotate_score, the all-entity ranking ops.RotateRanker (by
distance), and the score matrices are float32 sigmoid(E).  There is no top-k, relation prediction, 1-N training or
fused ensemble membership for RotatE."""
import math

import torch

from .. import ops
from .bilinear_diag import BilinearDiag

DEFAULT_MARGIN = 12.0


def parse_margin(settings):
    """Margin gamma of [Decoder] (default 12): any finite float."""
    gamma = float(settings['Margin']) if 'Margin' in settings else DEFAULT_MARGIN
    if not math.isfinite(gamma):
        raise ValueError("Margin must be finite, got %r" % (gamma,))
    return gamma


class Rotate(BilinearDiag):
    ONE_TO_N = "rotate"
    # ranks by distance: the ensemble's fused kernel combines scoring-GEMM members only
    ensemble_fused = False

    def __init__(self, dimension, settings, next_component=None):
        if dimension % 4:
            raise ValueError("the RotatE decoder needs CodeDimension %% 4 == 0, got %d" % dimension)
        self.dimension = dimension
        BilinearDiag.__init__(self, next_component, settings)

    def parse_settings(self):
        BilinearDiag.parse_settings(self)
        self.margin = parse_margin(self.settings)

    def _score_op(self):
        return lambda codes, rel, X, Y: ops.rotate_score(codes, rel, X, Y, gamma=self.margin)

    def _self_adversarial_args(self):
        return {'gamma': self.margin}

    def _ranker(self, codes, rel):
        return ops.RotateRanker(codes, rel, self.relation_count)

    def _all_scores(self, queries, candidates):
        """float32 sigmoid(gamma - D) [n, V] of the query rows q [n, d] against every candidate row, D summed over k."""
        h = self.dimension // 2
        D = torch.zeros((queries.shape[0], candidates.shape[0]), dtype=queries.dtype, device=queries.device)
        for k in range(h):
            D += torch.hypot(queries[:, k, None] - candidates[None, :, k],
                             queries[:, h + k, None] - candidates[None, :, h + k])
        return torch.sigmoid(self.margin - D)

    def _rotated(self, x, theta):
        """x e^{i theta} for rows x [n, d] and phases theta [n, h]."""
        h = self.dimension // 2
        cs, sn = torch.cos(theta), torch.sin(theta)
        return torch.cat([x[:, :h] * cs - x[:, h:2 * h] * sn, x[:, :h] * sn + x[:, h:2 * h] * cs], 1)

    def predict_all_subject_scores(self):
        """[n, V]: every entity as the subject, q = c e^{-i theta} (|a e^{i theta} - c| = |a - c e^{-i theta}|)."""
        e1s, rs, e2s = self.compute_codes(mode='test')
        all_subject_codes = self.next_component.get_all_subject_codes(mode='test')
        return self._all_scores(self._rotated(e2s, -rs[:, :self.dimension // 2]), all_subject_codes)

    def predict_all_object_scores(self):
        """[n, V]: every entity as the object, q = a e^{i theta}."""
        e1s, rs, e2s = self.compute_codes(mode='test')
        all_object_codes = self.next_component.get_all_object_codes(mode='test')
        return self._all_scores(self._rotated(e1s, rs[:, :self.dimension // 2]), all_object_codes)
