"""ComplEx decoder (reference: decoders/complex.py).

Same plugin protocol, placeholders, per-instance caches and fused paths as BilinearDiag; only the scorer
(ops.complex_score), the ranker (ops.ComplexRanker) and the all-entity score matrices differ.  Unlike the reference,
whose `encoder_cache` is a class-level dict (complex.py:9), every instance keeps its own cache."""
import torch

from .. import ops
from .bilinear_diag import BilinearDiag


class Complex(BilinearDiag):
    ONE_TO_N = "complex"

    def __init__(self, dimension, settings, next_component=None):
        BilinearDiag.__init__(self, next_component, settings)
        self.dimension = dimension

    def _score_op(self):
        return ops.complex_score   # energies (:38-41), reduce_mean(weighted CE, pos_weight 1) (:43-45), L2 (:108-114)

    def _ranker(self, codes, rel):
        return ops.ComplexRanker(codes, rel, self.relation_count)

    def extract_real_and_imaginary(self, composite_vector):
        """(:71-75) columns [0, h) and [h, 2h) with h = int(dimension / 2)."""
        h = int(self.dimension / 2)
        return composite_vector[:, :h], composite_vector[:, h:2 * h]

    def predict_all_subject_scores(self):
        """(:77-91) sigmoid(all_subject_codes @ Q_s^T)^T, [n, V]."""
        e1s, rs, e2s = self.compute_codes(mode='test')
        all_subject_codes = self.next_component.get_all_subject_codes(mode='test')
        e1s_r, e1s_i = self.extract_real_and_imaginary(all_subject_codes)
        e2s_r, e2s_i = self.extract_real_and_imaginary(e2s)
        rs_r, rs_i = self.extract_real_and_imaginary(rs)
        all_energies = e1s_r @ (rs_r * e2s_r).T + e1s_i @ (rs_r * e2s_i).T \
            + e1s_r @ (rs_i * e2s_i).T - e1s_i @ (rs_i * e2s_r).T
        return torch.sigmoid(all_energies.T)

    def predict_all_object_scores(self):
        """(:93-106) sigmoid(Q_o @ all_object_codes^T), [n, V]."""
        e1s, rs, e2s = self.compute_codes(mode='test')
        all_object_codes = self.next_component.get_all_object_codes(mode='test')
        e1s_r, e1s_i = self.extract_real_and_imaginary(e1s)
        e2s_r, e2s_i = self.extract_real_and_imaginary(all_object_codes)
        rs_r, rs_i = self.extract_real_and_imaginary(rs)
        all_energies = (e1s_r * rs_r) @ e2s_r.T + (e1s_i * rs_r) @ e2s_i.T \
            + (e1s_r * rs_i) @ e2s_i.T - (e1s_i * rs_i) @ e2s_r.T
        return torch.sigmoid(all_energies)
