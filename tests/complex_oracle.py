"""CPU oracle for the ComplEx decoder -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates decoders/complex.py of the reference op for op in torch-CPU (float64 capable); backward is
torch.autograd over the restated forward, standing in for tf.gradients.  It builds on the shared helpers of
oracle/rgcn_oracle.py (dtype conversion, the TF weighted cross-entropy) and is pinned by
tests/golden/reference_complex_golden.npz, the outputs of the reference's own Complex class
(tests/test_complex_cpu.py, 1e-10).  Line numbers cite code/decoders/complex.py."""
import numpy as np
import torch

from oracle.rgcn_oracle import _t, weighted_cross_entropy_with_logits


def complex_real_and_imaginary(x, d):
    """extract_real_and_imaginary (:71-75): columns [0, h) and [h, 2h), h = int(d / 2)."""
    h = int(d / 2)
    return x[:, :h], x[:, h:2 * h]


def complex_energies(codes, rel, X, dtype=torch.float32):
    """Energies (:38-41) and the gathered rows (:22-25)."""
    codes, rel = _t(codes, dtype), _t(rel, dtype)
    X = torch.as_tensor(np.asarray(X).astype(np.int64)) if not isinstance(X, torch.Tensor) else X.long()
    e1s, rs, e2s = codes[X[:, 0]], rel[X[:, 1]], codes[X[:, 2]]
    d = codes.shape[1]
    e1s_r, e1s_i = complex_real_and_imaginary(e1s, d)
    e2s_r, e2s_i = complex_real_and_imaginary(e2s, d)
    rs_r, rs_i = complex_real_and_imaginary(rs, d)
    energies = (e1s_r * rs_r * e2s_r).sum(1) + (e1s_i * rs_r * e2s_i).sum(1) \
        + (e1s_r * rs_i * e2s_i).sum(1) - (e1s_i * rs_i * e2s_r).sum(1)
    return energies, (e1s, rs, e2s)


def complex_loss(codes, rel, X, Y, dtype=torch.float32):
    """Returns (loss, reg_unscaled, energies): loss = reduce_mean(weighted CE, pos_weight forced to 1) (:43-45);
    reg = mean(e1^2) + mean(r^2) + mean(e2^2) over the gathered rows, all d columns (:108-114)."""
    energies, (e1s, rs, e2s) = complex_energies(codes, rel, X, dtype)
    loss = weighted_cross_entropy_with_logits(_t(Y, dtype), energies, 1).mean()
    reg = (e1s ** 2).mean() + (rs ** 2).mean() + (e2s ** 2).mean()
    return loss, reg, energies


def complex_predict_all_objects(codes, rel, X, dtype=torch.float32):
    """predict_all_object_scores (:93-106): [n, V]."""
    _, (e1s, rs, _) = complex_energies(codes, rel, X, dtype)
    c = _t(codes, dtype)
    d = c.shape[1]
    e1s_r, e1s_i = complex_real_and_imaginary(e1s, d)
    e2s_r, e2s_i = complex_real_and_imaginary(c, d)
    rs_r, rs_i = complex_real_and_imaginary(rs, d)
    return torch.sigmoid((e1s_r * rs_r) @ e2s_r.T + (e1s_i * rs_r) @ e2s_i.T
                         + (e1s_r * rs_i) @ e2s_i.T - (e1s_i * rs_i) @ e2s_r.T)


def complex_predict_all_subjects(codes, rel, X, dtype=torch.float32):
    """predict_all_subject_scores (:77-91): [n, V]."""
    _, (_, rs, e2s) = complex_energies(codes, rel, X, dtype)
    c = _t(codes, dtype)
    d = c.shape[1]
    e1s_r, e1s_i = complex_real_and_imaginary(c, d)
    e2s_r, e2s_i = complex_real_and_imaginary(e2s, d)
    rs_r, rs_i = complex_real_and_imaginary(rs, d)
    return torch.sigmoid((e1s_r @ (rs_r * e2s_r).T + e1s_i @ (rs_r * e2s_i).T
                          + e1s_r @ (rs_i * e2s_i).T - e1s_i @ (rs_i * e2s_r).T).T)
