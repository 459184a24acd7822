"""CPU oracle for the basis layer with per-channel sigmoid coefficients (DiagonalCoefficients=Yes) -- TEST
INFRASTRUCTURE, NOT PRODUCT CODE.

Restates encoders/message_gcns/gcn_basis_times_diag.py of the reference (with message_gcn.py:49-79) in torch-CPU
(float64 capable), and the encoder chain model_builder.py:121-184 + :273-309 builds with it, on top of the
restatements of oracle/rgcn_oracle.py and tests/highway_oracle.py; backward is torch.autograd, standing in for
tf.gradients.  Pinned by tests/golden/reference_times_diag_golden.npz, the outputs of the reference's own classes
(tests/test_times_diag_cpu.py, 1e-10).  Line numbers cite code/encoders/message_gcns/gcn_basis_times_diag.py."""
import numpy as np
import torch

import highway_oracle as hw
from oracle import rgcn_oracle as oracle


def times_diag_forward(H, triples, W_forward, W_backward, C_forward, C_backward, W_self, b, norm_f, norm_b,
                       drop_mask=None, keep=1.0, use_nonlinearity=True, dtype=torch.float64):
    H = oracle._t(H, dtype)
    Vf, Vb, Ws = oracle._t(W_forward, dtype), oracle._t(W_backward, dtype), oracle._t(W_self, dtype)
    Cf, Cb, bb = oracle._t(C_forward, dtype), oracle._t(C_backward, dtype), oracle._t(b, dtype)
    s_idx, r_idx, o_idx = (torch.as_tensor(a.astype(np.int64)) for a in oracle.process_triples(triples))
    V, d = H.shape
    B = Vf.shape[1]
    # :47-52 compute_coefficients: sigmoid of the gathered [E, B, d] coefficient rows
    forward_type_scaling = torch.sigmoid(Cf[r_idx])
    backward_type_scaling = torch.sigmoid(Cb[r_idx])
    # :54-72 basis terms of the gathered sender / receiver rows, [E, B, d]
    sender_terms = (H[s_idx] @ Vf.reshape(Vf.shape[0], -1)).reshape(-1, B, Vf.shape[2])
    receiver_terms = (H[o_idx] @ Vb.reshape(Vb.shape[0], -1)).reshape(-1, B, Vb.shape[2])
    # :40-43
    forward_messages = (sender_terms * forward_type_scaling).sum(1)
    backward_messages = (receiver_terms * backward_type_scaling).sum(1)
    # message_gcn.py:57-64 self loop, dropout in train mode only
    self_loop = oracle.dropout_with_mask(H @ Ws, None if drop_mask is None else oracle._t(drop_mask, dtype), keep)
    # :79-87 two SpMMs, then the bias (added in this layer) and the nonlinearity
    cf = oracle.sparse_dense_matmul(o_idx, oracle._t(norm_f, dtype), forward_messages, V)
    cb = oracle.sparse_dense_matmul(s_idx, oracle._t(norm_b, dtype), backward_messages, V)
    new_embedding = self_loop + cf + cb + bb
    return torch.relu(new_embedding) if use_nonlinearity else new_embedding


def weight_names(n_layers, outproj, highway=False):
    """get_weights() order, deepest first: the input AffineTransform [W, b], per layer its six weights (followed by the
    highway [W, b] that wraps it), (the output AffineTransform [W, b],) RelationEmbedding."""
    per = ["W_forward", "W_backward", "C_forward", "C_backward", "W_self", "b"]
    names = ["W_in", "b_in"]
    for l in range(n_layers):
        names += ["L%d.%s" % (l, k) for k in per]
        if highway:
            names += ["HW%d.W" % l, "HW%d.b" % l]
    return names + (["W_out", "b_out"] if outproj else []) + ["W_relation"]


def encode(leaves, n_layers, outproj, highway, triples, V, mode, masks, keep, norm_mode, dtype=torch.float64,
           norm_dtype=np.float64):
    nf, nb = oracle.graph_norms(triples, V, norm_mode, norm_dtype)
    H = oracle.affine_onehot(leaves["W_in"], leaves["b_in"])
    for l in range(n_layers):
        lp = {k.split(".")[1]: v for k, v in leaves.items() if k.startswith("L%d." % l)}
        relu = l < n_layers - 1
        mask = masks[l] if mode == "train" else None
        k = keep if mode == "train" else 1.0
        L = times_diag_forward(H, triples, lp["W_forward"], lp["W_backward"], lp["C_forward"], lp["C_backward"],
                               lp["W_self"], lp["b"], nf, nb, mask, k, relu, dtype)
        H = hw.highway(L, H, leaves["HW%d.W" % l], leaves["HW%d.b" % l]) if highway else L
    if outproj:
        H = H @ leaves["W_out"] + leaves["b_out"]
    return H
