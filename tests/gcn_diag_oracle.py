"""CPU oracle for the diagonal R-GCN encoder (Encoder Name=gcn_diag) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates encoders/message_gcns/gcn_diag.py of the reference (with message_gcn.py:49-79, the `tf.mul` of :35-36 read
as the element-wise product) and the encoder chain model_builder.py:71-119 builds with it, in torch-CPU (float64
capable), on top of the restatements of oracle/rgcn_oracle.py; backward is torch.autograd, standing in for
tf.gradients.  Pinned by tests/golden/reference_gcn_diag_golden.npz, the outputs of the reference's own classes
(tests/test_gcn_diag_cpu.py, 1e-10).  Line numbers cite code/encoders/message_gcns/gcn_diag.py."""
import numpy as np
import torch

from oracle import rgcn_oracle as oracle


def diag_forward(H, triples, D_forward, D_backward, W_self, b, norm_f, norm_b, drop_mask=None, keep=1.0,
                 use_nonlinearity=True, dtype=torch.float64):
    H = oracle._t(H, dtype)
    Df, Db, Ws, bb = (oracle._t(x, dtype) for x in (D_forward, D_backward, W_self, b))
    s_idx, r_idx, o_idx = (torch.as_tensor(a.astype(np.int64)) for a in oracle.process_triples(triples))
    V = H.shape[0]
    # :31-38 per-message diagonals gathered by relation, element-wise products with the sender / receiver rows
    forward_messages = H[s_idx] * Df[r_idx]
    backward_messages = H[o_idx] * Db[r_idx]
    # message_gcn.py:57-64 self loop, dropout in train mode only
    self_loop = oracle.dropout_with_mask(H @ Ws, None if drop_mask is None else oracle._t(drop_mask, dtype), keep)
    # :42-55 two SpMMs, then the bias (added in this layer) and the nonlinearity
    cf = oracle.sparse_dense_matmul(o_idx, oracle._t(norm_f, dtype), forward_messages, V)
    cb = oracle.sparse_dense_matmul(s_idx, oracle._t(norm_b, dtype), backward_messages, V)
    new_embedding = self_loop + cf + cb + bb
    return torch.relu(new_embedding) if use_nonlinearity else new_embedding


def weight_names(n_layers, outproj):
    """get_weights() order, deepest first: the input AffineTransform [W, b], per layer [D_types_forward,
    D_types_backward, W_self, b] (:26-28), (the output AffineTransform [W, b],) RelationEmbedding."""
    names = ["W_in", "b_in"]
    for l in range(n_layers):
        names += ["L%d.%s" % (l, k) for k in ("D_types_forward", "D_types_backward", "W_self", "b")]
    return names + (["W_out", "b_out"] if outproj else []) + ["W_relation"]


def encode(leaves, n_layers, outproj, triples, V, mode, masks, keep, norm_mode, dtype=torch.float64,
           norm_dtype=np.float64):
    nf, nb = oracle.graph_norms(triples, V, norm_mode, norm_dtype)
    H = oracle.affine_onehot(leaves["W_in"], leaves["b_in"])      # model_builder.py:89-94: always, bias + ReLU
    for l in range(n_layers):
        lp = {k.split(".")[1]: v for k, v in leaves.items() if k.startswith("L%d." % l)}
        H = diag_forward(H, triples, lp["D_types_forward"], lp["D_types_backward"], lp["W_self"], lp["b"], nf, nb,
                         masks[l] if mode == "train" else None, keep if mode == "train" else 1.0, l < n_layers - 1,
                         dtype)
    if outproj:
        H = H @ leaves["W_out"] + leaves["b_out"]
    return H
