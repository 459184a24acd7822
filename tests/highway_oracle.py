"""CPU oracle for the highway skip connection -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates extras/highway_layer.py of the reference in torch-CPU (float64 capable) and the encoder chain that
model_builder.py:273-309 builds with SkipConnections=Highway, on top of the layer restatements of
oracle/rgcn_oracle.py; backward is torch.autograd, standing in for tf.gradients.  Pinned by
tests/golden/reference_highway_golden.npz, the outputs of the reference's own classes (tests/test_highway_cpu.py,
1e-10).  Line numbers cite code/extras/highway_layer.py and code/common/model_builder.py."""
import numpy as np
import torch

from oracle import rgcn_oracle as oracle


def highway(c1, c2, W, b):
    """compute_vertex_embeddings / get_gates (:14-38): g = sigmoid(c2 W + b), g c1 + (1 - g) c2."""
    g = torch.sigmoid(c2 @ W + b)
    return g * c1 + (1 - g) * c2


def weight_names(variant, n_layers, outproj):
    """get_weights() order, deepest first: (AffineTransform [W, b],) then per layer its weights followed by the
    highway [W, b] that wraps it (a one-hot layer 0 is not wrapped), (output AffineTransform [W, b],) RelationEmbedding.
    variant: 'block', 'basis', or 'onehot' (basis with UseInputTransform=No)."""
    per = ["W_forward", "W_backward", "W_self", "b"] if variant == "block" else \
        ["W_forward", "W_backward", "C_forward", "C_backward", "W_self", "b"]
    names = [] if variant == "onehot" else ["W_in", "b_in"]
    for l in range(n_layers):
        names += ["L%d.%s" % (l, k) for k in per]
        if not (variant == "onehot" and l == 0):
            names += ["HW%d.W" % l, "HW%d.b" % l]
    return names + (["W_out", "b_out"] if outproj else []) + ["W_relation"]


def encode(leaves, variant, n_layers, outproj, triples, V, mode, masks, keep, norm_mode, dtype=torch.float64,
           norm_dtype=np.float64):
    """The encoder chain of model_builder.py:140-176 + :273-309 with every feature-input layer wrapped.

    variant 'onehot' restates what the reference computes there, not a textbook highway: layer 1's HighwayLayer reads
    its carry input through BasisGcn0.get_all_codes(), which returns the class-level MessageGcn cache -- by then
    holding layer 1's own output -- so code_2 = code_1 and out = g L1 + (1 - g) L1."""
    nf, nb = oracle.graph_norms(triples, V, norm_mode, norm_dtype)
    if variant == "onehot":
        H = torch.eye(V, dtype=dtype)
    else:
        H = oracle.affine_onehot(leaves["W_in"], leaves["b_in"])
    for l in range(n_layers):
        lp = {k.split(".")[1]: v for k, v in leaves.items() if k.startswith("L%d." % l)}
        relu = l < n_layers - 1
        mask = masks[l] if mode == "train" else None
        k = keep if mode == "train" else 1.0
        if variant == "block":
            L = oracle.concat_gcn_forward(H, triples, lp["W_forward"], lp["W_backward"], lp["W_self"], nf, nb, mask, k,
                                          relu, dtype)
        else:
            L = oracle.basis_gcn_forward(H, triples, lp["W_forward"], lp["W_backward"], lp["C_forward"],
                                         lp["C_backward"], lp["W_self"], nf, nb, mask, k, relu, dtype)
        if variant == "onehot" and l == 0:
            H = L
        elif variant == "onehot":
            H = highway(L, L, leaves["HW%d.W" % l], leaves["HW%d.b" % l])   # the dead gate
        else:
            H = highway(L, H, leaves["HW%d.W" % l], leaves["HW%d.b" % l])
    if outproj:
        H = H @ leaves["W_out"] + leaves["b_out"]
    return H
