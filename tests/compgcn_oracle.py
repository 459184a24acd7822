"""CPU oracle for the CompGCN encoder (Encoder Name=compgcn) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A float64 torch restatement of DESIGN §1 (there is no reference code for CompGCN); backward is torch.autograd.
  layer     one CompGCN layer over explicit messages (dst, src, weight id, norm), halo rows allowed (V_src > V_dst)
  encode    the encoder chain model_builder builds for Name=compgcn over a triple list: a bias-free linear one-hot
            embedding, then the layers; returns (entity codes, relation codes Z^L[0:R])."""
import numpy as np
import torch

from oracle import rgcn_oracle as oracle

DT = torch.float64


def phi(h, z, composition):
    if composition == "mult":
        return h * z
    if composition == "sub":
        return h - z
    raise ValueError(composition)


def layer(H, Z, z_loop, W_cat, W_rel, b, dst, src, relw, norm, V_dst, composition="mult", drop_mask=None, keep=1.0,
          relu=True, dtype=DT):
    """(out [V_dst, d_out], Z_next [2R, d_out]) of one layer; relw < R is a forward message, relw >= R its inverse."""
    H, Z, z_loop, W_cat, W_rel, b = (oracle._t(x, dtype) for x in (H, Z, z_loop, W_cat, W_rel, b))
    dst, src, relw = (torch.as_tensor(np.asarray(a, np.int64)) for a in (dst, src, relw))
    norm = oracle._t(norm, dtype)
    R = Z.shape[0] // 2
    d = H.shape[1]
    msgs = norm[:, None] * phi(H[src], Z[relw], composition)
    fwd = relw < R
    A_f = torch.zeros(V_dst, d, dtype=dtype).index_add(0, dst[fwd], msgs[fwd])
    A_b = torch.zeros(V_dst, d, dtype=dtype).index_add(0, dst[~fwd], msgs[~fwd])
    A = torch.cat([A_f, A_b], 1)
    if drop_mask is not None:
        A = A * oracle._t(drop_mask, dtype) / keep
    Cat = torch.cat([A, phi(H[:V_dst], z_loop, composition)], 1) / 3
    out = Cat @ W_cat + b
    if relu:
        out = torch.relu(out)
    return out, Z @ W_rel


def triple_messages(triples, R, norm_f, norm_b):
    """(dst, src, weight id, norm) of a triple list: s -> o with weight id r and norm_f, o -> s with R + r and norm_b."""
    s, r, o = oracle.process_triples(triples)
    return (np.concatenate([o, s]), np.concatenate([s, o]), np.concatenate([r, r + R]),
            np.concatenate([np.asarray(norm_f, np.float64), np.asarray(norm_b, np.float64)]))


def weight_names(n_layers):
    """get_weights() order, deepest first: the one-hot embedding [W, b] (b is not read), layer 0 [Z, z_loop, W_cat,
    W_rel, b], every further layer [z_loop, W_cat, W_rel, b]."""
    names = ["W_in", "b_in"]
    for l in range(n_layers):
        names += ["L%d.%s" % (l, k) for k in (("Z",) if l == 0 else ()) + ("z_loop", "W_cat", "W_rel", "b")]
    return names


def encode(leaves, n_layers, triples, V, R, mode, masks, keep, norm_f, norm_b, composition="mult", dtype=DT):
    dst, src, relw, norm = triple_messages(triples, R, norm_f, norm_b)
    H = oracle._t(leaves["W_in"], dtype)
    Z = leaves["L0.Z"]
    for l in range(n_layers):
        p = {k.split(".")[1]: v for k, v in leaves.items() if k.startswith("L%d." % l)}
        train = mode == "train" and masks is not None
        H, Z = layer(H, Z, p["z_loop"], p["W_cat"], p["W_rel"], p["b"], dst, src, relw, norm, V, composition,
                     masks[l] if train else None, keep if train else 1.0, l < n_layers - 1, dtype)
    return H, Z[:R]
