"""Float64 restatement of 1-N training (ops.one_to_n_loss) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE."""
import numpy as np
import torch


def queries(triples):
    """numpy restatement of ops.one_to_n_queries: the set of (anchor, r, side) rows, sorted by (side, r, anchor)."""
    rows = {(o, r, 0) for s, r, o in np.asarray(triples).reshape(-1, 3).tolist()}
    rows |= {(s, r, 1) for s, r, o in np.asarray(triples).reshape(-1, 3).tolist()}
    return np.array(sorted(rows, key=lambda q: (q[2], q[1], q[0])), dtype=np.int32).reshape(-1, 3)


def dense_labels(train, qs, V):
    """[n, V] float64 0/1: entity e completes query t in the training triples."""
    y = np.zeros((len(qs), V))
    obj, subj = {}, {}
    for s, r, o in np.asarray(train).reshape(-1, 3).tolist():
        obj.setdefault((s, r), set()).add(o)
        subj.setdefault((o, r), set()).add(s)
    for t, (a, r, side) in enumerate(np.asarray(qs).tolist()):
        for e in (obj if side == 1 else subj).get((a, r), ()):
            y[t, e] = 1.0
    return y


def bits(y):
    """the uint32 [n, ceil(V/32)] bit rows (as int32) of a dense 0/1 label matrix"""
    n, V = y.shape
    words = (V + 31) // 32
    padded = np.zeros((n, words * 32), np.uint64)
    padded[:, :V] = y != 0
    w = (padded.reshape(n, words, 32) << np.arange(32, dtype=np.uint64)).sum(axis=2)
    return w.astype(np.uint32).view(np.int32)


def unbits(b, V):
    b = np.asarray(b).view(np.uint32).astype(np.uint64)
    return ((b[:, :, None] >> np.arange(32, dtype=np.uint64)) & 1).reshape(len(b), -1)[:, :V].astype(np.float64)


def query_rows(codes, rel, qs, decoder):
    q = torch.as_tensor(np.asarray(qs, dtype=np.int64), device=codes.device)
    a, r, side = codes[q[:, 0]], rel[q[:, 1]], q[:, 2:3].to(codes.dtype)
    if decoder == "distmult":
        return a * r
    h = codes.shape[1] // 2
    kr, ki, br, bi = a[:, :h], a[:, h:2 * h], r[:, :h], r[:, h:2 * h]
    q1 = torch.cat([kr * br - ki * bi, ki * br + kr * bi], 1)       # side 1: e_s * r
    q0 = torch.cat([br * kr + bi * ki, br * ki - bi * kr], 1)       # side 0: conj(r) * e_o
    return side * q1 + (1 - side) * q0


def loss(codes, rel, qs, y, eps, decoder):
    """(loss, reg) of ops.one_to_n_loss in the dtype of codes; y dense [n, V]."""
    n, V = y.shape
    z = query_rows(codes, rel, qs, decoder) @ codes.T
    yt = (1 - eps) * y + eps / V
    L = (torch.clamp(z, min=0) - z * yt + torch.log1p(torch.exp(-z.abs()))).sum() / (n * V)
    q = torch.as_tensor(np.asarray(qs, dtype=np.int64), device=codes.device)
    reg = ((codes[q[:, 0]] ** 2).sum() + (rel[q[:, 1]] ** 2).sum()) / (n * codes.shape[1])
    return L, reg
