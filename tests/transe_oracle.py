"""float64 restatement of the TransE decoder (ops.transe_score, ops.self_adversarial_loss(decoder="transe"),
ops.TransERanker) with torch autograd.

Entity and relation rows are plain real vectors.  With h = codes[s], r = rel[r], t = codes[o]:
u_k = h_k + r_k - t_k,  D = sum_k |u_k|,  E = gamma - D.  The gradient of |u| is sign(u), and 0 where u = 0 (the
subgradient the library uses; torch's abs has the same).  The L2 term covers all three gathered rows."""
import numpy as np
import torch

import self_adversarial_oracle as so


def gather(codes, rel, X, gathered_rel=None):
    X = torch.as_tensor(np.asarray(X, dtype=np.int64).reshape(-1, 3), device=codes.device)
    b = rel[X[:, 1]] if gathered_rel is None else gathered_rel
    return codes[X[:, 0]], b, codes[X[:, 2]]


def energies(codes, rel, X, gamma, gathered_rel=None):
    """E [N]; gathered_rel, if given, is rel[X[:, 1]] as its own leaf (its gradient holds the per-triple slices)"""
    h, r, t = gather(codes, rel, X, gathered_rel)
    return gamma - (h + r - t).abs().sum(1)


def l2(codes, rel, X, gathered_rel=None):
    """mean(h^2) + mean(r^2) + mean(t^2) over the gathered rows, each over N d elements"""
    h, r, t = gather(codes, rel, X, gathered_rel)
    return (h ** 2).mean() + (r ** 2).mean() + (t ** 2).mean()


def ns_loss(codes, rel, X, Y, gamma, gathered_rel=None):
    """(loss, reg, energies) of the NegativeSampling objective: mean stable sigmoid cross-entropy over the N triples"""
    e = energies(codes, rel, X, gamma, gathered_rel)
    y = torch.as_tensor(Y).to(e)
    L = (torch.clamp(e, min=0) - e * y + torch.log1p(torch.exp(-e.abs()))).mean()
    return L, l2(codes, rel, X, gathered_rel), e


def self_adversarial_loss(codes, rel, X, K, alpha, gamma, gathered_rel=None, p=None):
    """(loss, reg, energies) of the self-adversarial objective in the sampler's layout (self_adversarial_oracle.loss
    with the TransE energy and L2 term); p, if given, replaces the weights"""
    e = energies(codes, rel, X, gamma, gathered_rel)
    n = e.shape[0] // (K + 1)
    blocks = e.reshape(K + 1, n)
    if p is None:
        p = so.weights(e, K, alpha)
    L = (so.softplus(-blocks[0]) + (p * so.softplus(blocks[1:])).sum(0)).sum() / (2 * n)
    return L, l2(codes, rel, X, gathered_rel), e


def queries(codes, rel, X, side):
    """float64 (q [n, d], candidates [C, d], gold [n]): side 1 q = h + r against the entities (gold o), side 0
    q = t - r (gold s), side "relation" q = t - h against the relation rows (gold r)"""
    codes, rel = torch.as_tensor(codes).double(), torch.as_tensor(rel).double().to(codes.device)
    X = torch.as_tensor(np.asarray(X, np.int64).reshape(-1, 3), device=codes.device)
    if side == "relation":
        return codes[X[:, 2]] - codes[X[:, 0]], rel, X[:, 1]
    if side == 1:
        return codes[X[:, 0]] + rel[X[:, 1]], codes, X[:, 2]
    return codes[X[:, 2]] - rel[X[:, 1]], codes, X[:, 0]


def distances(codes, rel, X, side, count=None):
    """float64 (D [n, C], D_gold [n], gold [n]) torch tensors on codes' device; C = the first `count` candidate rows
    (default: all)"""
    q, cand, gold = queries(codes, rel, X, side)
    cand = cand if count is None else cand[:count]
    D = torch.zeros((q.shape[0], cand.shape[0]), dtype=torch.float64, device=q.device)
    for k in range(q.shape[1]):
        D += (q[:, k, None] - cand[None, :, k]).abs()
    return D, D[torch.arange(len(gold), device=q.device), gold], gold


def ranks(codes, rel, X, side, known_lists=None, count=None):
    """numpy (raw [n], filtered [n] or None): raw = #{v : D_v <= D_gold}, filtered = raw - #{known v : D_v <= D_gold}
    + 1"""
    D, Dg, _ = distances(codes, rel, X, side, count)
    hit = (D <= Dg[:, None]).cpu().numpy()
    raw = hit.sum(1)
    if known_lists is None:
        return raw, None
    kn = np.array([int(hit[t, np.asarray(k, np.int64)].sum()) if len(k) else 0 for t, k in enumerate(known_lists)])
    return raw, raw - kn + 1


def top_k(D, k, gamma, exclude_lists=None):
    """numpy (ids [n, k] int64, energies gamma - D [n, k]) of every row's k smallest D, the smaller id first on ties,
    never an id of exclude_lists[t]; the tail of a row with fewer than k eligible ids is (-1, -inf)"""
    D = np.asarray(D.cpu() if torch.is_tensor(D) else D, np.float64)
    n, C = D.shape
    ids = np.full((n, k), -1, np.int64)
    en = np.full((n, k), -np.inf)
    for t in range(n):
        ok = np.ones(C, bool)
        if exclude_lists is not None and len(exclude_lists[t]):
            ok[np.asarray(exclude_lists[t], np.int64)] = False
        cols = np.nonzero(ok)[0]
        order = cols[np.lexsort((cols, D[t, cols]))][:k]
        ids[t, :len(order)] = order
        en[t, :len(order)] = gamma - D[t, order]
    return ids, en
