"""float64 restatement of the QuatE decoder (ops.quate_score, ops.self_adversarial_loss(decoder="quate"),
ops.one_to_n_loss(decoder="quate"), ops.QuatERanker, ops.quate_query_rows) with torch autograd.

Quaternion k of a row x is x[..., 4k:4k+4] = (a, b, c, d) = a + b i + c j + d k.  With h = codes[s], r = rel[r],
t = codes[o]:  rh_k = r_k / max(|r_k|, 1e-12) (torch.nn.functional.normalize),  E = sum_k <h_k (x) rh_k, t_k>.
The L2 term is DistMult's over the raw rows."""
import numpy as np
import torch

import self_adversarial_oracle as so

EPS = 1e-12


def quats(x):
    return x.reshape(*x.shape[:-1], -1, 4)


def qmul(p, q):
    """the Hamilton product of quaternions along the last axis (4)"""
    a1, b1, c1, d1 = p.unbind(-1)
    a2, b2, c2, d2 = q.unbind(-1)
    return torch.stack([a1 * a2 - b1 * b2 - c1 * c2 - d1 * d2,
                        a1 * b2 + b1 * a2 + c1 * d2 - d1 * c2,
                        a1 * c2 - b1 * d2 + c1 * a2 + d1 * b2,
                        a1 * d2 + b1 * c2 - c1 * b2 + d1 * a2], -1)


def qconj(q):
    return q * torch.tensor([1.0, -1.0, -1.0, -1.0], dtype=q.dtype, device=q.device)


def normalize(r):
    """rows of quaternions [.., d] -> each quaternion / max(|quaternion|, EPS)"""
    q = quats(r)
    return (q / q.norm(dim=-1, keepdim=True).clamp_min(EPS)).reshape(r.shape)


def flat(q):
    return q.reshape(*q.shape[:-2], -1)


def _ids(X, device):
    return torch.as_tensor(np.asarray(X, dtype=np.int64).reshape(-1, 3), device=device)


def gather(codes, rel, X, gathered_rel=None):
    X = _ids(X, codes.device)
    b = rel[X[:, 1]] if gathered_rel is None else gathered_rel
    return codes[X[:, 0]], b, codes[X[:, 2]]


def energies(codes, rel, X, gathered_rel=None):
    """E [N]; gathered_rel, if given, is rel[X[:, 1]] as its own leaf (its gradient holds the per-triple slices)"""
    h, r, t = gather(codes, rel, X, gathered_rel)
    return (flat(qmul(quats(h), quats(normalize(r)))) * t).sum(1)


def l2(codes, rel, X, gathered_rel=None):
    """mean(h^2) + mean(r^2) + mean(t^2) over the gathered raw rows, each over N d elements"""
    h, r, t = gather(codes, rel, X, gathered_rel)
    return (h ** 2).mean() + (r ** 2).mean() + (t ** 2).mean()


def ns_loss(codes, rel, X, Y, gathered_rel=None):
    """(loss, reg, energies) of the NegativeSampling objective: mean stable sigmoid cross-entropy over the N triples"""
    e = energies(codes, rel, X, gathered_rel)
    y = torch.as_tensor(Y).to(e)
    L = (torch.clamp(e, min=0) - e * y + torch.log1p(torch.exp(-e.abs()))).mean()
    return L, l2(codes, rel, X, gathered_rel), e


def self_adversarial_loss(codes, rel, X, K, alpha, gathered_rel=None, p=None):
    """(loss, reg, energies) of the self-adversarial objective in the sampler's layout; p, if given, replaces the
    weights"""
    e = energies(codes, rel, X, gathered_rel)
    n = e.shape[0] // (K + 1)
    blocks = e.reshape(K + 1, n)
    if p is None:
        p = so.weights(e, K, alpha)
    L = (so.softplus(-blocks[0]) + (p * so.softplus(blocks[1:])).sum(0)).sum() / (2 * n)
    return L, l2(codes, rel, X, gathered_rel), e


def queries(codes, rel, X, side):
    """(Q [n, d], candidates [C, d], gold [n]) in the dtype of codes: side 1 Q = h (x) rh against the entities (gold
    o), side 0 Q = t (x) conj(rh) (gold s), side "relation" Q = conj(h) (x) t against the normalised relation rows
    (gold r)"""
    X = _ids(X, codes.device)
    h, t = quats(codes[X[:, 0]]), quats(codes[X[:, 2]])
    if side == "relation":
        return flat(qmul(qconj(h), t)), normalize(rel), X[:, 1]
    rh = quats(normalize(rel[X[:, 1]]))
    if side == 1:
        return flat(qmul(h, rh)), codes, X[:, 2]
    return flat(qmul(t, qconj(rh))), codes, X[:, 0]


def scores(codes, rel, X, side, count=None):
    """float64 (S [n, C], S_gold [n], gold [n]): the energies of every candidate, C = the first `count` (default all)"""
    codes = torch.as_tensor(codes).double()
    rel = torch.as_tensor(rel).double().to(codes.device)
    Q, cand, gold = queries(codes, rel, X, side)
    cand = cand if count is None else cand[:count]
    S = Q @ cand.T
    return S, S[torch.arange(len(gold), device=S.device), gold], gold


def ranks(S, gold, known_lists=None):
    """numpy (raw [n], filtered [n] or None) by the rules of distmult_rank on the energies S [n, C]: raw = #{v : S_v
    >= S_gold}, filtered = raw - #{known v : S_v >= S_gold} + 1 (energy order: callers keep S where the float32
    sigmoid is strictly increasing, or compare away from ties)"""
    S = np.asarray(S.cpu() if torch.is_tensor(S) else S, np.float64)
    gold = np.asarray(gold.cpu() if torch.is_tensor(gold) else gold, np.int64)
    hit = S >= S[np.arange(len(S)), gold][:, None]
    raw = hit.sum(1)
    if known_lists is None:
        return raw, None
    kn = np.array([int(hit[t, np.asarray(k, np.int64)].sum()) if len(k) else 0 for t, k in enumerate(known_lists)])
    return raw, raw - kn + 1


def top_k(S, k, exclude_lists=None):
    """numpy (ids [n, k] int64, energies [n, k]) of every row's k largest S, the smaller id first on ties, never an id
    of exclude_lists[t]; the tail of a row with fewer than k eligible ids is (-1, -inf)"""
    S = np.asarray(S.cpu() if torch.is_tensor(S) else S, np.float64)
    n, C = S.shape
    ids = np.full((n, k), -1, np.int64)
    en = np.full((n, k), -np.inf)
    for t in range(n):
        ok = np.ones(C, bool)
        if exclude_lists is not None and len(exclude_lists[t]):
            ok[np.asarray(exclude_lists[t], np.int64)] = False
        cols = np.nonzero(ok)[0]
        order = cols[np.lexsort((cols, -S[t, cols]))][:k]
        ids[t, :len(order)] = order
        en[t, :len(order)] = S[t, order]
    return ids, en


def one_to_n_loss(codes, rel, qs, y, eps):
    """(loss, reg) of ops.one_to_n_loss(decoder="quate") in the dtype of codes; qs (anchor, r, side) [n, 3], y dense
    [n, V].  The L2 term is DistMult's: the anchor and the raw relation row."""
    q = torch.as_tensor(np.asarray(qs, dtype=np.int64), device=codes.device)
    a, rh = quats(codes[q[:, 0]]), quats(normalize(rel[q[:, 1]]))
    side = q[:, 2:3].to(codes.dtype)
    Q = side * flat(qmul(a, rh)) + (1 - side) * flat(qmul(a, qconj(rh)))
    n, V = y.shape
    z = Q @ codes.T
    yt = (1 - eps) * y + eps / V
    L = (torch.clamp(z, min=0) - z * yt + torch.log1p(torch.exp(-z.abs()))).sum() / (n * V)
    reg = ((codes[q[:, 0]] ** 2).sum() + (rel[q[:, 1]] ** 2).sum()) / (n * codes.shape[1])
    return L, reg
