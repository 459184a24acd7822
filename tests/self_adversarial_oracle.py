"""float64 restatement of self-adversarial negative sampling (ops.self_adversarial_loss) with torch autograd.

The fed triples X [N, 3] follow the negative sampler's layout: N = n (K + 1), rows 0..n-1 the positives, row i + n j
(j = 1..K) the j-th corruption of positive i.  The softmax weights p are detached, so no gradient flows through them."""
import numpy as np
import torch


def softplus(x):
    return x.clamp(min=0) + torch.log1p(torch.exp(-x.abs()))


def energies(a, b, c, decoder):
    """energies of gathered rows a = codes[s], b = rel[r], c = codes[o] (ComplEx rows are [real | imaginary])"""
    if decoder == "distmult":
        return (a * b * c).sum(1)
    h = a.shape[1] // 2
    ar, ai, br, bi, cr, ci = a[:, :h], a[:, h:2 * h], b[:, :h], b[:, h:2 * h], c[:, :h], c[:, h:2 * h]
    return (br * (ar * cr + ai * ci) + bi * (ar * ci - ai * cr)).sum(1)


def weights(e, K, alpha):
    """p [K, n]: the softmax over each positive's corruptions of alpha * energy, detached"""
    return torch.softmax(alpha * e.detach().reshape(K + 1, -1)[1:], dim=0)


def loss(codes, rel, X, K, alpha, decoder, gathered_rel=None, p=None):
    """(loss, reg, energies); gathered_rel, if given, is rel[X[:, 1]] as its own leaf, so that its gradient holds the
    per-triple relation slices whose squared sum is the relation table's IndexedSlices norm; p, if given, replaces
    the weights (weights(energies, K, alpha))"""
    X = torch.as_tensor(np.asarray(X, dtype=np.int64).reshape(-1, 3), device=codes.device)
    N, d = X.shape[0], codes.shape[1]
    n = N // (K + 1)
    assert n * (K + 1) == N
    a, c = codes[X[:, 0]], codes[X[:, 2]]
    b = rel[X[:, 1]] if gathered_rel is None else gathered_rel
    e = energies(a, b, c, decoder)
    blocks = e.reshape(K + 1, n)              # blocks[0]: the positives, blocks[j]: their j-th corruptions
    if p is None:
        p = weights(e, K, alpha)
    L = (softplus(-blocks[0]) + (p * softplus(blocks[1:])).sum(0)).sum() / (2 * n)
    reg = ((a ** 2).sum() + (b ** 2).sum() + (c ** 2).sum()) / (N * d)
    return L, reg, e
