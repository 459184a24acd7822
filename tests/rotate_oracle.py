"""float64 restatement of the RotatE decoder (ops.rotate_score, ops.self_adversarial_loss(decoder="rotate"),
ops.RotateRanker) with torch autograd.

Entity rows are [re | im] with h = d / 2 columns each; the first h columns of a relation row are its phases.  With
a = codes[s], c = codes[o]:  u_k = a_k e^{i theta_k} - c_k,  D = sum_k |u_k|,  E = gamma - D.  The modulus' gradient is
u / |u|, and 0 where u = 0 (the subgradient the library uses)."""
import numpy as np
import torch

import self_adversarial_oracle as so


class _Modulus(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ur, ui):
        m = torch.hypot(ur, ui)
        ctx.save_for_backward(ur, ui, m)
        return m

    @staticmethod
    def backward(ctx, g):
        ur, ui, m = ctx.saved_tensors
        gm = torch.where(m > 0, g / torch.where(m > 0, m, torch.ones_like(m)), torch.zeros_like(m))
        return gm * ur, gm * ui


def residual(a, theta, c):
    """(u_re, u_im) [N, h] of u = a e^{i theta} - c for gathered rows a, c [N, d] and phases theta [N, >= h]"""
    h = a.shape[1] // 2
    t = theta[:, :h]
    cs, sn = torch.cos(t), torch.sin(t)
    return a[:, :h] * cs - a[:, h:2 * h] * sn - c[:, :h], a[:, :h] * sn + a[:, h:2 * h] * cs - c[:, h:2 * h]


def gather(codes, rel, X, gathered_rel=None):
    X = torch.as_tensor(np.asarray(X, dtype=np.int64).reshape(-1, 3), device=codes.device)
    b = rel[X[:, 1]] if gathered_rel is None else gathered_rel
    return codes[X[:, 0]], b, codes[X[:, 2]]


def energies(codes, rel, X, gamma, gathered_rel=None):
    """E [N]; gathered_rel, if given, is rel[X[:, 1]] as its own leaf (its gradient holds the per-triple slices)"""
    a, b, c = gather(codes, rel, X, gathered_rel)
    return gamma - _Modulus.apply(*residual(a, b, c)).sum(1)


def l2(codes, X):
    """mean(a^2) + mean(c^2) over the gathered entity rows, each over N d elements"""
    a, _, c = gather(codes, codes, X)
    return (a ** 2).mean() + (c ** 2).mean()


def ns_loss(codes, rel, X, Y, gamma, gathered_rel=None):
    """(loss, reg, energies) of the NegativeSampling objective: mean stable sigmoid cross-entropy over the N triples"""
    e = energies(codes, rel, X, gamma, gathered_rel)
    y = torch.as_tensor(Y).to(e)
    L = (torch.clamp(e, min=0) - e * y + torch.log1p(torch.exp(-e.abs()))).mean()
    return L, l2(codes, X), e


def self_adversarial_loss(codes, rel, X, K, alpha, gamma, gathered_rel=None, p=None):
    """(loss, reg, energies) of the self-adversarial objective in the sampler's layout (self_adversarial_oracle.loss
    with the RotatE energy and L2 term); p, if given, replaces the weights"""
    e = energies(codes, rel, X, gamma, gathered_rel)
    n = e.shape[0] // (K + 1)
    blocks = e.reshape(K + 1, n)
    if p is None:
        p = so.weights(e, K, alpha)
    L = (so.softplus(-blocks[0]) + (p * so.softplus(blocks[1:])).sum(0)).sum() / (2 * n)
    return L, l2(codes, X), e


def distances(codes, rel, X, side):
    """float64 (D [n, V], D_gold [n], gold [n]) torch tensors on codes' device for the all-entity ranking: side 1
    q = a e^{i theta} against every entity (gold o), side 0 q = c e^{-i theta} (gold s)"""
    codes, rel = torch.as_tensor(codes).double(), torch.as_tensor(rel).double().to(codes.device)
    X = torch.as_tensor(np.asarray(X, np.int64).reshape(-1, 3), device=codes.device)
    h = codes.shape[1] // 2
    kept, gold = (X[:, 2], X[:, 0]) if side == 0 else (X[:, 0], X[:, 2])
    theta = rel[X[:, 1], :h] * (-1.0 if side == 0 else 1.0)
    cs, sn = torch.cos(theta), torch.sin(theta)
    qr = codes[kept, :h] * cs - codes[kept, h:2 * h] * sn
    qi = codes[kept, :h] * sn + codes[kept, h:2 * h] * cs
    D = torch.zeros((len(X), len(codes)), dtype=torch.float64, device=codes.device)
    for k in range(h):
        D += torch.hypot(qr[:, k, None] - codes[None, :, k], qi[:, k, None] - codes[None, :, h + k])
    return D, D[torch.arange(len(X), device=codes.device), gold], gold


def ranks(codes, rel, X, side, known_lists=None):
    """numpy (raw [n], filtered [n] or None): raw = #{v : D_v <= D_gold}, filtered = raw - #{known v : D_v <= D_gold}
    + 1"""
    D, Dg, _ = distances(codes, rel, X, side)
    hit = (D <= Dg[:, None]).cpu().numpy()
    raw = hit.sum(1)
    if known_lists is None:
        return raw, None
    kn = np.array([int(hit[t, np.asarray(k, np.int64)].sum()) if len(k) else 0 for t, k in enumerate(known_lists)])
    return raw, raw - kn + 1
