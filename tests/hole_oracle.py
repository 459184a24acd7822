"""float64 restatement of the HolE decoder (ops.hole_transform, ops.hole_score, ops.self_adversarial_loss(decoder=
"hole"), ops.one_to_n_loss(decoder="hole"), ops.HolERanker, ops.hole_query_rows) with torch autograd.

With h = codes[s], r = rel[r], t = codes[o] (raw rows, d % 4 == 0):  E = sum_k r_k [h * t]_k  with the circular
correlation [h * t]_k = sum_i h_i t_{(i + k) mod d} (`energies`; `correlate_direct` writes the sum out, `correlate`
forms it by FFT).  The library works on rows in
the real Fourier basis x~ = x U (`basis`), where E = sqrt(d) (h~0 r~0 t~0 + h~1 r~1 t~1) + sqrt(d/2) sum_f
Re(conj(h~f r~f) t~f) (`fourier_energies`); the query rows (`queries`) are in that basis too.  The L2 term is DistMult's
over the raw rows."""
import numpy as np
import torch

import self_adversarial_oracle as so
from quate_oracle import ranks, top_k  # noqa: F401  (DistMult's rank and top-k rules, restated there)


def basis(d, dtype=torch.float64):
    """U [d, d]: column 0 = 1/sqrt(d), column 1 = (-1)^k / sqrt(d), columns 2f, 2f+1 =
    sqrt(2/d) (cos, -sin)(2 pi f k / d)"""
    k = np.arange(d)[:, None]
    f = np.arange(1, d // 2)[None, :]
    U = np.empty((d, d))
    U[:, 0] = 1 / np.sqrt(d)
    U[:, 1] = (-1.0) ** np.arange(d) / np.sqrt(d)
    ang = 2 * np.pi * ((f * k) % d) / d
    U[:, 2::2] = np.sqrt(2 / d) * np.cos(ang)
    U[:, 3::2] = -np.sqrt(2 / d) * np.sin(ang)
    return torch.as_tensor(U, dtype=dtype)


def transform(x):
    return x @ basis(x.shape[-1], x.dtype).to(x.device)


def correlate_direct(h, t):
    """[h * t]_k = sum_i h_i t_{(i + k) mod d} along the last axis, the O(d^2) sum as written"""
    d = h.shape[-1]
    return torch.stack([(h * torch.roll(t, -k, dims=-1)).sum(-1) for k in range(d)], -1)


def correlate(h, t):
    """[h * t]_k as irfft(conj(rfft(h)) rfft(t)): the same numbers as correlate_direct to float64 rounding
    (test_hole_cpu), without its O(N d^2) memory under autograd at the GPU tests' sizes"""
    d = h.shape[-1]
    return torch.fft.irfft(torch.conj(torch.fft.rfft(h)) * torch.fft.rfft(t), n=d)


def _ids(X, device):
    return torch.as_tensor(np.asarray(X, dtype=np.int64).reshape(-1, 3), device=device)


def gather(codes, rel, X, gathered_rel=None):
    X = _ids(X, codes.device)
    b = rel[X[:, 1]] if gathered_rel is None else gathered_rel
    return codes[X[:, 0]], b, codes[X[:, 2]]


def energies(codes, rel, X, gathered_rel=None):
    """E [N] of raw rows, <r, h * t>; gathered_rel, if given, is rel[X[:, 1]] as its own leaf (its gradient
    holds the per-triple slices)"""
    h, r, t = gather(codes, rel, X, gathered_rel)
    return (r * correlate(h, t)).sum(1)


def _weights(d, dtype, device):
    w = torch.full((d,), np.sqrt(d / 2), dtype=dtype, device=device)
    w[:2] = np.sqrt(d)
    return w


def _mul(a, b, conj_a=False):
    """w (a b) or w conj(a) b on rows in the basis: columns 0, 1 real, then (re, im) pairs"""
    d = a.shape[-1]
    ar, ai, br, bi = a[..., 2::2], a[..., 3::2], b[..., 2::2], b[..., 3::2]
    if conj_a:
        ai = -ai
    out = torch.empty(torch.broadcast_shapes(a.shape, b.shape), dtype=a.dtype, device=a.device)
    out[..., :2] = a[..., :2] * b[..., :2]
    out[..., 2::2] = ar * br - ai * bi
    out[..., 3::2] = ar * bi + ai * br
    return out * _weights(d, a.dtype, a.device)


def fourier_energies(ct, rt, X):
    """E [N] of rows already in the basis: <w (h~ r~), t~>"""
    h, r, t = gather(ct, rt, X)
    return (_mul(h, r) * t).sum(1)


def l2(codes, rel, X, gathered_rel=None):
    """mean(h^2) + mean(r^2) + mean(t^2) over the gathered rows, each over N d elements"""
    h, r, t = gather(codes, rel, X, gathered_rel)
    return (h ** 2).mean() + (r ** 2).mean() + (t ** 2).mean()


def ns_loss(codes, rel, X, Y, gathered_rel=None):
    """(loss, reg, energies) of the NegativeSampling objective on raw rows"""
    e = energies(codes, rel, X, gathered_rel)
    y = torch.as_tensor(Y).to(e)
    L = (torch.clamp(e, min=0) - e * y + torch.log1p(torch.exp(-e.abs()))).mean()
    return L, l2(codes, rel, X, gathered_rel), e


def self_adversarial_loss(codes, rel, X, K, alpha, gathered_rel=None, p=None):
    """(loss, reg, energies) of the self-adversarial objective in the sampler's layout on raw rows; p, if given,
    replaces the weights"""
    e = energies(codes, rel, X, gathered_rel)
    n = e.shape[0] // (K + 1)
    blocks = e.reshape(K + 1, n)
    if p is None:
        p = so.weights(e, K, alpha)
    L = (so.softplus(-blocks[0]) + (p * so.softplus(blocks[1:])).sum(0)).sum() / (2 * n)
    return L, l2(codes, rel, X, gathered_rel), e


def queries(ct, rt, X, side):
    """(Q [n, d], candidates [C, d], gold [n]) of rows in the basis: side 1 Q = w (h~ r~) against the entities (gold
    o), side 0 Q = w conj(r~) t~ (gold s), side "relation" Q = w conj(h~) t~ against the relation rows (gold r)"""
    X = _ids(X, ct.device)
    h, r, t = ct[X[:, 0]], rt[X[:, 1]], ct[X[:, 2]]
    if side == "relation":
        return _mul(h, t, conj_a=True), rt, X[:, 1]
    if side == 1:
        return _mul(h, r), ct, X[:, 2]
    return _mul(r, t, conj_a=True), ct, X[:, 0]


def scores(ct, rt, X, side, count=None):
    """float64 (S [n, C], S_gold [n], gold [n]) of rows in the basis: the energies of every candidate, C = the first
    `count` (default all)"""
    ct = torch.as_tensor(ct).double()
    rt = torch.as_tensor(rt).double().to(ct.device)
    Q, cand, gold = queries(ct, rt, X, side)
    cand = cand if count is None else cand[:count]
    S = Q @ cand.T
    return S, S[torch.arange(len(gold), device=S.device), gold], gold


def one_to_n_loss(codes, rel, qs, y, eps):
    """(loss, reg) of ops.one_to_n_loss(decoder="hole") on raw rows in the dtype of codes; qs (anchor, r, side) [n, 3],
    y dense [n, V].  The L2 term is DistMult's: the anchor and the relation row."""
    q = torch.as_tensor(np.asarray(qs, dtype=np.int64), device=codes.device)
    ct, rt = transform(codes), transform(rel)
    a, r = ct[q[:, 0]], rt[q[:, 1]]
    side = q[:, 2:3].to(codes.dtype)
    Q = side * _mul(a, r) + (1 - side) * _mul(r, a, conj_a=True)
    n, V = y.shape
    z = Q @ ct.T
    yt = (1 - eps) * y + eps / V
    L = (torch.clamp(z, min=0) - z * yt + torch.log1p(torch.exp(-z.abs()))).sum() / (n * V)
    reg = ((codes[q[:, 0]] ** 2).sum() + (rel[q[:, 1]] ** 2).sum()) / (n * codes.shape[1])
    return L, reg
