"""float64 restatement of the R-GCN+ ensemble's top-k and relation prediction -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

  u   = w sigma(-E_A) + (1 - w) sigma(-E_B),  sigma(-E) = 1 / (1 + exp(E)) in float64 of the float32 energy E
  top-k: u ascending, the smaller id first on ties; padding id -1, u +inf, score 0; score = 1 - u
  relation energies: the member's relation query row against rel[0:R]
Ranks reuse tests/ensemble_oracle.py (combine, ranks) with relations as the candidates."""
import numpy as np

import ensemble_oracle as oracle


def sigmoid_neg64(e):
    """sigma(-E) in float64 of the energies rounded to float32, as the kernel forms it."""
    x = np.asarray(e).astype(np.float32).astype(np.float64)
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + np.exp(x))


def u_of(w, ea, eb):
    w = float(w)
    return w * sigmoid_neg64(ea) + (1.0 - w) * sigmoid_neg64(eb)   # numpy never fuses these into an FMA


def top_k(u, k, exclude_lists=None):
    """(ids int64 [n, k], u [n, k], scores [n, k]) of every row of u [n, N] by (u, id) ascending."""
    u = np.asarray(u, np.float64)
    n, N = u.shape
    ids = np.full((n, k), -1, np.int64)
    uu = np.full((n, k), np.inf)
    sc = np.zeros((n, k))
    for t in range(n):
        ok = np.ones(N, bool)
        if exclude_lists is not None and len(exclude_lists[t]):
            ok[np.asarray(exclude_lists[t], np.int64)] = False
        cand = np.nonzero(ok)[0]
        order = cand[np.lexsort((cand, u[t, cand]))][:k]
        m = len(order)
        ids[t, :m], uu[t, :m], sc[t, :m] = order, u[t, order], 1.0 - u[t, order]
    return ids, uu, sc


def relation_energies(decoder, codes, rel, X, R):
    """[n, R] float64 energies of every relation r < R for the pairs (X[t, 0], X[t, 2])."""
    c, r = np.asarray(codes, np.float64), np.asarray(rel, np.float64)[:R]
    h, t = c[X[:, 0]], c[X[:, 2]]
    if decoder == oracle.DISTMULT:
        q = h * t
    else:
        d = c.shape[1] // 2
        hr, hi, tr, ti = h[:, :d], h[:, d:], t[:, :d], t[:, d:]
        q = np.concatenate([hr * tr + hi * ti, hr * ti - hi * tr], 1)
    return q @ r.T


def check_top_k(ids, u, scores, ref_u_full, k, exclude_lists=None, rtol_u=1e-4, tie=1e-5):
    """The kernel's answer against the float64 restatement: u within rtol_u of the reference u of the returned id,
    each position's u within rtol_u of the reference's, and a different id at a position only where the two ids'
    float64 u agree to `tie` relative.  Padding must match exactly."""
    rid, ru, rs = top_k(ref_u_full, k, exclude_lists)
    assert ids.shape == rid.shape
    pad = rid < 0
    np.testing.assert_array_equal(ids < 0, pad)
    assert np.all(np.isinf(u[pad])) and np.all(scores[pad] == 0)
    rows, cols = np.nonzero(~pad)
    got_u = ref_u_full[rows, ids[rows, cols]]
    np.testing.assert_allclose(u[rows, cols], got_u, rtol=rtol_u, atol=1e-300)
    np.testing.assert_allclose(u[rows, cols], ru[rows, cols], rtol=rtol_u, atol=1e-300)
    np.testing.assert_allclose(scores[rows, cols], 1.0 - u[rows, cols], rtol=0, atol=0)
    diff = ids[rows, cols] != rid[rows, cols]
    if diff.any():
        a, b = got_u[diff], ru[rows, cols][diff]
        assert np.all(np.abs(a - b) <= tie * np.maximum(np.abs(a), np.abs(b))), (a, b)
    if exclude_lists is not None:
        for t in range(len(ids)):
            assert not set(ids[t][ids[t] >= 0].tolist()) & set(exclude_lists[t])
    return diff.mean() if diff.size else 0.0
