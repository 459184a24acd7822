"""numpy oracle of the R-GCN+ ensemble ranks -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

  s_X = float32 sigmoid of member X's float64 energies (DistMult or ComplEx, all entities)
  c   = w s_A + (1 - w) s_B in float64 (separately rounded, as the reference's tools/ensemble.py computes it)
  raw = #{v : c_v >= c_gold},  filtered = raw - #{known v : c_v >= c_gold} + 1

The rank stage is pinned by tests/golden/reference_ensemble_golden.npz (the reference tool's own ranks)."""
import numpy as np

DISTMULT, COMPLEX = 0, 1


def energies(decoder, codes, rel, X, side):
    """[n, V] float64 energies of every entity in the corrupted position (side 0: subjects, 1: objects)."""
    c, r = np.asarray(codes, np.float64), np.asarray(rel, np.float64)
    s, p, o = X[:, 0], X[:, 1], X[:, 2]
    if decoder == DISTMULT:
        q = r[p] * c[o] if side == 0 else c[s] * r[p]
    else:
        h = c.shape[1] // 2
        rr, ri = r[p, :h], r[p, h:]
        if side == 0:
            er, ei = c[o, :h], c[o, h:]
            q = np.concatenate([rr * er + ri * ei, rr * ei - ri * er], 1)
        else:
            er, ei = c[s, :h], c[s, h:]
            q = np.concatenate([er * rr - ei * ri, ei * rr + er * ri], 1)
    return q @ c.T


def sigmoid32(e):
    """The library's float32 sigmoid 1 / (1 + expf(-x)) of float64 energies rounded to float32, every step rounded
    to float32 (exp correctly rounded; the device's expf may differ from it by an ulp or two)."""
    x = np.asarray(e).astype(np.float32)
    with np.errstate(over="ignore"):
        ex = np.exp(-x.astype(np.float64)).astype(np.float32)
        return (np.float32(1) / (np.float32(1) + ex)).astype(np.float32)


def combine(w, sa, sb):
    return float(w) * np.asarray(sa, np.float64) + (1.0 - float(w)) * np.asarray(sb, np.float64)


def ranks(c, gold, known_lists=None):
    """(raw, filtered or None) int64 [n] of the combined scores c [n, V] with the gold column `gold` [n]."""
    rows = np.arange(len(gold))
    g = c[rows, gold]
    ge = c >= g[:, None]
    raw = ge.sum(1)
    if known_lists is None:
        return raw, None
    kn = np.array([int(ge[i, np.asarray(k, np.int64)].sum()) if len(k) else 0 for i, k in enumerate(known_lists)],
                  np.int64)
    return raw, raw - kn + 1


def near_tie_rows(ca, cb, w, gold, tol):
    """Rows where another entity's combined score lies within tol of the gold's without an exact reason to tie:
    there the float32 rounding of energies and sigmoids can move that entity across the gold score.  An entity whose
    scores equal the gold's for a reason that holds on any device -- the same energy, or both energies far into the
    saturation of the float32 sigmoid to 1 -- in both members (or, at w = 0.5, swapped) is not a near tie.
    ca, cb: [n, V] float64 energies of the members."""
    rows = np.arange(len(gold))
    c = combine(w, sigmoid32(ca), sigmoid32(cb))
    g = c[rows, gold][:, None]
    ga, gb = ca[rows, gold][:, None], cb[rows, gold][:, None]

    def same(e, ge):
        return (e == ge) | (np.minimum(e, ge) >= 18.0)   # exp(-18) < 2^-25: 1 + expf(-x) rounds to 1

    exact = same(ca, ga) & same(cb, gb)
    if w == 0.5:
        exact |= same(ca, gb) & same(cb, ga)
    return np.any((np.abs(c - g) <= tol) & ~exact, axis=1)
