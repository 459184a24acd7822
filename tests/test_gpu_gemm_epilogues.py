"""GPU: every kernel of the 3xTF32 GEMM library (tests/gemm_kernels.py) through its public entry point, against float64
references computed on the GPU in torch, at the GEMM's own boundaries:

  M (rows, queries)    1, 127, 128, 129, tile counts below the SM count, and CTAs that walk 1, 2 and >= 16 tiles
  N (columns)          4, 124, 128, 132, 14541 (N % 128 in {0, 4, 124}; N % 32 != 0 for the bitmaps' last word);
                       60, 64, 68 for the ensemble's 64-wide tiles
  K (contraction)      4, 28, 32, 36, 96, 100, 500, 512: one partial k-block, exactly one, and k-block counts per CTA
                       (total_g) of 0, 1 and 2 mod 3, the producer's unroll and the 3-stage ring (4 for the ensemble)

Two kinds of operands.  Gaussian ones for the continuous outputs, at the library's 1e-5 relative bar (max |error| /
max |reference|) where the output is a GEMM plus an elementwise epilogue.  Exact-arithmetic ones for ranks, top-k and
the ensemble at w in {0, 1}: small integers, so that every product and partial sum is exact in TF32 and fp32 (an
integer of magnitude below 2^11 is its own TF32 hi part, lo = 0) and the GEMM, the prepare kernels and float64 agree
bit for bit; ranks, tie orders and top-k ids are then compared exactly.  Rank energies stay within |z| <= 14, where
the float32 sigmoid is strictly increasing on the integers.  The STORE epilogue and the TN kernel are covered by
tests/test_gpu_gemm.py and tests/test_gpu_gemm_tn_schedule.py."""
import numpy as np
import pytest
import torch

import fresh_process
import gemm_kernels as gk
import one_to_n_oracle as oo
import test_gpu_compgcn as tcg
import test_gpu_one_to_n as t1n
from relationprediction_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-5


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-30))


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def rows(m, n_tiles_n=1, bn=128):
    """M itself, or for "<t>w" the rows that give every persistent CTA exactly t tiles (n_tiles_n tiles per M tile)"""
    if isinstance(m, str):
        t = int(m[:-1])
        return bn * max(1, t * sms() // n_tiles_n)
    return m


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ---------------------------------------------------------------------------------------------------------------------
# exact-arithmetic DistMult operands
# ---------------------------------------------------------------------------------------------------------------------
def int_tables(V, d, R, seed):
    """codes in {-1, 0, 1}; relation rows +-1 at one position per k-block (at most 14 blocks, the first and the last
    always: the partial last k-block counts), zero elsewhere.  Every energy is an integer with |z| <= 14."""
    g = gen(seed)
    codes = torch.randint(-1, 2, (V, d), generator=g, device=DEV).float()
    relt = torch.zeros(R, d, device=DEV)
    nkb = (d + 31) // 32
    blocks = sorted(set(np.linspace(0, nkb - 1, min(nkb, 14)).round().astype(int).tolist()))
    rng = np.random.default_rng(seed)
    for r in range(R):
        for b in blocks:
            k = b * 32 + int(rng.integers(0, min(32, d - b * 32)))
            relt[r, k] = float(rng.choice([-1.0, 1.0]))
    return codes, relt


def triples(n, V, R, seed):
    g = gen(seed + 1)
    return torch.stack([torch.randint(0, V, (n,), generator=g, device=DEV), torch.randint(0, R, (n,), generator=g,
                                                                                        device=DEV),
                        torch.randint(0, V, (n,), generator=g, device=DEV)], 1).int().contiguous()


def energies(codes, relt, X, side):
    """[n, V] float64 DistMult energies of every entity in the corrupted position"""
    c, r = codes.double(), relt.double()
    kept = X[:, 2] if side == 0 else X[:, 0]
    return (c[kept.long()] * r[X[:, 1].long()]) @ c.T


def bitmask(n, N, seed, density=0.3, boundary=True):
    """([n, ceil(N/32)] int32 bit rows, [n, N] bool): random bits, every row's bits at the word and tile boundaries
    31, 32, 127, 128 and N - 1 set, and the padding bits of the last word (columns >= N) set too."""
    words = (N + 31) // 32
    dense = torch.rand(n, words * 32, generator=gen(seed + 2), device=DEV) < density
    if boundary:
        for c in (31, 32, 127, 128, N - 1):
            if c < N:
                dense[:, c] = True
    dense[:, N:] = True
    return _pack(dense, n, words), dense[:, :N]


def _pack(dense, n, words):
    """int32 bit words of a [n, 32 words] bool matrix"""
    w = (dense.view(n, words, 32).long() << torch.arange(32, device=DEV)).sum(2)
    w = torch.where(w >= 2 ** 31, w - 2 ** 32, w)
    return w.to(torch.int32).contiguous()


def ref_ranks(E, gold, known):
    """(raw, filtered) of DistMultRanker.rank: raw = #{v : E_v >= E_gold}, filtered = raw - #{known v counted} + 1"""
    Eg = E.gather(1, gold[:, None].long())
    ge = E >= Eg
    raw = ge.sum(1)
    return raw, raw - (ge & known).sum(1) + 1


def ref_topk(E, excl, k):
    """(ids, energies) of top_k: energy descending, the smaller id first on ties, excluded columns never; the tail
    past the eligible columns is (-1, -inf)"""
    key = torch.where(excl, torch.full_like(E, float("inf")), -E)
    if k > key.shape[1]:   # fewer columns than k
        key = torch.cat([key, torch.full((key.shape[0], k - key.shape[1]), float("inf"), device=DEV,
                                         dtype=key.dtype)], 1)
    s, idx = torch.sort(key, dim=1, stable=True)
    s, idx = s[:, :k], idx[:, :k]
    none = torch.isinf(s)
    return torch.where(none, -1, idx).int(), torch.where(none, float("-inf"), -s)


RANK_SHAPES = [(1, 4, 4), (127, 124, 28), (128, 128, 32), (129, 132, 36), (129, 14541, 96), (300, 14541, 100),
               (64, 14541, 500), (129, 256, 512), ("1w", 124, 96), ("2w", 128, 36), ("16w", 4, 4)]


@pytest.mark.parametrize("n,V,d", RANK_SHAPES)
def test_rank_exact(n, V, d):
    """k_gemm_tf32x3<1>: exact raw and filtered ranks (ties counted), known bits at word / tile boundaries, padding
    bits past N set in the mask, rows >= M and columns >= N never counted"""
    n = rows(n, (V + 127) // 128)
    codes, relt = int_tables(V, d, 5, seed=V + d)
    X = triples(n, V, 5, seed=d)
    side = n % 2
    E = energies(codes, relt, X, side)
    assert float(E.abs().max()) <= 14
    gold = X[:, 0] if side == 0 else X[:, 2]
    known, known_dense = bitmask(n, V, seed=n)
    raw, filt = ops.DistMultRanker(codes, relt).rank(X, side, known)
    want_raw, want_filt = ref_ranks(E, gold, known_dense)
    assert torch.equal(raw.long(), want_raw)
    assert torch.equal(filt.long(), want_filt)


@pytest.mark.parametrize("R,d", [(4, 36), (132, 100), (124, 512)])
def test_relation_rank_exact(R, d):
    """k_gemm_tf32x3<1> with N = R: the pair queries (h, ?, t) against rel[0:R], exact"""
    V, n = 300, 129
    codes, relt = int_tables(V, d, R + 3, seed=R)   # rows R.. are never candidates
    codes = codes * (torch.rand(V, d, generator=gen(R), device=DEV) < 0.5)
    X = triples(n, V, R, seed=R + d)
    c, r = codes.double(), relt.double()
    E = (c[X[:, 0].long()] * c[X[:, 2].long()]) @ r[:R].T
    assert float(E.abs().max()) <= 14
    known, known_dense = bitmask(n, R, seed=d)
    raw, filt = ops.DistMultRanker(codes, relt, R).rank_relations(X, known)
    want_raw, want_filt = ref_ranks(E, X[:, 1], known_dense)
    assert torch.equal(raw.long(), want_raw) and torch.equal(filt.long(), want_filt)


def gauss_tables(V, d, R, seed, scale=0.3):
    g = gen(seed)
    return (torch.randn(V, d, generator=g, device=DEV) * scale, torch.randn(R, d, generator=g, device=DEV) * scale)


def energy_err(codes, relt, X, side):
    """a bound on |GEMM energy - float64 energy| per entity, from the split error of split_tf32_trunc (the query rows:
    |a - hi - lo| < 2^-20 |a|), the dropped lo*lo term and the RN split of the codes (2^-22 |b| each), and the
    truncating fp32 accumulation (an ulp, 2^-23 relative, per k-step of the sum of |products|): 2^-17 sum |q_k b_k|
    covers all of them with a margin of four"""
    c, r = codes.double(), relt.double()
    kept = X[:, 2] if side == 0 else X[:, 0]
    return 2.0 ** -17 * ((c[kept.long()] * r[X[:, 1].long()]).abs() @ c.abs().T) + 1e-30


@pytest.mark.parametrize("n,V,d", [(129, 14541, 100), (300, 132, 36)])
def test_rank_gaussian_band(n, V, d):
    """Gaussian operands: the raw rank lies in the band of the entities whose float64 energy is within the GEMM's
    error of the gold's (the float32 sigmoid is strictly increasing, so the energy order decides outside the band)"""
    codes, relt = gauss_tables(V, d, 5, seed=d)
    X = triples(n, V, 5, seed=n)
    E = energies(codes, relt, X, 1)
    tol = energy_err(codes, relt, X, 1)
    Eg = E.gather(1, X[:, 2:3].long())
    tg = tol.gather(1, X[:, 2:3].long())
    # sigmoid spacing: float32 sigmoid values closer than an ulp of 1 may round together; widen the band by that
    slack = tol + tg + 2.0 ** -22
    lo = (E > Eg + slack).sum(1) + 1
    hi = (E >= Eg - slack).sum(1)
    raw, _ = ops.DistMultRanker(codes, relt).rank(X, 1)
    assert bool(((raw.long() >= lo) & (raw.long() <= hi)).all())


def test_rank_with_a_bitwise_copy_of_the_gold():
    """Another entity whose code row is a bitwise copy of the gold's has the gold's float64 energy, so the reference
    counts it (>= on one score matrix).  With Gaussian values the kernel compares the copy's GEMM energy with the
    prepare kernel's gold dot product, formed differently, so it may miss the copy (DESIGN.md, section 3, "Rank ties
    with the gold"); it never misses anything else, and always counts the gold itself."""
    V, d, n = 2000, 100, 256
    codes, relt = gauss_tables(V, d, 5, seed=3)
    X = triples(n, V, 5, seed=4)
    X[:, 2] = torch.arange(n, device=DEV, dtype=torch.int32) * 2          # gold entity 2t, its copy 2t + 1
    codes[1:2 * n:2] = codes[0:2 * n:2]
    E = energies(codes, relt, X, 1)
    Eg = E.gather(1, X[:, 2:3].long())
    tol = energy_err(codes, relt, X, 1) * 2 + 2.0 ** -22
    clean = ((E - Eg).abs() <= tol).sum(1) == 2                             # the gold and its copy only
    assert int(clean.sum()) > n // 2
    raw, _ = ops.DistMultRanker(codes, relt).rank(X, 1)
    want = (E >= Eg).sum(1)
    got = raw.long()[clean]
    assert bool(((got == want[clean]) | (got == want[clean] - 1)).all())
    # integer operands: both energies are exact, and the copy is always counted
    codes, relt = int_tables(V, d, 5, seed=5)
    codes[1:2 * n:2] = codes[0:2 * n:2]
    E = energies(codes, relt, X, 1)
    raw, _ = ops.DistMultRanker(codes, relt).rank(X, 1)
    assert torch.equal(raw.long(), (E >= E.gather(1, X[:, 2:3].long())).sum(1))


TOPK_SHAPES = [(1, 4, 4), (127, 124, 28), (129, 132, 36), (129, 14541, 96), (300, 2000, 100), (64, 4000, 500),
               (128, 256, 512), ("1w", 128, 32), ("2w", 124, 36), ("16w", 4, 4)]


def topk_exclusions(n, V, seed):
    excl, dense = bitmask(n, V, seed, density=0.2)
    dense = dense.clone()
    dense[0::3, :min(V, 128)] = True               # a tile with every column excluded: its (-inf, -1) tail
    dense[1::3, :] = True
    dense[1::3, :V:max(1, V // 5)] = False         # rows with fewer eligible columns than k
    words = (V + 31) // 32
    full = torch.ones(n, words * 32, dtype=torch.bool, device=DEV)
    full[:, :V] = dense
    return _pack(full, n, words), dense


@pytest.mark.parametrize("n,V,d", TOPK_SHAPES)
@pytest.mark.parametrize("k", [1, 10, 127, 128])
def test_topk_exact(n, V, d, k):
    """k_gemm_tf32x3<4>: ids and energies exactly, ties by the smaller id, excluded tiles and short rows"""
    if isinstance(n, str) and k > 10:
        pytest.skip("the persistent walk is exercised at k <= 10")
    n = rows(n, (V + 127) // 128)
    codes, relt = int_tables(V, d, 5, seed=V + d + k)
    codes = codes * 3   # top-k reads energies, not sigmoids: |z| <= 126 is exact too, with fewer ties
    X = triples(n, V, 5, seed=k)
    excl, dense = topk_exclusions(n, V, seed=d)
    ids, e = ops.DistMultRanker(codes, relt).top_k(X, 1, k, excl)
    want_ids, want_e = ref_topk(energies(codes, relt, X, 1), dense, k)
    assert torch.equal(ids, want_ids)
    assert torch.equal(e.double(), want_e)


@pytest.mark.parametrize("R,k", [(4, 10), (132, 128), (124, 1)])
def test_relation_topk_exact(R, k):
    V, d, n = 300, 36, 129
    codes, relt = int_tables(V, d, R + 3, seed=R + 1)
    X = triples(n, V, R, seed=R)
    c, r = codes.double(), relt.double()
    E = (c[X[:, 0].long()] * c[X[:, 2].long()]) @ r[:R].T
    excl, dense = topk_exclusions(n, R, seed=k)
    ids, e = ops.DistMultRanker(codes, relt, R).top_k_relations(X, k, excl)
    want_ids, want_e = ref_topk(E, dense, k)
    assert torch.equal(ids, want_ids) and torch.equal(e.double(), want_e)


# ---------------------------------------------------------------------------------------------------------------------
# ensemble
# ---------------------------------------------------------------------------------------------------------------------
ENS_SHAPES = [(1, 60, 36, 96), (129, 64, 100, 32), (127, 68, 28, 4), (300, 14541, 36, 100), ("2w", 64, 4, 36)]


def ens_members(V, d_a, d_b, seed):
    ca, ra = int_tables(V, d_a, 5, seed)
    cb, rb = int_tables(V, d_b, 5, seed + 1)
    return ops.DistMultRanker(ca, ra), ops.DistMultRanker(cb, rb)


@pytest.mark.parametrize("n,V,d_a,d_b", ENS_SHAPES)
def test_ensemble_w01_reproduces_the_members(n, V, d_a, d_b):
    """k_gemm_ensemble<EnsRankEpi> / <EnsTopKEpi> at w = 1 (0): member A's (B's) ranks and top-k ids exactly"""
    n = rows(n, (V + 63) // 64, bn=128)
    a, b = ens_members(V, d_a, d_b, seed=V + d_a)
    X = triples(n, V, 5, seed=d_b)
    known, _ = bitmask(n, V, seed=7)
    excl, _ = topk_exclusions(n, V, seed=8)
    for w, single in ((1.0, a), (0.0, b)):
        ens = ops.EnsembleRanker(a, b, w)
        r_e, f_e = ens.rank(X, 1, known)
        r_s, f_s = single.rank(X, 1, known)
        assert torch.equal(r_e, r_s) and torch.equal(f_e, f_s), w
        for k in (1, 10, 128):
            ids_e, u, _ = ens.top_k(X, 1, k, excl)
            ids_s, _ = single.top_k(X, 1, k, excl)
            assert torch.equal(ids_e, ids_s), (w, k)
            assert bool(torch.isinf(u[ids_e < 0]).all())


def sigmoid32(E):
    """the library's float32 sigmoid 1 / (1 + expf(-x)) of exact integer energies"""
    x = E.float()
    return 1.0 / (1.0 + torch.exp(-x))


@pytest.mark.parametrize("n,V,d_a,d_b", ENS_SHAPES)
def test_ensemble_mixed_weight(n, V, d_a, d_b):
    """0 < w < 1 against float64: ranks in the band of the near ties (exact ties of both members count), top-k u
    within 1e-12 of float64 and every returned id's u within that of the reference's at its place"""
    n = rows(n, (V + 63) // 64, bn=128)
    w = 0.3
    a, b = ens_members(V, d_a, d_b, seed=V + d_b)
    X = triples(n, V, 5, seed=d_a)
    Ea, Eb = energies(a.codes, a.rel, X, 1), energies(b.codes, b.rel, X, 1)
    gold = X[:, 2:3].long()
    c = w * sigmoid32(Ea).double() + (1 - w) * sigmoid32(Eb).double()
    G = c.gather(1, gold)
    same = (Ea == Ea.gather(1, gold)) & (Eb == Eb.gather(1, gold))
    tol = 1e-6
    lo = ((c > G + tol) | same).sum(1)
    hi = ((c >= G - tol) | same).sum(1)
    raw, _ = ops.EnsembleRanker(a, b, w).rank(X, 1)
    assert bool(((raw.long() >= lo) & (raw.long() <= hi)).all())
    k = 10
    excl, dense = topk_exclusions(n, V, seed=9)
    ids, u, scores = ops.EnsembleRanker(a, b, w).top_k(X, 1, k, excl)
    uref = w * torch.sigmoid(-Ea) + (1 - w) * torch.sigmoid(-Eb)
    uref = torch.where(dense, torch.full_like(uref, float("inf")), uref)
    best = torch.sort(uref, dim=1).values[:, :k]
    got = uref.gather(1, ids.clamp(min=0).long())
    real = ids >= 0
    assert torch.equal(real, torch.isfinite(best))
    assert bool(((got - best).abs()[real] <= 1e-12).all())
    assert bool(((u - got).abs()[real] <= 1e-12).all())
    assert bool((torch.diff(u.masked_fill(~real, 2.0), dim=1) >= 0).all())
    assert torch.equal(scores[real], 1 - u[real])


# ---------------------------------------------------------------------------------------------------------------------
# continuous epilogues
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [1, 129, "2w"])
@pytest.mark.parametrize("d", [4, 24, 200, 500, 512])
def test_highway_matches_float64(V, d):
    """k_gemm_tf32x3<2>: out and gate elementwise (A = c2 with K = N = d)"""
    V = rows(V, (d + 127) // 128)
    g = gen(V + d)
    c1, c2 = torch.randn(V, d, generator=g, device=DEV), torch.randn(V, d, generator=g, device=DEV)
    W, b = torch.randn(d, d, generator=g, device=DEV) / np.sqrt(d), torch.randn(d, generator=g, device=DEV)
    with torch.no_grad():
        out = ops.highway(c1, c2, W, b)
    gate = torch.sigmoid(c2.double() @ W.double() + b.double())
    want = c2.double() + gate * (c1.double() - c2.double())
    assert rel(out, want) < TOL


@pytest.mark.parametrize("V", [1, 129, "2w"])
@pytest.mark.parametrize("d,w", [(4, 4), (24, 64), (200, 68), (500, 100), (512, 64)])
def test_variational_matches_float64(V, d, w):
    """k_gemm_tf32x3<3> and k_split_b_interleave: P = (mu, log sigma) interleaved, z and the summed KL"""
    V = rows(V, (2 * w + 127) // 128)
    g = gen(V + d + w)
    H = torch.randn(V, d, generator=g, device=DEV).requires_grad_(True)
    Wm, Ws = (torch.randn(d, w, generator=g, device=DEV) / np.sqrt(d) for _ in range(2))
    bm, bs = torch.randn(w, generator=g, device=DEV), 0.1 * torch.randn(w, generator=g, device=DEV)
    eps = torch.randn(V, w, generator=g, device=DEV)
    z, kl = ops.variational(H, Wm, bm, Ws, bs, eps)
    P = z.grad_fn.saved_tensors[3]
    H64 = H.detach().double()
    mu, ls = H64 @ Wm.double() + bm.double(), H64 @ Ws.double() + bs.double()
    assert rel(P[:, 0::2], mu) < TOL and rel(P[:, 1::2], ls) < TOL
    assert rel(z, mu + torch.exp(ls) * eps.double()) < TOL
    want_kl = -0.0005 * torch.sum(1 + 2 * ls - mu ** 2 - torch.exp(2 * ls))
    assert rel(kl, want_kl) < TOL


@pytest.mark.parametrize("V,d,n", [(4, 28, 1), (124, 36, 127), (128, 96, 128), (132, 100, 129), (14541, 4, 129),
                                   (300, 500, 300)])
@pytest.mark.parametrize("grads", [True, False], ids=["loss+Gt", "loss-only"])
def test_bce_matches_float64(V, d, n, grads):
    """k_gemm_tf32x3<5>: the loss (and, with gradients, Gt through dcodes / drel) against float64; Gt = null and
    g_scale = null for the loss alone, g_scale on the device with Gt"""
    codes, relt, qs, y = t1n.case("distmult", V, d, n, seed=V + d)
    if grads:
        t1n.check("distmult", codes, relt, qs, y, 0.1)
        return
    with torch.no_grad():
        loss, _ = ops.one_to_n_loss(codes.to(DEV), relt.to(DEV), qs, torch.as_tensor(oo.bits(y), device=DEV), 0.1,
                                    "distmult", 5)
    L, _ = oo.loss(codes.to(DEV).double(), relt.to(DEV).double(), qs, torch.as_tensor(y, device=DEV), 0.1, "distmult")
    assert rel(loss, L) < TOL


def test_bce_large_energies():
    """|z| up to 50: the loss terms of saturated sigmoids, both label values"""
    codes, relt, qs, y = t1n.case("distmult", 300, 16, 60, seed=5, scale=1.5)
    z = oo.query_rows(codes.double(), relt.double(), qs, "distmult") @ codes.double().T
    assert 30 < float(z.abs().max()) < 100
    t1n.check("distmult", codes, relt, qs, y, 0.0)


@pytest.mark.parametrize("V,d_in,d_out", [(1, 4, 4), (129, 32, 124), (300, 100, 132), ("1w", 4, 128)])
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "linear"])
def test_bias_act_matches_float64(V, d_in, d_out, relu):
    """k_gemm_tf32x3<6> (K = 3 d_in): act(Cat W_cat + b) with a negative bias shift, so that ReLU clamps a good share
    of the pre-activations.  1e-4: Cat comes from the message walk's fp32 sums (the layer's bar)"""
    V = rows(V)
    R = 3
    msgs = tcg.make_messages(V, V, R, 4 * V + 8, seed=V + d_in)
    w, _ = tcg.make_inputs(V, V, R, d_in, d_out, seed=d_out, mask=False)
    w["b"] = w["b"] - 0.3
    graph = ops.Graph.from_messages(*msgs, V, V, 2 * R, device=0)
    t = {k: v.to(DEV).float().contiguous() for k, v in w.items()}
    with torch.no_grad():
        out, _ = ops.compgcn_layer(*(t[k] for k in tcg.NAMES), graph, "mult", None, 1.0, relu)
    pre, _, _ = tcg.reference(msgs, V, w, "mult", None, relu)
    want = torch.relu(pre) if relu else pre
    if relu:
        assert V * d_out < 100 or 0.2 < float((pre < 0).double().mean()) < 0.9
        assert bool((out[pre.to(DEV) < -1e-3] == 0).all())
    assert rel(out.cpu(), want) < 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# split kernels: hi + lo reconstructs the input
# ---------------------------------------------------------------------------------------------------------------------
def _tf32(x):
    return bool(((x.view(torch.int32) & 0x1fff) == 0).all())


@pytest.mark.parametrize("b_is_nk", [False, True])
def test_split_b_reconstructs(b_is_nk):
    """k_split_b (round to nearest twice): |b - hi - lo| <= 2^-22 |b|, both parts TF32, both orientations"""
    lib = _lib.load()
    M, N, K = 8, 132, 100
    A = torch.randn(M, K, device=DEV)
    B = torch.randn(*((N, K) if b_is_nk else (K, N)), device=DEV) * torch.logspace(-3, 3, K if b_is_nk else N,
                                                                                        device=DEV)
    ws = torch.full((2 * N * K,), float("nan"), device=DEV)
    C = torch.empty(M, N, device=DEV)
    _lib.check(lib.rgcn_gemm_tf32x3(ops._ptr(A), K, ops._ptr(B), B.stride(0), int(b_is_nk), ops._ptr(C), N, M, N, K, 0,
                                    ops._ptr(ws), ws.numel() * 4, ops._stream(A.device)), "rgcn_gemm_tf32x3")
    torch.cuda.synchronize()
    hi, lo = ws[:N * K].view(N, K), ws[N * K:].view(N, K)
    Bt = B if b_is_nk else B.T
    assert _tf32(hi) and _tf32(lo)
    assert bool(((hi.double() + lo.double() - Bt.double()).abs() <= 2.0 ** -22 * Bt.double().abs()).all())


def test_split_b_interleave_and_trunc_reconstruct(monkeypatch):
    """k_split_b_interleave (the forward's W_int^T, rows 2j = W_mu[:, j], 2j + 1 = W_sigma[:, j]) within 2^-22, and
    k_split_trunc (the ensemble's query rows, in place) within 2^-20 with hi the truncation of the input"""
    seen = []
    real = ops._workspace
    monkeypatch.setattr(ops, "_workspace", lambda nb, dev: seen.append(real(nb, dev)) or seen[-1])
    d, w, V = 36, 8, 5
    g = gen(1)
    Wm, Ws = torch.randn(d, w, generator=g, device=DEV), torch.randn(d, w, generator=g, device=DEV)
    ops.variational(torch.randn(V, d, generator=g, device=DEV), Wm, torch.zeros(w, device=DEV), Ws,
                    torch.zeros(w, device=DEV), torch.randn(V, w, generator=g, device=DEV))
    torch.cuda.synchronize()
    f = seen[-1].view(torch.float32)
    hi, lo = f[:2 * w * d].view(2 * w, d), f[2 * w * d:4 * w * d].view(2 * w, d)
    Wint_t = torch.stack([Wm.T, Ws.T], 1).reshape(2 * w, d)
    assert _tf32(hi) and _tf32(lo)
    assert bool(((hi.double() + lo.double() - Wint_t.double()).abs() <= 2.0 ** -22 * Wint_t.double().abs()).all())
    # the ensemble: workspace [hi_a | lo_a | hi_b | lo_b | q_a | ql_a | ...], each part 256-byte aligned
    V, d_a, d_b, n = 64, 36, 8, 5
    ca, ra = gauss_tables(V, d_a, 5, seed=2)
    cb, rb = gauss_tables(V, d_b, 5, seed=3)
    ens = ops.EnsembleRanker(ops.DistMultRanker(ca, ra), ops.DistMultRanker(cb, rb), 0.5)
    X = triples(n, V, 5, seed=1)
    ens.rank(X, 1)
    torch.cuda.synchronize()
    al = lambda nbytes: (nbytes + 255) // 256 * 256
    off = 2 * al(V * d_a * 4) + 2 * al(V * d_b * 4)
    f = ens._ws.view(torch.float32)
    qh = f[off // 4:off // 4 + n * d_a].view(n, d_a)
    ql = f[(off + al(n * d_a * 4)) // 4:(off + al(n * d_a * 4)) // 4 + n * d_a].view(n, d_a)
    q = ca[X[:, 0].long()] * ra[X[:, 1].long()]
    assert _tf32(qh) and _tf32(ql)
    assert torch.equal(qh.view(torch.int32), q.view(torch.int32) & ~0x1fff)
    assert bool(((qh.double() + ql.double() - q.double()).abs() <= 2.0 ** -20 * q.double().abs()).all())


# ---------------------------------------------------------------------------------------------------------------------
# launcher validation: refused without a launch
# ---------------------------------------------------------------------------------------------------------------------
def refused(fn):
    torch.cuda.synchronize()
    before = _lib.launch_count()
    with pytest.raises(_lib.RgcnError):
        fn()
    return _lib.launch_count() == before


def test_invalid_arguments_launch_nothing():
    lib = _lib.load()

    def gemm(M, N, K, lda, ldc):
        A = torch.zeros(M, max(lda, K), device=DEV)
        B = torch.zeros(N, K, device=DEV)
        C = torch.zeros(M, max(ldc, N), device=DEV)
        ws = torch.zeros(2 * N * K + 4, device=DEV)
        _lib.check(lib.rgcn_gemm_tf32x3(ops._ptr(A), lda, ops._ptr(B), K, 1, ops._ptr(C), ldc, M, N, K, 0,
                                        ops._ptr(ws), ws.numel() * 4, ops._stream(A.device)), "rgcn_gemm_tf32x3")

    assert refused(lambda: gemm(8, 8, 6, 6, 8))        # K % 4
    assert refused(lambda: gemm(8, 6, 8, 8, 8))        # N % 4
    assert refused(lambda: gemm(8, 8, 8, 10, 8))       # lda % 4
    assert refused(lambda: gemm(8, 8, 8, 8, 10))       # ldc % 4
    assert refused(lambda: gemm(8, 8, 0, 8, 8))        # K = 0 (see gemm_kernels.UNREACHABLE)
    codes, relt = gauss_tables(64, 6, 3, seed=1)
    X = triples(4, 64, 3, seed=1)
    assert refused(lambda: ops.DistMultRanker(codes, relt).rank(X, 1))                       # d % 4
    codes, relt = gauss_tables(64, 8, 3, seed=1)
    for k in (0, 129):
        assert refused(lambda: ops.DistMultRanker(codes, relt).top_k(X, 1, k))
        ens = ops.EnsembleRanker(ops.DistMultRanker(codes, relt), ops.DistMultRanker(codes, relt), 0.5)
        assert refused(lambda: ens.top_k(X, 1, k))
    c6, r6 = gauss_tables(64, 6, 3, seed=2)
    assert refused(lambda: ops.EnsembleRanker(ops.DistMultRanker(codes, relt), ops.DistMultRanker(c6, r6),
                                              0.5).rank(X, 1))
    assert refused(lambda: ops.highway(*(torch.zeros(5, 6, device=DEV) for _ in range(2)), torch.zeros(6, 6, device=DEV),
                                       torch.zeros(6, device=DEV)))
    H = torch.zeros(5, 8, device=DEV)
    assert refused(lambda: ops.variational(H, torch.zeros(8, 3, device=DEV), torch.zeros(3, device=DEV),
                                           torch.zeros(8, 3, device=DEV), torch.zeros(3, device=DEV),
                                           torch.zeros(5, 3, device=DEV)))     # w odd


# ---------------------------------------------------------------------------------------------------------------------
# every row launches its kernel
# ---------------------------------------------------------------------------------------------------------------------
_TRACE = """
import json
import numpy as np
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile
import gemm_kernels as gk
import one_to_n_oracle as oo
import test_gpu_compgcn as tcg
import test_gpu_gemm_epilogues as tg
from relationprediction_b200 import ops

DEV = tg.DEV


def kernels(fn):
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sorted({gk.canonical(e.name) for e in prof.events() if e.device_type == DeviceType.CUDA} - {None})


codes, relt = tg.int_tables(300, 36, 5, seed=1)
X = tg.triples(129, 300, 5, seed=1)
dm = ops.DistMultRanker(codes, relt)
ens = ops.EnsembleRanker(dm, ops.DistMultRanker(*tg.int_tables(300, 8, 5, seed=2)), 0.5)
c1n, r1n, qs, y = tg.t1n.case("distmult", 300, 24, 40)
labels = torch.as_tensor(oo.bits(y), device=DEV)
msgs = tcg.make_messages(40, 40, 3, 200, seed=1)
w, _ = tcg.make_inputs(40, 40, 3, 8, 12, seed=1, mask=False)
graph = ops.Graph.from_messages(*msgs, 40, 40, 6, device=0)
t = {k: v.to(DEV).float().contiguous() for k, v in w.items()}
A = torch.randn(129, 36, device=DEV)
calls = {
    "gemm": lambda: ops.gemm_tf32x3(A, torch.randn(36, 132, device=DEV)),
    "gemm_tn": lambda: ops.gemm_tn_tf32x3(A, torch.randn(129, 132, device=DEV)),
    "rank": lambda: dm.rank(X, 1),
    "topk": lambda: dm.top_k(X, 1, 10),
    "highway": lambda: ops.highway(*(torch.randn(129, 24, device=DEV) for _ in range(2)),
                                   torch.randn(24, 24, device=DEV), torch.randn(24, device=DEV)),
    "variational": lambda: ops.variational(torch.randn(129, 24, device=DEV), torch.randn(24, 8, device=DEV),
                                           torch.zeros(8, device=DEV), torch.randn(24, 8, device=DEV),
                                           torch.zeros(8, device=DEV), torch.randn(129, 8, device=DEV)),
    "one_to_n": lambda: ops.one_to_n_loss(c1n.to(DEV), r1n.to(DEV), qs, labels, 0.1, "distmult", 5),
    "compgcn": lambda: ops.compgcn_layer(*(t[k] for k in tcg.NAMES), graph, "mult", None, 1.0, True),
    "ensemble_rank": lambda: ens.rank(X, 1),
    "ensemble_topk": lambda: ens.top_k(X, 1, 10),
}
with torch.no_grad():
    for fn in calls.values():   # warm-up (module load)
        fn()
    torch.cuda.synchronize()
    res = {name: kernels(fn) for name, fn in calls.items()}
print("RESULT " + json.dumps(res))
"""

# the call of the trace that reaches each row's kernel
LAUNCHED_BY = {
    "k_gemm_tf32x3<0>": "gemm", "k_gemm_tf32x3<1>": "rank", "k_gemm_tf32x3<2>": "highway",
    "k_gemm_tf32x3<3>": "variational", "k_gemm_tf32x3<4>": "topk", "k_gemm_tf32x3<5>": "one_to_n",
    "k_gemm_tf32x3<6>": "compgcn", "k_gemm_tn_tf32x3": "gemm_tn", "k_gemm_ensemble<EnsRankEpi>": "ensemble_rank",
    "k_gemm_ensemble<EnsTopKEpi>": "ensemble_topk", "k_split_b": "gemm", "k_split_b_interleave": "variational",
    "k_split_trunc": "ensemble_rank",
}


def test_every_row_launches_its_kernel():
    assert set(LAUNCHED_BY) == set(gk.ROWS)
    traced = fresh_process.run_json(_TRACE)
    for kernel, call in LAUNCHED_BY.items():
        assert kernel in traced[call], (kernel, call, traced[call])
