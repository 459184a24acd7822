"""Secondary measurements (not the headline bench): DistMult and ComplEx scorer fwd/bwd bandwidth and fused
ranking, basis layer
(WN18 shape, BASELINE configs[2]; shipped gcn_basis.exp shape), block layer train-step graph, and the one-hot
(UseInputTransform=No) first basis layer and the per-channel-coefficient basis layer (DiagonalCoefficients=Yes) at
the same shapes next to the feature-input basis layer, the highway
skip connection next to the plain GEMM of its shape, and the diagonal R-GCN layer (Name=gcn_diag) next to the basis
layer and at bench.py's synthetic shape.  `python scripts/bench_secondary.py --gcn-diag` runs only that last section;
`--variational` runs only the variational head (both variants at the FB15k-237 shape) next to an unfused torch
composition; `--topk` runs only the fused top-k prediction at the FB15k-237 test shape next to the fused rank and an
unfused torch top-k."""
import json
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
from bench import synthetic_kg  # noqa: E402
from relationprediction_b200 import _lib, ops  # noqa: E402
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag  # noqa: E402

dev = torch.device("cuda", 0)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, n=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(n):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        tot += a.elapsed_time(b)
    return tot / n


out = {}
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()


# ---- diagonal R-GCN layer (Name=gcn_diag) next to the basis layer, alternated in one run ----
def gcn_diag_walk_bytes(tr, V, R, d):
    """Algorithmic bytes of the two message walks (DESIGN.md 3).  Forward: per message the gathered H row and the
    index, weight id and norm, M (4d + 12), plus the self-loop row read and the output row written, 8 V_dst d.
    Backward: per message the gathered G row and the same 12 bytes, M (4d + 12), plus H read, dH read and written,
    12 V_src d, plus one d-wide vector reduction into dD per (source, weight id) run, 4 d each."""
    t = torch.as_tensor(tr, device=dev).long()
    s, r, o = t[:, 0], t[:, 1], t[:, 2]
    runs = torch.unique(torch.cat([s * (2 * R) + r, o * (2 * R) + R + r])).numel()
    M = 2 * len(tr)
    return M * (4 * d + 12) + 8 * V * d, M * (4 * d + 12) + 12 * V * d + runs * 4 * d, runs


def gcn_diag_case(name, V, R, E, d, B=None, skewed=True, rounds=3):
    """ops.diag_layer forward and forward + backward (ReLU on, no dropout mask, L2 flushed between calls), alternated
    `rounds` times with ops.basis_layer at B bases when B is given; medians.  Stages from the library's event marks
    in a separate profiled pass."""
    g = torch.Generator(device=dev).manual_seed(0)
    tr = synthetic_kg(V, R, E, seed=1234, skewed=skewed)
    _lib.set_option("graph_views", 1)         # the diagonal layer walks the CSR views only
    try:
        gr = ops.Graph.from_device_triples(torch.as_tensor(tr, device=dev), V, R)
    finally:
        _lib.set_option("graph_views", 3)
    H = torch.randn(V, d, device=dev, generator=g).requires_grad_(True)
    dOut = torch.randn(V, d, device=dev, generator=g)
    std = 3.0 / np.sqrt(2 * d)
    wd = [torch.randn(R, d, device=dev, generator=g).requires_grad_(True) for _ in range(2)]
    wd.append((torch.randn(d, d, device=dev, generator=g) * std).requires_grad_(True))
    wd.append(torch.zeros(d, device=dev).requires_grad_(True))
    fd = lambda: ops.diag_layer(H, wd[0], wd[1], wd[2], wd[3], gr, None, 1.0, True)
    fns = {"gcn_diag": fd}
    if B is not None:
        gb = ops.Graph.from_device_triples(torch.as_tensor(tr, device=dev), V, R)
        wb = [(torch.randn(d, B, d, device=dev, generator=g) * std).requires_grad_(True) for _ in range(2)]
        wb += [torch.randn(R, B, device=dev, generator=g).requires_grad_(True) for _ in range(2)]
        wb.append((torch.randn(d, d, device=dev, generator=g) * std).requires_grad_(True))
        fns["basis"] = lambda: ops.basis_layer(H, wb[0], wb[1], wb[2], wb[3], wb[4], gb, None, 1.0, True)

    def step(f):
        H.grad = None
        f().backward(dOut)

    def fwd(f):
        with torch.no_grad():
            f()
    ms = {k: {"fwd": [], "fwd_bwd": []} for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            ms[k]["fwd"].append(timeit(lambda: fwd(f), n=10))
            ms[k]["fwd_bwd"].append(timeit(lambda: step(f), n=10))
    med = {k: {p: float(np.median(v[p])) for p in v} for k, v in ms.items()}
    _lib.profile_enable(True)
    acc = {}
    for _ in range(5):
        flush.zero_()
        step(fd)
        torch.cuda.synchronize()
        for nm, v in _lib.profile_read():
            acc[nm] = acc.get(nm, 0.0) + v / 5
    _lib.profile_enable(False)
    by_f, by_b, runs = gcn_diag_walk_bytes(tr, V, R, d)
    t_f, t_b = acc.get("diag_walk_fwd", 0.0), acc.get("diag_walk_bwd", 0.0)
    res = {"V": V, "R": R, "E": E, "M": 2 * E, "d": d, "gpu": card, "medians_ms": med, "runs_ms": ms,
           "bwd_source_weight_runs": runs, "fwd_walk_bytes_algorithmic": by_f, "bwd_walk_bytes_algorithmic": by_b,
           "fwd_walk_TBps": by_f / t_f / 1e9 if t_f > 0 else None,
           "bwd_walk_TBps": by_b / t_b / 1e9 if t_b > 0 else None,
           "frac_of_3350_GBps": {"fwd_walk": by_f / t_f / 1e9 / 3.35 if t_f > 0 else None,
                                 "bwd_walk": by_b / t_b / 1e9 / 3.35 if t_b > 0 else None},
           "stages_ms": {k: round(v, 4) for k, v in acc.items()}}
    if B is not None:
        res["basis_B"] = B
        res["ratio_to_basis"] = {p: med["gcn_diag"][p] / med["basis"][p] for p in ("fwd", "fwd_bwd")}
    out[name] = res
    del H, dOut, wd, fns, gr
    torch.cuda.empty_cache()


def gcn_diag_section():
    gcn_diag_case("gcn_diag_fb15k237_d500 (vs basis B5)", 14541, 237, 272115, 500, B=5)
    gcn_diag_case("gcn_diag_fb15k237_d500_trainstep_E15000 (vs basis B5)", 14541, 237, 15000, 500, B=5)
    gcn_diag_case("gcn_diag_wn18_d200 (vs basis B2)", 40943, 18, 141442, 200, B=2)
    # bench.py's synthetic workload at x0.5 (uniform endpoints); the block layer's step there is 386.6 ms (DESIGN 4)
    gcn_diag_case("gcn_diag_synthetic_x0.5_V5M_E50M_d512", 5_000_000, 1000, 50_000_000, 512, skewed=False, rounds=2)


if "--gcn-diag" in sys.argv:
    gcn_diag_section()
    print(json.dumps(out, indent=1))
    sys.exit(0)


# ---- variational head (Name=variational_embedding / variational_gcn_basis) next to an unfused torch composition ----
def variational_case(name, V, d, w, rounds=3):
    """ops.variational forward and forward + backward (g = 1 on the KL term, L2 flushed between calls), alternated
    `rounds` times with the same head written as separate torch ops (two fp32 matmuls, exp, multiply-add, the KL
    reduction; autograd backward); medians.  d = 0 is the embedding variant (mu = W_mu, log sigma = W_sigma [V, w])."""
    g = torch.Generator(device=dev).manual_seed(0)
    r = lambda *s, sc=1.0: (torch.randn(*s, device=dev, generator=g) * sc).requires_grad_(True)
    if d:
        H, Wm, Ws = r(V, d), r(d, w, sc=1 / np.sqrt(d)), r(d, w, sc=0.5 / np.sqrt(d))
    else:
        H, Wm, Ws = None, r(V, w), r(V, w, sc=0.5)
    bm, bs = r(w), r(w, sc=0.2)
    eps, dz = torch.randn(V, w, device=dev, generator=g), torch.randn(V, w, device=dev, generator=g)

    def unfused():
        mu, ls = (H @ Wm + bm, H @ Ws + bs) if d else (Wm, Ws)
        return mu + torch.exp(ls) * eps, -0.0005 * torch.sum(1 + 2 * ls - mu * mu - torch.exp(2 * ls))
    fns = {"fused": lambda: ops.variational(H, Wm, bm, Ws, bs, eps), "unfused_torch": unfused}

    def step(f):
        z, kl = f()
        torch.autograd.backward([z, kl], [dz, torch.ones((), device=dev)])

    def fwd(f):
        with torch.no_grad():
            f()
    with torch.no_grad():
        zf, klf = fns["fused"]()
        zu, klu = unfused()
    ms = {k: {"fwd": [], "fwd_bwd": []} for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            ms[k]["fwd"].append(timeit(lambda: fwd(f), n=20))
            ms[k]["fwd_bwd"].append(timeit(lambda: step(f), n=20))
    med = {k: {p: float(np.median(v[p])) for p in v} for k, v in ms.items()}
    _lib.profile_enable(True)
    acc = {}
    for _ in range(5):
        flush.zero_()
        step(fns["fused"])
        torch.cuda.synchronize()
        for nm, v in _lib.profile_read():
            acc[nm] = acc.get(nm, 0.0) + v / 5
    _lib.profile_enable(False)
    out[name] = {"V": V, "d": d, "w": w, "gpu": card, "medians_ms": med, "runs_ms": ms,
                 "speedup_vs_unfused": {p: med["unfused_torch"][p] / med["fused"][p] for p in ("fwd", "fwd_bwd")},
                 "max_rel_z_vs_unfused": float((zf - zu).abs().max() / zu.abs().max()),
                 "rel_kl_vs_unfused": float((klf - klu).abs() / klu.abs()),
                 "stages_ms": {k: round(v, 4) for k, v in acc.items()}}
    torch.cuda.empty_cache()


if "--variational" in sys.argv:
    variational_case("variational_gcn_fb15k237_V14541_d500_w500", 14541, 500, 500)
    variational_case("variational_embedding_fb15k237_V14541_w500", 14541, 0, 500)
    print(json.dumps(out, indent=1))
    sys.exit(0)

# ---- top-k prediction (distmult_topk / rgcn_complex_topk) next to the fused rank and an unfused torch top-k ----
def topk_case(name, ranker_cls, V, d, n, ks, chunk=4096, rounds=3):
    """All n queries on both sides: the fused top-k, the fused rank of the same queries (rank_all's loop) and the
    unfused torch path (q @ codes.T, masked fill, torch.topk; query rows formed by torch), alternated `rounds`
    times, L2 flushed between calls; medians.  Every path gets the same random exclusion masks (~20 entities a
    row).  Algorithmic bytes of the fused top-k: codes read once per 128-query M tile (hi + lo planes), the query
    rows and masks, the candidate slab written and read back, the answers; flops 2 n V d x 3 (3xTF32)."""
    g = torch.Generator(device=dev).manual_seed(0)
    cd = torch.randn(V, d, device=dev, generator=g) * 0.3
    rl = torch.randn(237, d, device=dev, generator=g)
    Xq = torch.stack([torch.randint(0, V, (n,), device=dev, generator=g), torch.randint(0, 237, (n,), device=dev, generator=g),
                      torch.randint(0, V, (n,), device=dev, generator=g)], 1).int().contiguous()
    words = (V + 31) // 32
    rng = np.random.RandomState(0)
    excl = rng.randint(0, V, (n, 20))
    mask = torch.as_tensor(BilinearDiag.known_bit_mask(list(excl), V), device=dev)
    dense = torch.zeros(n, V, dtype=torch.bool, device=dev)
    dense[torch.arange(n, device=dev).repeat_interleave(20), torch.as_tensor(excl.reshape(-1), device=dev)] = True
    complex_ = ranker_cls is ops.ComplexRanker

    def torch_q(X, side):
        kept = cd[X[:, 2].long()] if side == 0 else cd[X[:, 0].long()]
        b = rl[X[:, 1].long()]
        if not complex_:
            return b * kept
        h = d // 2
        kr, ki, br, bi = kept[:, :h], kept[:, h:], b[:, :h], b[:, h:]
        if side == 0:
            return torch.cat([br * kr + bi * ki, br * ki - bi * kr], 1)
        return torch.cat([kr * br - ki * bi, ki * br + kr * bi], 1)

    res = {"V": V, "d": d, "n": n, "gpu": card, "decoder": "complex" if complex_ else "distmult", "k": {}}
    for k in ks:
        def fused():
            rk = ranker_cls(cd, rl)
            for c0 in range(0, n, chunk):
                for side in (0, 1):
                    rk.top_k(Xq[c0:c0 + chunk], side, k, mask[c0:c0 + chunk])

        def rank():
            rk = ranker_cls(cd, rl)
            for c0 in range(0, n, chunk):
                for side in (0, 1):
                    rk.rank(Xq[c0:c0 + chunk], side, mask[c0:c0 + chunk])

        def unfused():
            with torch.no_grad():
                for c0 in range(0, n, chunk):
                    for side in (0, 1):
                        e = torch_q(Xq[c0:c0 + chunk], side) @ cd.T
                        e.masked_fill_(dense[c0:c0 + chunk], float("-inf"))
                        torch.topk(e, k, dim=1)
        fns = {"fused_topk": fused, "fused_rank": rank, "unfused_torch_topk": unfused}
        ms = {nm: [] for nm in fns}
        for _ in range(rounds):
            for nm, f in fns.items():
                ms[nm].append(timeit(f, n=3, warm=1))
        med = {nm: float(np.median(v)) for nm, v in ms.items()}
        tn = (V + 127) // 128
        by = 2 * (2 * n * V * d * 4 / 128) + 2 * n * (d * 4 + words * 4 + 2 * tn * k * 8 + k * 8)
        fl = 2 * 2 * n * V * d * 3
        res["k"][k] = {"medians_ms": med, "runs_ms": ms, "topk_over_rank": med["fused_topk"] / med["fused_rank"],
                       "speedup_vs_unfused": med["unfused_torch_topk"] / med["fused_topk"],
                       "bytes_algorithmic": by, "flops": fl, "topk_TFLOPs": fl / med["fused_topk"] / 1e9}
    out[name] = res
    del cd, rl, Xq, dense, mask
    torch.cuda.empty_cache()


if "--topk" in sys.argv:
    for cls in (ops.DistMultRanker, ops.ComplexRanker):
        topk_case("topk_fb15k237_%s_V14541_d500_n20466_both_sides" % cls.__name__, cls, 14541, 500, 20466, (1, 10, 100))
    print(json.dumps(out, indent=1))
    sys.exit(0)

# ---- DistMult: FB15k-237 train-step decoder shape: N = 330000 triples, d = 500 ----
V, d, N = 14541, 500, 330000
g = torch.Generator(device=dev).manual_seed(0)
codes = torch.randn(V, d, device=dev, generator=g).requires_grad_(True)
rel = torch.randn(V, d, device=dev, generator=g).requires_grad_(True)
X = torch.stack([torch.randint(0, V, (N,), device=dev, generator=g), torch.randint(0, 237, (N,), device=dev, generator=g),
                 torch.randint(0, V, (N,), device=dev, generator=g)], 1).int().contiguous()
Y = (torch.rand(N, device=dev, generator=g) < 0.09).float()


def dm_fwd():
    with torch.no_grad():
        ops.distmult(codes, rel, X, Y)


def dm_fwd_bwd():
    codes.grad = None
    rel.grad = None
    e, l, r = ops.distmult(codes, rel, X, Y)
    (l + 0.01 * r).backward()


t_f = timeit(dm_fwd)
t_fb = timeit(dm_fwd_bwd)
alg_f = N * (12 * d + 16)
alg_b = N * (12 * d + 16) + N * 12 * d * 2
out["distmult"] = {"N": N, "d": d, "fwd_ms": t_f, "fwd_bwd_ms": t_fb, "fwd_GBps_algorithmic": alg_f / t_f / 1e6,
                   "bwd_GBps_algorithmic": alg_b / max(t_fb - t_f, 1e-6) / 1e6,
                   "note": "codes (29 MB) are L2-resident: gathers run above the HBM roofline"}
# DistMult on a table larger than L2
V2, N2 = 1_000_000, 2_000_000
codes2 = torch.randn(V2, 512, device=dev, generator=g)
rel2 = torch.randn(1000, 512, device=dev, generator=g)
X2 = torch.stack([torch.randint(0, V2, (N2,), device=dev, generator=g), torch.randint(0, 1000, (N2,), device=dev, generator=g),
                  torch.randint(0, V2, (N2,), device=dev, generator=g)], 1).int().contiguous()
Y2 = (torch.rand(N2, device=dev, generator=g) < 0.09).float()
t2 = timeit(lambda: ops.distmult(codes2, rel2, X2, Y2), n=5)
out["distmult_hbm"] = {"V": V2, "N": N2, "d": 512, "fwd_ms": t2, "fwd_GBps_algorithmic": N2 * (12 * 512 + 16) / t2 / 1e6,
                       "frac_of_measured_hbm_6569.6": N2 * (8 * 512 + 16) / t2 / 1e6 / 6569.6,
                       "note": "2 of the 3 rows per triple come from HBM (entity table 2 GB), the relation row from L2"}
del codes2, rel2, X2, Y2


# ---- ComplEx at the same shape (complex.exp: d = 500, so the imaginary half is 8-byte aligned: float2 path) ----
def cx_fwd():
    with torch.no_grad():
        ops.complex_score(codes, rel, X, Y)


def cx_fwd_bwd():
    codes.grad = None
    rel.grad = None
    e, l, r = ops.complex_score(codes, rel, X, Y)
    (l + 0.01 * r).backward()


# fused ranking of the FB15k-237 test set (20466 triples) under both corruptions, one split for all chunks
n_rank = 20466
X_rank = torch.stack([torch.randint(0, V, (n_rank,), device=dev, generator=g),
                      torch.randint(0, 237, (n_rank,), device=dev, generator=g),
                      torch.randint(0, V, (n_rank,), device=dev, generator=g)], 1).int().contiguous()
codes_d, rel_d = codes.detach(), rel.detach()


def rank_all(ranker_cls, chunk=4096):
    ranker = ranker_cls(codes_d, rel_d)
    for c0 in range(0, n_rank, chunk):
        for side in (0, 1):
            ranker.rank(X_rank[c0:c0 + chunk], side, None)


# the two decoders alternate in one run so that both see the same card state
t_dm_f, t_dm_fb, t_cx_f, t_cx_fb = timeit(dm_fwd), timeit(dm_fwd_bwd), timeit(cx_fwd), timeit(cx_fwd_bwd)
t_dm_r, t_cx_r = timeit(lambda: rank_all(ops.DistMultRanker), n=5), timeit(lambda: rank_all(ops.ComplexRanker), n=5)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                     capture_output=True, text=True).stdout.strip()
out["complex"] = {"N": N, "d": d, "V": V, "gpu": gpu, "fwd_ms": t_cx_f, "fwd_bwd_ms": t_cx_fb,
                  "fwd_GBps_algorithmic": alg_f / t_cx_f / 1e6,
                  "bwd_GBps_algorithmic": alg_b / max(t_cx_fb - t_cx_f, 1e-6) / 1e6,
                  "rank_triples": n_rank, "rank_both_sides_ms": t_cx_r,
                  "distmult_same_run": {"fwd_ms": t_dm_f, "fwd_bwd_ms": t_dm_fb, "rank_both_sides_ms": t_dm_r},
                  "ratio_to_distmult": {"fwd": t_cx_f / t_dm_f, "fwd_bwd": t_cx_fb / t_dm_fb, "rank": t_cx_r / t_dm_r}}


# ---- layers ----
def layer_case(name, V, R, E, d, B, variant, skewed):
    tr = synthetic_kg(V, R, E, seed=1234, skewed=skewed)
    gr = ops.Graph(tr, V, R, device=0)
    H = torch.randn(V, d, device=dev, generator=g).requires_grad_(True)
    dOut = torch.randn(V, d, device=dev, generator=g)
    if variant == "block":
        s = d // B
        std = 3.0 / np.sqrt(R + s)
        ws = [(torch.randn(R, B, s, s, device=dev, generator=g) * std).requires_grad_(True) for _ in range(2)]
        ws.append((torch.randn(d, d, device=dev, generator=g) * std).requires_grad_(True))
        f = lambda: ops.block_layer(H, ws[0], ws[1], ws[2], gr, B, None, 1.0, True)
    elif variant == "times_diag":     # DiagonalCoefficients=Yes: [R, B, d] coefficient tables and a bias
        std = 3.0 / np.sqrt(2 * d)
        ws = [(torch.randn(d, B, d, device=dev, generator=g) * std).requires_grad_(True) for _ in range(2)]
        ws += [torch.randn(R, B, d, device=dev, generator=g).requires_grad_(True) for _ in range(2)]
        ws.append((torch.randn(d, d, device=dev, generator=g) * std).requires_grad_(True))
        ws.append(torch.zeros(d, device=dev).requires_grad_(True))
        f = lambda: ops.basis_diagcoef_layer(H, ws[0], ws[1], ws[2], ws[3], ws[4], ws[5], gr, None, 1.0, True)
    else:
        std = 3.0 / np.sqrt(2 * d)
        ws = [(torch.randn(d, B, d, device=dev, generator=g) * std).requires_grad_(True) for _ in range(2)]
        ws += [torch.randn(R, B, device=dev, generator=g).requires_grad_(True) for _ in range(2)]
        ws.append((torch.randn(d, d, device=dev, generator=g) * std).requires_grad_(True))
        f = lambda: ops.basis_layer(H, ws[0], ws[1], ws[2], ws[3], ws[4], gr, None, 1.0, True)

    def step():
        H.grad = None
        for w in ws:
            w.grad = None
        f().backward(dOut)
    ms = timeit(step, n=10)
    with torch.no_grad():
        ms_f = timeit(lambda: f(), n=10)
    _lib.profile_enable(True)
    acc = {}
    for _ in range(5):
        flush.zero_()
        step()
        torch.cuda.synchronize()
        for nm, v in _lib.profile_read():
            acc[nm] = acc.get(nm, 0.0) + v / 5
    _lib.profile_enable(False)
    out[name] = {"V": V, "R": R, "E": E, "d": d, "B": B, "variant": variant, "fwd_ms": ms_f, "fwd_bwd_ms": ms,
                 "M_edges_per_s": E / ms / 1e3, "stages_ms": {k: round(v, 4) for k, v in acc.items()}}
    if variant == "times_diag":
        # the forward walk gathers one P_dir row (B*d floats) plus its sigmoid row (L2-resident) per message and
        # reads the index, weight id and norm: M * (4 B d + 12) bytes from memory
        walk = 2 * E * (4 * B * d + 12)
        t_walk = acc.get("diagcoef_walk_fwd", 0.0)
        out[name].update({"gpu": gpu, "fwd_walk_bytes_algorithmic": walk,
                          "fwd_walk_GBps_algorithmic": walk / t_walk / 1e6 if t_walk > 0 else None})


def onehot_case(name, V, R, E, d, B):
    """The featureless first basis layer (ops.basis_onehot_layer), no dropout mask, ReLU on.  Algorithmic bytes:
    forward = distinct (source, direction) table rows * B*d*4 + M*(4d + 12) (one 4d-byte reduction and the index,
    weight id and norm per message) + 4 [V, d] passes (W_self copy, ReLU); backward = the same table rows (dC) and
    M*(4d + 12) (G gathers) + both dW tables written in full + 3 [V, d] passes (dOut and out read, G = dW_self
    written)."""
    tr = synthetic_kg(V, R, E, seed=1234, skewed=True)
    gr = ops.Graph(tr, V, R, device=0)
    std = 3.0 / np.sqrt(V + d)
    ws = [(torch.randn(V, B, d, device=dev, generator=g) * std).requires_grad_(True) for _ in range(2)]
    ws += [torch.randn(R, B, device=dev, generator=g).requires_grad_(True) for _ in range(2)]
    ws.append((torch.randn(V, d, device=dev, generator=g) * std).requires_grad_(True))
    dOut = torch.randn(V, d, device=dev, generator=g)
    f = lambda: ops.basis_onehot_layer(ws[0], ws[1], ws[2], ws[3], ws[4], gr, None, 1.0, True)

    def step():
        for w in ws:
            w.grad = None
        f().backward(dOut)
    ms = timeit(step, n=10)
    with torch.no_grad():
        ms_f = timeit(lambda: f(), n=10)
    _lib.profile_enable(True)
    acc = {}
    for _ in range(5):
        flush.zero_()
        step()
        torch.cuda.synchronize()
        for nm, v in _lib.profile_read():
            acc[nm] = acc.get(nm, 0.0) + v / 5
    _lib.profile_enable(False)
    M = 2 * E
    rows = len(np.unique(tr[:, 0])) + len(np.unique(tr[:, 2]))     # (source, direction) pairs with messages
    table = rows * B * d * 4
    msgs = M * (4 * d + 12)
    alg_f = table + msgs + 4 * V * d * 4
    alg_b = table + msgs + 2 * V * B * d * 4 + 3 * V * d * 4
    out[name] = {"V": V, "R": R, "E": E, "M": M, "d": d, "B": B, "gpu": gpu, "fwd_ms": ms_f, "fwd_bwd_ms": ms,
                 "source_dir_rows": rows, "fwd_bytes_algorithmic": alg_f, "bwd_bytes_algorithmic": alg_b,
                 "fwd_GBps_algorithmic": alg_f / ms_f / 1e6, "bwd_GBps_algorithmic": alg_b / max(ms - ms_f, 1e-6) / 1e6,
                 "frac_of_3350_GBps": {"fwd": alg_f / ms_f / 1e6 / 3350, "bwd": alg_b / max(ms - ms_f, 1e-6) / 1e6 / 3350},
                 "stages_ms": {k: round(v, 4) for k, v in acc.items()}}


layer_case("wn18_basis_B2_d200 (BASELINE configs[2])", 40943, 18, 141442, 200, 2, "basis", True)
layer_case("fb15k237_basis_B5_d500 (shipped gcn_basis.exp)", 14541, 237, 272115, 500, 5, "basis", True)
layer_case("fb15k237_basis_B5_d500_trainstep_E15000", 14541, 237, 15000, 500, 5, "basis", True)
layer_case("wn18_times_diag_B2_d200 (DiagonalCoefficients=Yes)", 40943, 18, 141442, 200, 2, "times_diag", True)
layer_case("fb15k237_times_diag_B5_d500 (gcn_basis.exp, DiagonalCoefficients=Yes)", 14541, 237, 272115, 500, 5,
           "times_diag", True)
layer_case("fb15k237_times_diag_B5_d500_trainstep_E15000", 14541, 237, 15000, 500, 5, "times_diag", True)
onehot_case("wn18_onehot_B2_d200 (UseInputTransform=No)", 40943, 18, 141442, 200, 2)
onehot_case("fb15k237_onehot_B5_d500 (gcn_basis.exp, UseInputTransform=No)", 14541, 237, 272115, 500, 5)
onehot_case("fb15k237_onehot_B5_d500_trainstep_E15000", 14541, 237, 15000, 500, 5)
layer_case("fb15k237_block_trainstep_E15000", 14541, 237, 15000, 500, 100, "block", True)
layer_case("fb15k_block_B100_d500 (BASELINE configs[3] shape, 1 GPU)", 14951, 1345, 483142, 500, 100, "block", True)


# ---- highway skip connection (SkipConnections=Highway) next to the plain 3xTF32 GEMM of the same [V,d]x[d,d] shape ----
def highway_case(name, V, d):
    """ops.highway forward (gate GEMM + blend epilogue) and forward+backward (prologue, dc2 += dz W^T, dW = c2^T dz),
    alternating with rgcn_gemm_tf32x3 (C = A W) in the same run.  Algorithmic bytes: forward reads c1, c2 and writes
    out, g (4 [V, d] streams); backward reads c1, c2, g, dOut and writes dc1, dc2 (6 streams).  Flops: 2 V d^2 forward,
    4 V d^2 backward.  Share of peak: the larger of bytes / 3.35 TB/s and flops / (495 / 3) TFLOP/s (three TF32 MMAs
    per product) over the measured time."""
    c1 = torch.randn(V, d, device=dev, generator=g).requires_grad_(True)
    c2 = torch.randn(V, d, device=dev, generator=g).requires_grad_(True)
    W = (torch.randn(d, d, device=dev, generator=g) / np.sqrt(d)).requires_grad_(True)
    b = torch.ones(d, device=dev).requires_grad_(True)
    dOut = torch.randn(V, d, device=dev, generator=g)
    C = torch.empty(V, d, device=dev)
    A, Wd = c2.detach(), W.detach()

    def step():
        for t in (c1, c2, W, b):
            t.grad = None
        ops.highway(c1, c2, W, b).backward(dOut)

    def fwd():
        with torch.no_grad():
            ops.highway(c1, c2, W, b)
    gemm = lambda: ops.gemm_tf32x3(A, Wd, out=C)
    ms = {"gemm": [], "fwd": [], "fwd_bwd": []}
    for _ in range(3):                      # alternate, so that all three see the same card state
        ms["gemm"].append(timeit(gemm, n=10))
        ms["fwd"].append(timeit(fwd, n=10))
        ms["fwd_bwd"].append(timeit(step, n=5))
    t_g, t_f, t_fb = (float(np.median(ms[k])) for k in ("gemm", "fwd", "fwd_bwd"))
    _lib.profile_enable(True)
    acc = {}
    for _ in range(3):
        flush.zero_()
        step()
        torch.cuda.synchronize()
        for nm, v in _lib.profile_read():
            acc[nm] = acc.get(nm, 0.0) + v / 3
    _lib.profile_enable(False)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    by_f, by_b = 4 * V * d * 4, 6 * V * d * 4
    fl_f, fl_b = 2 * V * d * d, 4 * V * d * d
    bound = lambda by, fl: max(by / 3.35e12, fl / 165e12) * 1e3       # ms
    out[name] = {"V": V, "d": d, "gpu": card, "gemm_ms": t_g, "fwd_ms": t_f, "fwd_bwd_ms": t_fb,
                 "runs_ms": ms, "fwd_over_gemm": t_f / t_g, "fwd_bwd_over_gemm": t_fb / t_g,
                 "fwd_bytes_algorithmic": by_f, "bwd_bytes_algorithmic": by_b, "fwd_flops": fl_f, "bwd_flops": fl_b,
                 "fwd_GBps_algorithmic": by_f / t_f / 1e6, "fwd_TFLOPs": fl_f / t_f / 1e9,
                 "share_of_peak": {"fwd": bound(by_f, fl_f) / t_f, "bwd": bound(by_b, fl_b) / max(t_fb - t_f, 1e-6)},
                 "stages_ms": {k: round(v, 4) for k, v in acc.items()}}
    del c1, c2, W, b, dOut, C, A, Wd


highway_case("highway_fb15k237_V14541_d500", 14541, 500)
highway_case("highway_V2M_d512", 2_000_000, 512)
gcn_diag_section()
print(json.dumps(out, indent=1))
