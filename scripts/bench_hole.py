"""The HolE decoder on the GPU: training calls beside ComplEx and DistMult under all three objectives, entity ranks and
top-k and relation ranks and top-10 beside ComplEx, the cost of the basis transform on its own, and one large-table
training row.  The protocol is scripts/bench_quate.py's.

Training: the shipped shape, N = 330 000 fed triples (30 000 positives, NegativeSampleRate K = 10), d = 500,
FB15k-237's V = 14 541 entities and R = 237 relations, random codes and corruptions in the sampler's layout.  A call
is the loss and the gradient of loss + 0.01 reg with respect to the raw tables, with the relation slice norm on:
NegativeSampling and SelfAdversarial over the N fed triples, 1-N over the de-duplicated queries of the 30 000 positives
with their label rows (label smoothing 0.1).  A HolE call includes both forward transforms and both inverse transforms
of the gradients, as a training step of the decoder runs them.  The paths alternate --rounds times on the same inputs;
every call is timed alone with CUDA events after an L2 flush (a 256 MB write), and the median round is reported.

Entity queries: an FB15k-237-sized test set (--n-test = 20 466 random triples, both sides, random known masks with the
gold set), filtered ranks and top-k at k in {1, 10, 100}, on tables the decoder has transformed once.  Every decoder's
query tables are scaled so that its energies have standard deviation 4 (`matched`).  Relation
queries: filtered ranks and top-10 at the FB15k-237 and FB15k shapes.  Transform: x U of the FB15k-237 entity table and
relation table, forward and inverse.  Large table: NegativeSampling calls at V = 1 000 000 (the same N), where the
transforms of the whole table are a larger share of the step.

Prints one JSON line with the card's name and power limit; writes nothing."""
import argparse
import json
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from relationprediction_b200 import ops  # noqa: E402
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


_FLUSH = None


def timed(fn, warmup, iters):
    """mean ms of fn over iters calls, each after an L2 flush, each timed alone with CUDA events"""
    global _FLUSH
    if _FLUSH is None:
        _FLUSH = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")
    for _ in range(warmup):
        fn()
    ev = []
    for _ in range(iters):
        _FLUSH.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        ev.append((e0, e1))
    torch.cuda.synchronize()
    return float(np.mean([a.elapsed_time(b) for a, b in ev]))


def stats(ts):
    return {"median": round(float(np.median(ts)), 4), "spread": [round(min(ts), 4), round(max(ts), 4)]}


def test_set(rng, V, R, n, dev, relation=False):
    T = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, V, n)], 1).astype(np.int32)
    C = R if relation else V
    masks = []
    for gold in ((T[:, 1],) if relation else (T[:, 0], T[:, 2])):
        lists = [[int(x)] + rng.integers(0, C, 3).tolist() for x in gold]
        masks.append(torch.as_tensor(BilinearDiag.known_bit_mask(lists, C), device=dev))
    return torch.as_tensor(T, device=dev), masks


def fed_triples(rng, V, R, n, K, dev):
    pos = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, V, n)], 1)
    neg = np.tile(pos, (K, 1))
    neg[np.arange(n * K), rng.integers(0, 2, n * K) * 2] = rng.integers(0, V, n * K)
    X = torch.as_tensor(np.concatenate([pos, neg]).astype(np.int32), device=dev)
    Y = torch.cat([torch.ones(n), torch.zeros(n * K)]).to(dev)
    return pos, X, Y


def matched(c, r, score, rng, std=4.0):
    """(c, r) scaled by one factor so that the decoder's energies over 4096 random triples have standard deviation
    `std`, as a trained model's do.  Unscaled N(0, 1) rows give HolE energies of standard deviation d and ComplEx ones
    of about sqrt(d): most float32 sigmoids, which the rank epilogue compares, are then 1.0, and the epilogue's work
    depends on how many candidates tie with the gold.  Matched spreads compare the decoders on the same work."""
    V, R = c.shape[0], r.shape[0]
    Xs = torch.as_tensor(np.stack([rng.integers(0, V, 4096), rng.integers(0, R, 4096), rng.integers(0, V, 4096)],
                                  1).astype(np.int32), device=c.device)
    with torch.no_grad():
        e = score(c, r, Xs)[0]
    s = (std / float(e.std())) ** (1.0 / 3.0)   # the energy is linear in each of its three rows
    return (c * s).contiguous(), (r * s).contiguous()


def hole(fn):
    """fn over the tables in the HolE basis: the decoder's two transforms, and their inverses in the backward"""
    return lambda codes, rel, *a: fn(ops.hole_transform(codes), ops.hole_transform(rel), *a)


SCORERS = {"hole": hole(ops.hole_score), "complex": ops.complex_score, "distmult": ops.distmult}


def training_paths(codes, rel, X, Y, K, R, queries=None, labels=None):
    def step(fn):
        def run():
            loss, reg = fn()
            torch.autograd.grad(loss + 0.01 * reg, [codes, rel])
        return run
    paths = {}
    for dec, score in SCORERS.items():
        sa = hole(ops.self_adversarial_loss) if dec == "hole" else ops.self_adversarial_loss
        onen = hole(ops.one_to_n_loss) if dec == "hole" else ops.one_to_n_loss
        paths[dec + "/NegativeSampling"] = step(lambda score=score: score(codes, rel, X, Y)[1:])
        if queries is None:
            continue
        paths[dec + "/SelfAdversarial"] = step(lambda sa=sa, dec=dec: sa(codes, rel, X, K, 1.0, dec)[:2])
        paths[dec + "/1-N"] = step(lambda onen=onen, dec=dec: onen(codes, rel, queries, labels, 0.1, dec, R))
    return paths


def run_rounds(paths, rounds, warmup, iters):
    times = {p: [] for p in paths}
    for _ in range(rounds):
        for p, fn in paths.items():
            times[p].append(timed(fn, warmup if not p.endswith("1-N") else 1, iters if not p.endswith("1-N") else 3))
    return {p: stats(ts) for p, ts in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--V", type=int, default=14541)
    ap.add_argument("--R", type=int, default=237)
    ap.add_argument("--d", type=int, default=500)
    ap.add_argument("--n", type=int, default=30000, help="positives per step (GraphBatchSize)")
    ap.add_argument("--K", type=int, default=10, help="NegativeSampleRate")
    ap.add_argument("--n-test", type=int, default=20466, help="ranked triples (FB15k-237's test split)")
    ap.add_argument("--large-V", type=int, default=1000000, help="entities of the large-table training row")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_hole: no CUDA device")
    dev = torch.device("cuda:0")
    ops.set_slice_norms(True)
    g = torch.Generator(device=dev).manual_seed(0)
    V, R, d, n, K = args.V, args.R, args.d, args.n, args.K
    rng = np.random.default_rng(0)
    codes = (torch.randn(V, d, device=dev, generator=g) * 0.1).requires_grad_(True)
    rel = (torch.randn(R, d, device=dev, generator=g) * 0.1).requires_grad_(True)
    pos, X, Y = fed_triples(rng, V, R, n, K, dev)
    queries = ops.one_to_n_queries(pos)
    labels = ops.OneToNLabels(pos, V, R, dev).rows(queries)
    name, power = card()
    out = {"gpu": name, "power_limit": power, "V": V, "R": R, "d": d, "N": X.shape[0], "K": K,
           "one_to_n_queries": len(queries)}
    out["training_call_ms"] = run_rounds(training_paths(codes, rel, X, Y, K, R, queries, labels), args.rounds,
                                         args.warmup, args.iters)

    # the transform on its own: the entity and relation tables, forward and inverse (the basis is cached)
    c, r = codes.detach(), rel.detach()
    out["transform_ms"] = {
        "entities_forward": stats([timed(lambda: ops.hole_transform(c), 3, 10) for _ in range(3)]),
        "entities_inverse": stats([timed(lambda: ops.hole_transform(c, inverse=True), 3, 10) for _ in range(3)]),
        "relations_forward": stats([timed(lambda: ops.hole_transform(r), 3, 10) for _ in range(3)])}
    del codes, rel, X, Y, labels, c, r

    # entity queries: an FB15k-237-sized test set, both sides, filtered; HolE on tables transformed once
    c = torch.randn(V, d, device=dev, generator=g).contiguous()
    r = (torch.randn(R, d, device=dev, generator=g) * 0.5).contiguous()
    Xt, masks = test_set(rng, V, R, args.n_test, dev)
    ct, rt = matched(ops.hole_transform(c), ops.hole_transform(r), ops.hole_score, rng)
    rankers = {"hole": ops.HolERanker(ct, rt), "complex": ops.ComplexRanker(*matched(c, r, ops.complex_score, rng)),
               "distmult": ops.DistMultRanker(*matched(c, r, ops.distmult, rng))}
    rank_ms, topk_ms = {}, {str(k): {} for k in (1, 10, 100)}
    for dec, rk in rankers.items():
        rank_ms[dec] = stats([timed(lambda: [rk.rank(Xt, s, masks[s]) for s in (0, 1)], 1, 3) for _ in range(3)])
        for k in (1, 10, 100):
            topk_ms[str(k)][dec] = stats([timed(lambda: [rk.top_k(Xt, s, k, masks[s]) for s in (0, 1)], 1, 3)
                                          for _ in range(3)])
    out["entity"] = {"n_test": args.n_test, "both_sides": True, "rank_ms": rank_ms, "top_k_ms": topk_ms}

    # relation queries at the FB15k-237 and FB15k shapes
    out["relation"] = {}
    for label, (Vs, Rs, ns) in (("FB15k-237", (14541, 237, 20466)), ("FB15k", (14951, 1345, 59071))):
        c = torch.randn(Vs, d, device=dev, generator=g).contiguous()
        r = (torch.randn(Rs, d, device=dev, generator=g) * 0.5).contiguous()
        Xr, (mr,) = test_set(rng, Vs, Rs, ns, dev, relation=True)
        res = {"V": Vs, "R": Rs, "n": ns}
        ct, rt = matched(ops.hole_transform(c), ops.hole_transform(r), ops.hole_score, rng)
        for dec, rk in (("hole", ops.HolERanker(ct, rt)),
                        ("complex", ops.ComplexRanker(*matched(c, r, ops.complex_score, rng)))):
            res[dec] = {"rank_ms": stats([timed(lambda: rk.rank_relations(Xr, mr), 1, 3) for _ in range(3)]),
                        "top10_ms": stats([timed(lambda: rk.top_k_relations(Xr, 10, mr), 1, 3) for _ in range(3)])}
        out["relation"][label] = res
    del c, r, ct, rt, rankers

    # one large-table training row: NegativeSampling at V = large_V, the same fed triples' shape
    VL = args.large_V
    codes = (torch.randn(VL, d, device=dev, generator=g) * 0.1).requires_grad_(True)
    rel = (torch.randn(R, d, device=dev, generator=g) * 0.1).requires_grad_(True)
    _, X, Y = fed_triples(rng, VL, R, n, K, dev)
    large = run_rounds(training_paths(codes, rel, X, Y, K, R), 3, 2, 5)
    c = codes.detach()
    large["hole/transform_entities_forward"] = stats([timed(lambda: ops.hole_transform(c), 2, 5) for _ in range(3)])
    out["large_table"] = {"V": VL, "training_call_ms": large}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
