"""The TransE decoder on the GPU: scorer forward + backward beside DistMult and RotatE, entity ranks and top-k beside a
chunked torch restatement and RotatE's ranker, and relation ranks and top-10.

Training: the shipped shape, N = 330 000 fed triples (30 000 positives, NegativeSampleRate K = 10), d = 500, FB15k-237's
V = 14 541 entities and R = 237 relations, random codes and corruptions in the sampler's layout.  A call is the loss and
the gradient of loss + 0.01 reg with the relation slice norm on.  The paths (TransE NegativeSampling and
SelfAdversarial, DistMult, RotatE) alternate --rounds times on the same X; every call is timed alone with CUDA events
after an L2 flush (a 256 MB write), and the median round is reported.

Entity queries: an FB15k-237-sized test set (--n-test = 20 466 random triples, both sides, random known masks with the
gold set), ranks and top-k at k in {1, 10, 100} through ops.TransERanker; the same ranks and top-k from a torch
restatement (torch.cdist(p=1) per chunk of queries, then >= counts or torch.topk), and RotatE's ranks on the same
shape.  Column terms: 2 n_test V d.  Relation queries: ranks and top-10 at the FB15k-237 and FB15k shapes.

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


def bits(mask, C):
    cols = torch.arange(C, device=mask.device)
    return ((mask[:, cols >> 5] >> (cols & 31)) & 1).bool()


def torch_queries(codes, rel, X, side):
    Xl = X.long()
    if side == "relation":
        return codes[Xl[:, 2]] - codes[Xl[:, 0]], Xl[:, 1]
    if side == 1:
        return codes[Xl[:, 0]] + rel[Xl[:, 1]], Xl[:, 2]
    return codes[Xl[:, 2]] - rel[Xl[:, 1]], Xl[:, 0]


def torch_ranks(table, q, gold, mask, chunk=512):
    raw, filt = [], []
    for c0 in range(0, len(q), chunk):
        D = torch.cdist(q[c0:c0 + chunk], table, p=1)
        hit = D <= D[torch.arange(len(D), device=D.device), gold[c0:c0 + chunk]][:, None]
        r = hit.sum(1)
        raw.append(r)
        filt.append(r - (hit & bits(mask[c0:c0 + chunk], len(table))).sum(1) + 1)
    return torch.cat(raw), torch.cat(filt)


def torch_top_k(table, q, mask, k, chunk=512):
    ids = []
    for c0 in range(0, len(q), chunk):
        D = torch.cdist(q[c0:c0 + chunk], table, p=1)
        D.masked_fill_(bits(mask[c0:c0 + chunk], len(table)), float("inf"))
        ids.append(torch.topk(D, k, largest=False).indices)
    return torch.cat(ids)


def test_set(rng, V, R, n, dev, relation=False):
    T = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, V, n)], 1).astype(np.int32)
    C = R if relation else V
    masks = []
    for gold in ((T[:, 1],) if relation else (T[:, 0], T[:, 2])):
        lists = [[int(x)] + rng.integers(0, C, 3).tolist() for x in gold]
        masks.append(torch.as_tensor(BilinearDiag.known_bit_mask(lists, C), device=dev))
    return torch.as_tensor(T, device=dev), masks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--V", type=int, default=14541)
    ap.add_argument("--R", type=int, default=237)
    ap.add_argument("--d", type=int, default=500)
    ap.add_argument("--n", type=int, default=30000, help="positives per step (GraphBatchSize)")
    ap.add_argument("--K", type=int, default=10, help="NegativeSampleRate")
    ap.add_argument("--n-test", type=int, default=20466, help="ranked triples (FB15k-237's test split)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_transe: no CUDA device")
    dev = torch.device("cuda:0")
    ops.set_slice_norms(True)
    g = torch.Generator(device=dev).manual_seed(0)
    V, R, d, n, K = args.V, args.R, args.d, args.n, args.K
    N = n * (K + 1)
    codes = (torch.randn(V, d, device=dev, generator=g) * 0.1).requires_grad_(True)
    rel = (torch.randn(R, d, device=dev, generator=g) * 0.1).requires_grad_(True)
    rng = np.random.default_rng(0)
    pos = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, V, n)], 1)
    neg = np.tile(pos, (K, 1))
    neg[np.arange(n * K), rng.integers(0, 2, n * K) * 2] = rng.integers(0, V, n * K)
    X = torch.as_tensor(np.concatenate([pos, neg]).astype(np.int32), device=dev)
    Y = torch.cat([torch.ones(n), torch.zeros(n * K)]).to(dev)
    name, power = card()
    out = {"gpu": name, "power_limit": power, "V": V, "R": R, "d": d, "N": N, "K": K}

    def step(fn):
        def run():
            loss, reg = fn()
            torch.autograd.grad(loss + 0.01 * reg, [codes, rel])
        return run
    paths = {"transe": step(lambda: ops.transe_score(codes, rel, X, Y, gamma=12.0)[1:]),
             "transe_self_adversarial": step(lambda: ops.self_adversarial_loss(codes, rel, X, K, 1.0, "transe",
                                                                               gamma=12.0)[:2]),
             "distmult": step(lambda: ops.distmult(codes, rel, X, Y)[1:]),
             "rotate": step(lambda: ops.rotate_score(codes, rel, X, Y, gamma=12.0)[1:])}
    times = {p: [] for p in paths}
    for _ in range(args.rounds):
        for p, fn in paths.items():
            times[p].append(timed(fn, args.warmup, args.iters))
    out["scorer_fwd_bwd_ms"] = {p: stats(ts) for p, ts in times.items()}
    del codes, rel, X, Y

    # entity queries: an FB15k-237-sized test set, both sides, filtered
    c = torch.randn(V, d, device=dev, generator=g).contiguous()
    r = (torch.randn(R, d, device=dev, generator=g) * 0.5).contiguous()
    nt = args.n_test
    Xt, masks = test_set(rng, V, R, nt, dev)
    ranker = ops.TransERanker(c, r, gamma=12.0)
    rotate = ops.RotateRanker(c, r)
    ent = {"n_test": nt, "both_sides": True, "column_terms": 2 * nt * V * d}

    def fused_rank():
        return [ranker.rank(Xt, side, masks[side]) for side in (0, 1)]

    def rotate_rank():
        return [rotate.rank(Xt, side, masks[side]) for side in (0, 1)]
    qs = [torch_queries(c, r, Xt, side) for side in (0, 1)]

    def torch_rank():
        return [torch_ranks(c, qs[side][0], qs[side][1], masks[side]) for side in (0, 1)]
    ms = {"fused": [], "rotate": []}
    for _ in range(3):
        ms["fused"].append(timed(fused_rank, 1, 3))
        ms["rotate"].append(timed(rotate_rank, 1, 3))
    ent["rank_ms"] = {p: stats(ts) for p, ts in ms.items()}
    ent["rank_ms"]["torch_restatement"] = round(timed(torch_rank, 0, 1), 1)
    a, b = fused_rank(), torch_rank()
    fa, fb = torch.cat([x[1] for x in a]).double(), torch.cat([x[1] for x in b]).double()
    ent["filtered_identical"] = round(float((fa == fb).double().mean()), 5)
    ent["filtered_mrr"] = [round(float((1 / fa).mean()), 6), round(float((1 / fb).mean()), 6)]
    ent["top_k"] = {}
    for k in (1, 10, 100):
        def fused_topk():
            return [ranker.top_k(Xt, side, k, masks[side]) for side in (0, 1)]

        def torch_topk():
            return [torch_top_k(c, qs[side][0], masks[side], k) for side in (0, 1)]
        f = [timed(fused_topk, 1, 3) for _ in range(3)]
        t = timed(torch_topk, 0, 1)
        got = torch.cat([x[0] for x in fused_topk()]).long()
        ref = torch.cat(torch_topk())
        ent["top_k"][str(k)] = {"fused_ms": stats(f), "torch_restatement_ms": round(t, 1),
                                "ids_identical": round(float((got == ref).double().mean()), 5)}
    out["entity"] = ent
    del ranker, rotate

    # relation queries at the FB15k-237 and FB15k shapes
    out["relation"] = {}
    for label, (Vs, Rs, ns) in (("FB15k-237", (14541, 237, 20466)), ("FB15k", (14951, 1345, 59071))):
        c = torch.randn(Vs, d, device=dev, generator=g).contiguous()
        r = (torch.randn(Rs, d, device=dev, generator=g) * 0.5).contiguous()
        Xr, (mr,) = test_set(rng, Vs, Rs, ns, dev, relation=True)
        rk = ops.TransERanker(c, r, gamma=12.0)
        rank_ms = [timed(lambda: rk.rank_relations(Xr, mr), 1, 3) for _ in range(3)]
        topk_ms = [timed(lambda: rk.top_k_relations(Xr, 10, mr), 1, 3) for _ in range(3)]
        q, gold = torch_queries(c, r, Xr, "relation")
        t_ms = timed(lambda: torch_ranks(r, q, gold, mr), 0, 1)
        fa = rk.rank_relations(Xr, mr)[1].double()
        fb = torch_ranks(r, q, gold, mr)[1].double()
        out["relation"][label] = {"V": Vs, "R": Rs, "n": ns, "rank_ms": stats(rank_ms), "top10_ms": stats(topk_ms),
                                  "torch_restatement_rank_ms": round(t_ms, 1),
                                  "filtered_identical": round(float((fa == fb).double().mean()), 5)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
