"""Fused R-GCN+ ensemble ranking next to two single-model fused rankings and the unfused torch composition, at the
FB15k-237 and FB15k test shapes (both sides, d_A = d_B = 500, DistMult members, random codes, seeded):

  python scripts/bench_ensemble_rank.py [--reps N] [--chunk C] [--topk K] [--relations]

  fused ensemble   ops.EnsembleRanker.rank, both sides (two prepare kernels, the dual-accumulator rank GEMM)
  two singles      DistMultRanker.rank of member A plus that of member B, both sides
  torch            per chunk of C queries: fp32 matmuls of both members, sigmoid, the float64 combination
                   w s_A + (1 - w) s_B and the >= counts against the gold score (raw and filtered), both sides
--topk K times entity top-k instead (EnsembleRanker.top_k, both sides, no exclusions; the singles are
DistMultRanker.top_k; torch forms u = w sigma(-E_A) + (1 - w) sigma(-E_B) in float64 per chunk and takes torch.topk).
--relations times the relation queries (h, ?, t) over the R relations: rank_relations, or top_k_relations with
--topk; these legs alternate the three paths within every repetition and report the median of each.  The ranking
times are means.  Every time is a CUDA-event window with L2 flushed before it, after a warm-up.  The card's name and
power limit and one JSON line per shape are printed."""
import argparse
import json
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from relationprediction_b200 import ops  # noqa: E402
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag  # noqa: E402

SHAPES = {"FB15k-237": (20466, 14541, 237), "FB15k": (59071, 14951, 1345)}
D, W = 500, 0.5


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--chunk", type=int, default=4096, help="queries per torch matmul")
    ap.add_argument("--topk", type=int, default=None, metavar="K", help="time top-k prediction with K answers")
    ap.add_argument("--relations", action="store_true", help="time relation queries (h, ?, t)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ensemble_rank.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)

    def timeit(fn):
        fn()
        torch.cuda.synchronize()
        tot = 0.0
        for _ in range(args.reps):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            tot += a.elapsed_time(b)
        return tot / args.reps

    for name, (n, V, R) in SHAPES.items():
        g = torch.Generator(device=dev).manual_seed(0)
        members = [(torch.randn(V, D, device=dev, generator=g) * 0.3, torch.randn(R, D, device=dev, generator=g))
                   for _ in range(2)]
        rng = np.random.RandomState(0)
        X_np = np.stack([rng.randint(0, V, n), rng.randint(0, R, n), rng.randint(0, V, n)], 1).astype(np.int32)
        X = torch.as_tensor(X_np, device=dev)
        Xl = X.long()
        masks, dense = [], []
        for side in (0, 1):
            gold = X_np[:, 0] if side == 0 else X_np[:, 2]
            known = [sorted({int(t)} | set(rng.randint(0, V, rng.randint(0, 4)).tolist())) for t in gold]
            masks.append(torch.as_tensor(BilinearDiag.known_bit_mask(known, V), device=dev))
            rows = np.repeat(np.arange(n), [len(k) for k in known])
            dense.append((torch.as_tensor(rows, device=dev), torch.as_tensor(np.concatenate(known), device=dev)))
        ra, rb = (ops.DistMultRanker(c, r) for c, r in members)
        ens = ops.EnsembleRanker(ra, rb, W)
        if args.topk is not None or args.relations:
            leg = prediction_leg(args, name, n, V, R, members, X, Xl, masks, ra, rb, ens, flush)
            print(json.dumps({"shape": name, "n": n, "V": V, "R": R, "d": D, "weight": W, "card": card, **leg}))
            del ra, rb, ens, members
            torch.cuda.empty_cache()
            continue

        def fused():
            return [ens.rank(X, side, masks[side]) for side in (0, 1)]

        def singles():
            return [(ra.rank(X, side, masks[side]), rb.rank(X, side, masks[side])) for side in (0, 1)]

        def torch_path():
            out = []
            for side in (0, 1):
                gold = Xl[:, 0] if side == 0 else Xl[:, 2]
                raw_all, filt_all = [], []
                for c0 in range(0, n, args.chunk):
                    sl = slice(c0, min(n, c0 + args.chunk))
                    comb = None
                    for codes, rel in members:
                        q = rel[Xl[sl, 1]] * (codes[Xl[sl, 2]] if side == 0 else codes[Xl[sl, 0]])
                        s = torch.sigmoid(q @ codes.T).double()
                        comb = W * s if comb is None else comb + (1.0 - W) * s
                    ge = comb >= comb.gather(1, gold[sl, None])
                    raw = ge.sum(1)
                    kr, kc = dense[side]
                    sel = (kr >= c0) & (kr < sl.stop)
                    kn = torch.zeros_like(raw).index_add_(0, kr[sel] - c0, ge[kr[sel] - c0, kc[sel]].long())
                    raw_all.append(raw)
                    filt_all.append(raw - kn + 1)
                out.append((torch.cat(raw_all), torch.cat(filt_all)))
            return out

        # results first: the fused filtered ranks against torch's (near ties may move a rank by one or two)
        f, t = fused(), torch_path()
        agree = float(np.mean([float((f[s][1].long() == t[s][1]).float().mean()) for s in (0, 1)]))
        mrr = lambda r: float((1.0 / r.double()).mean())
        times = {"fused_ensemble_ms": timeit(fused), "two_single_ranks_ms": timeit(singles),
                 "torch_ms": timeit(torch_path)}
        times["fused_over_singles"] = times["fused_ensemble_ms"] / times["two_single_ranks_ms"]
        print(json.dumps({"shape": name, "n": n, "V": V, "d": D, "weight": W, "card": card,
                          **{k: round(v, 3) for k, v in times.items()},
                          "filtered_rank_agreement_with_torch": round(agree, 5),
                          "filtered_mrr": round(np.mean([mrr(f[s][1]) for s in (0, 1)]), 6),
                          "torch_filtered_mrr": round(np.mean([mrr(t[s][1]) for s in (0, 1)]), 6)}))
        del ra, rb, ens, members, f, t
        torch.cuda.empty_cache()


def interleaved_medians(fns, reps, flush):
    """Median CUDA-event time of each of fns (name -> callable), the calls alternating within every repetition (L2
    flushed before each call), after one warm-up call of each: host or clock drift hits all of them alike."""
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    times = {name: [] for name in fns}
    for _ in range(reps):
        for name, fn in fns.items():
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b))
    return {name: float(np.median(t)) for name, t in times.items()}


def prediction_leg(args, name, n, V, R, members, X, Xl, masks, ra, rb, ens, flush):
    """The --topk / --relations legs: fused ensemble, the two members' single fused calls, and torch."""
    k = args.topk
    rel_masks = None
    if args.relations and k is None:
        rng = np.random.RandomState(1)
        known = [sorted({int(t[1])} | set(rng.randint(0, R, rng.randint(0, 3)).tolist())) for t in X.cpu().numpy()]
        rel_masks = torch.as_tensor(BilinearDiag.known_bit_mask(known, R), device=X.device)

    def energies(codes, rel, sl, side):
        if args.relations:
            return (codes[Xl[sl, 0]] * codes[Xl[sl, 2]]) @ rel.T
        q = rel[Xl[sl, 1]] * (codes[Xl[sl, 2]] if side == 0 else codes[Xl[sl, 0]])
        return q @ codes.T

    sides = (0,) if args.relations else (0, 1)
    if args.relations and k is None:
        fused = lambda: ens.rank_relations(X, rel_masks)
        singles = lambda: (ra.rank_relations(X, rel_masks), rb.rank_relations(X, rel_masks))

        def torch_path():
            out = []
            for c0 in range(0, n, args.chunk):
                sl = slice(c0, min(n, c0 + args.chunk))
                comb = None
                for codes, rel in members:
                    s = torch.sigmoid(energies(codes, rel, sl, 0)).double()
                    comb = W * s if comb is None else comb + (1.0 - W) * s
                out.append((comb >= comb.gather(1, Xl[sl, 1:2])).sum(1))
            return torch.cat(out)
    else:
        if args.relations:
            fused = lambda: ens.top_k_relations(X, k)
            singles = lambda: (ra.top_k_relations(X, k), rb.top_k_relations(X, k))
        else:
            fused = lambda: [ens.top_k(X, side, k) for side in sides]
            singles = lambda: [(ra.top_k(X, side, k), rb.top_k(X, side, k)) for side in sides]

        def torch_path():
            out = []
            for side in sides:
                for c0 in range(0, n, args.chunk):
                    sl = slice(c0, min(n, c0 + args.chunk))
                    u = None
                    for codes, rel in members:
                        s = torch.sigmoid(-energies(codes, rel, sl, side).double())
                        u = W * s if u is None else u + (1.0 - W) * s
                    out.append(torch.topk(u, k, dim=1, largest=False, sorted=True))
            return out
    times = interleaved_medians({"fused_ensemble_ms": fused, "two_single_calls_ms": singles, "torch_ms": torch_path},
                                args.reps, flush)
    times["fused_over_singles"] = times["fused_ensemble_ms"] / times["two_single_calls_ms"]
    leg = "relation " if args.relations else "entity "
    leg += "top-%d" % k if k is not None else "ranks"
    return {"leg": leg, **{key: round(v, 3) for key, v in times.items()}}


if __name__ == "__main__":
    main()
