"""Fused relation prediction next to its unfused torch composition, at the FB15k-237 and FB15k test shapes:

  python scripts/bench_relation_rank.py [--decoder distmult|complex] [--reps N]

For n (head, ?, tail) queries over R relations at code width d (random codes, seeded):
  rank_relations         the fused path (pair-query prepare kernel + scoring GEMM with the rank epilogue over rel[0:R])
  top_k_relations k=10   the fused path (prepare + scoring GEMM with the top-k epilogue + merge)
  torch rank / top-k     Q = the pair-query rows (torch), E = Q @ rel[:R].T (fp32 matmul), then the sigmoid-space
                         >= counts against the gold score, or torch.topk on E with the known relations masked out
Times are means of CUDA-event windows (L2 flushed before each), after a warm-up of every shape.  The card's name and
power limit, the GEMM's launch shape (tiles, CTAs) and one JSON line per shape are printed."""
import argparse
import json
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from relationprediction_b200 import ops  # noqa: E402
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag  # noqa: E402

SHAPES = {"FB15k-237": (20466, 237, 500), "FB15k": (59071, 1345, 500)}
BM = BN = 128   # the scoring GEMM's tile (csrc/gemm_tf32x3.cu)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--decoder", choices=("distmult", "complex"), default="distmult")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--k", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_relation_rank.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    print("card:", card, "| SMs:", sms, "| decoder:", args.decoder)

    def timeit(fn):
        for _ in range(3):
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

    for name, (n, R, d) in SHAPES.items():
        V = 14541 if name == "FB15k-237" else 14951
        g = torch.Generator(device=dev).manual_seed(0)
        codes = torch.randn(V, d, device=dev, generator=g) * 0.3
        rel = torch.randn(V, d, device=dev, generator=g)           # an R-GCN style [V, d] table; rows 0..R-1 count
        rng = np.random.RandomState(0)
        X_np = np.stack([rng.randint(0, V, n), rng.randint(0, R, n), rng.randint(0, V, n)], 1).astype(np.int32)
        known = [sorted({int(r)} | set(rng.randint(0, R, rng.randint(0, 3)).tolist())) for r in X_np[:, 1]]
        X = torch.as_tensor(X_np, device=dev)
        mask = torch.as_tensor(BilinearDiag.known_bit_mask(known, R), device=dev)
        cls = ops.DistMultRanker if args.decoder == "distmult" else ops.ComplexRanker
        ranker = cls(codes, rel, R)
        Xl = X.long()
        gold = Xl[:, 1]
        known_dense = torch.zeros(n, R, dtype=torch.bool, device=dev)
        rows = torch.as_tensor(np.repeat(np.arange(n), [len(l) for l in known]), device=dev)
        known_dense[rows, torch.as_tensor(np.concatenate(known), device=dev)] = True

        def queries():
            a, b = codes[Xl[:, 0]], codes[Xl[:, 2]]
            if args.decoder == "distmult":
                return a * b
            h = d // 2
            ar, ai, br, bi = a[:, :h], a[:, h:], b[:, :h], b[:, h:]
            return torch.cat([ar * br + ai * bi, ar * bi - ai * br], 1)

        def torch_rank():
            s = torch.sigmoid(queries() @ rel[:R].T)
            ge = s >= s.gather(1, gold[:, None])
            raw = ge.sum(1)
            return raw, raw - (ge & known_dense).sum(1) + 1

        def torch_topk():
            e = (queries() @ rel[:R].T).masked_fill(known_dense, float("-inf"))
            return torch.topk(e, args.k, dim=1)

        fused_rank = lambda: ranker.rank_relations(X, mask)
        fused_topk = lambda: ranker.top_k_relations(X, args.k, mask)
        # results first: the fused ranks against torch's (fp32 matmul; near ties may move a rank by one or two)
        raw, filt = fused_rank()
        traw, tfilt = torch_rank()
        agree = float((filt == tfilt).float().mean())
        mrr = lambda r: float((1.0 / r.double()).mean())
        ids, _ = fused_topk()
        tids = torch_topk().indices
        top1 = float((ids[:, 0].long() == tids[:, 0]).float().mean())
        times = {"fused_rank_ms": timeit(fused_rank), "fused_topk_ms": timeit(fused_topk),
                 "torch_rank_ms": timeit(torch_rank), "torch_topk_ms": timeit(torch_topk)}
        tiles_m, tiles_n = (n + BM - 1) // BM, (R + BN - 1) // BN
        tiles = tiles_m * tiles_n
        launch = {"M": n, "N": R, "K": d, "tiles": [tiles_m, tiles_n], "ctas": min(tiles, sms),
                  "tiles_per_cta": round(tiles / min(tiles, sms), 2),
                  "n_columns_used": round(R / (tiles_n * BN), 3)}
        print("%s: n=%d R=%d d=%d  launch: %d x %d tiles on %d CTAs (%.2f tiles each), %.0f%% of the N tile width "
              "used" % (name, n, R, d, tiles_m, tiles_n, launch["ctas"], launch["tiles_per_cta"],
                        100 * launch["n_columns_used"]))
        print(json.dumps({"shape": name, "decoder": args.decoder, "card": card, "k": args.k, "launch": launch,
                          **{k: round(v, 3) for k, v in times.items()},
                          "filtered_rank_agreement_with_torch": round(agree, 5),
                          "filtered_mrr": round(mrr(filt), 6), "torch_filtered_mrr": round(mrr(tfilt), 6),
                          "top1_agreement_with_torch": round(top1, 5)}))
        del ranker, codes, rel, known_dense
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
