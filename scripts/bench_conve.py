"""The ConvE decoder on the GPU: the 1-N training step beside a torch fp32 composition and beside ComplEx, and filtered
all-entity ranking.

FB15k-237's shape: V = 14 541 entities, R = 237 relations, and n = --queries 1-N queries (60 000: what GraphBatchSize
30 000 gives, object and subject queries of 30 000 positives), random codes and labels (--label-rate of the entities per
query); two network shapes, d = 500 with EmbeddingHeight h = 20 and d = 200 with h = 10, C = 32 filters, the paper's
dropout (keep 0.8 / 0.8 / 0.7, masks drawn once).  A training call is the loss and the gradient of loss + 0.01 reg in
all seven tensors (ops.conve_one_to_n_loss); the forward alone is the same call under torch.no_grad().  The torch
composition is F.conv2d, F.linear, a matmul against every entity and binary_cross_entropy_with_logits under autograd,
with the same masks; the two losses are compared.  ComplEx is ops.one_to_n_loss(..., "complex") on the same queries.
Each variant is timed --iters calls with CUDA events after --warmup, the variants alternating for --rounds rounds;
the median round is reported.  Peak memory is torch.cuda.max_memory_allocated over each variant's own calls.

Ranking: --n-test = 20 466 random test triples, both sides, with random known masks, through ops.ConvERanker.

Prints one JSON line with the card's name and power limit; writes nothing."""
import argparse
import json
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as Fn

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


def timed(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def torch_step(codes, rel, weights, q, dense, eps, masks, keeps, backward):
    """the fp32 composition: the same network, loss and L2 term under autograd"""
    rel_inv, filters, conv_bias, W_fc, b_fc = weights
    h = weights.h
    n, d = len(q), codes.shape[1]
    a, r, s = q[:, 0], q[:, 1], q[:, 2]
    rho = torch.where(s.bool()[:, None], rel[r], rel_inv[r])
    img = torch.cat([codes[a], rho], 1) * masks[0] / keeps[0]
    x = torch.relu(Fn.conv2d(img.view(n, 1, 2 * h, d // h), filters[:, None], conv_bias))
    x = x * masks[1][:, :, None, None] / keeps[1]
    z = Fn.linear(x.reshape(n, -1), W_fc.T, b_fc) * masks[2] / keeps[2]
    E = torch.relu(z) @ codes.T
    V = codes.shape[0]
    loss = Fn.binary_cross_entropy_with_logits(E, dense * (1 - eps) + eps / V)
    reg = ((codes[a] ** 2).sum() + (rho ** 2).sum()) / (n * d)
    if backward:
        (loss + 0.01 * reg).backward()
    return loss


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=60000)
    ap.add_argument("--n-test", type=int, default=20466)
    ap.add_argument("--label-rate", type=float, default=1e-3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    V, R, C, n, eps = 14541, 237, 32, args.queries, 0.1
    name, power = card()
    out = {"gpu": name, "power_limit": power, "V": V, "R": R, "C": C, "queries": n, "n_test": args.n_test}
    rng = np.random.default_rng(0)
    q = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), (np.arange(n) >= n // 2).astype(np.int64)], 1)
    q = np.ascontiguousarray(q.astype(np.int32))
    dense = torch.rand(n, V, device=dev) < args.label_rate
    bits = np.zeros((n, (V + 31) // 32), np.uint32)
    rows, cols = np.nonzero(dense.cpu().numpy())
    np.bitwise_or.at(bits, (rows, cols >> 5), np.left_shift(np.uint32(1), (cols & 31).astype(np.uint32)))
    labels = torch.as_tensor(bits.view(np.int32), device=dev)
    dense = dense.float()
    qd = torch.as_tensor(q, device=dev).long()
    for d, h in ((500, 20), (200, 10)):
        g = torch.Generator(device=dev).manual_seed(d)
        F = C * (2 * h - 2) * (d // h - 2)
        codes = (torch.randn(V, d, device=dev, generator=g) * 0.3).requires_grad_(True)
        rel = (torch.randn(R, d, device=dev, generator=g) * 0.3).requires_grad_(True)
        net = [torch.randn(R, d, device=dev, generator=g) * 0.3, torch.randn(C, 3, 3, device=dev, generator=g) * 0.3,
               torch.zeros(C, device=dev), torch.randn(F, d, device=dev, generator=g) / F ** 0.5,
               torch.zeros(d, device=dev)]
        weights = ops.ConvEWeights(*[t.requires_grad_(True) for t in net], h=h)
        keeps = (0.8, 0.8, 0.7)
        masks = tuple((torch.rand(n, w, device=dev, generator=g) < k).to(torch.uint8)
                      for w, k in zip((2 * d, C, d), keeps))
        fmasks = tuple(m.float() for m in masks)
        crel = (torch.randn(R, d, device=dev, generator=g) * 0.3).requires_grad_(True)
        params = [codes, rel, crel] + list(weights)

        def zero():
            for p in params:
                p.grad = None

        def lib_step(backward=True):
            zero()
            if not backward:
                with torch.no_grad():
                    return ops.conve_one_to_n_loss(codes, rel, weights, q, labels, eps, masks, keeps)
            loss, reg = ops.conve_one_to_n_loss(codes, rel, weights, q, labels, eps, masks, keeps)
            (loss + 0.01 * reg).backward()
            return loss

        def ref_step(backward=True):
            zero()
            if not backward:
                with torch.no_grad():
                    return torch_step(codes, rel, weights, qd, dense, eps, fmasks, keeps, False)
            return torch_step(codes, rel, weights, qd, dense, eps, fmasks, keeps, True)

        def complex_step():
            zero()
            loss, reg = ops.one_to_n_loss(codes, crel, q, labels, eps, "complex")
            (loss + 0.01 * reg).backward()

        res = {}
        lib_loss = float(lib_step(False)[0])
        ref_loss = float(ref_step(False))
        res["loss_conve"], res["loss_torch"] = lib_loss, ref_loss
        res["loss_rel_diff"] = abs(lib_loss - ref_loss) / abs(ref_loss)
        variants = {"conve_fwd": lambda: lib_step(False), "conve_fwd_bwd": lib_step,
                    "torch_fwd": lambda: ref_step(False), "torch_fwd_bwd": ref_step, "complex_fwd_bwd": complex_step}
        times = {k: [] for k in variants}
        peak = {}
        for rnd in range(args.rounds):
            for k, fn in variants.items():
                torch.cuda.reset_peak_memory_stats(dev)
                times[k].append(timed(fn, args.warmup if rnd == 0 else 1, args.iters))
                peak[k] = max(peak.get(k, 0), torch.cuda.max_memory_allocated(dev))
        for k in variants:
            res[k + "_ms"] = round(float(np.median(times[k])), 3)
            res[k + "_peak_GB"] = round(peak[k] / 2 ** 30, 2)
        res["fc_gflop_per_step_fwd"] = round(2 * n * F * d / 1e9, 1)
        # filtered ranking of the test triples on both sides
        with torch.no_grad():
            X = torch.as_tensor(np.stack([rng.integers(0, V, args.n_test), rng.integers(0, R, args.n_test),
                                          rng.integers(0, V, args.n_test)], 1).astype(np.int32), device=dev)
            known = [BilinearDiag.known_bit_mask([[int(v)] for v in X[:, c].tolist()], V) for c in (0, 2)]
            frozen = ops.ConvEWeights(*[w.detach() for w in weights], h=h)
            ranker = ops.ConvERanker(codes.detach(), rel.detach(), frozen)
            masks_d = [torch.as_tensor(k, device=dev) for k in known]

            def rank_both():
                for side in (0, 1):
                    ranker.rank(X, side, masks_d[0 if side == 0 else 1])
            rank_both()
            torch.cuda.reset_peak_memory_stats(dev)
            res["rank_both_sides_ms"] = round(timed(rank_both, 1, 3), 2)
            res["rank_peak_GB"] = round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2)
        out["d%d_h%d" % (d, h)] = res
        del codes, rel, crel, net, weights, params
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
