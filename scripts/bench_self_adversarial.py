"""Self-adversarial negative sampling against the NegativeSampling scorer, forward + backward, on the GPU.

The shipped training shape: GraphBatchSize = 30 000 positives with NegativeSampleRate K = 10, so N = 330 000 fed
triples, d = 500, FB15k-237's V = 14 541 entities and R = 237 relations; random codes, random corruptions in the
sampler's layout.  For each decoder one call is ops.self_adversarial_loss (or ops.distmult / ops.complex_score with the
sampler's labels, on the same X) followed by the gradient of loss + 0.01 reg with the relation slice norm on, as a
training step with MaxGradientNorm runs it.  The two paths alternate --rounds times in this one process, each round
timing --iters calls with CUDA events after --warmup; the median round is reported.

Bytes per call are counted from shapes, as if every gathered row came from memory: the forward reads three d-float rows
and one X row per triple and writes the energies (self-adversarial: also the coefficients, and reads its energies back
once); the backward reads three rows, X and the per-triple gradient and adds three rows of gradient (counted as a read
and a write).  At this V the code table (29 MB) fits in the H100's L2, so the rate is a gather rate, not a DRAM
bandwidth.  Prints one JSON line with the card's name and power limit; writes nothing."""
import argparse
import json
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from relationprediction_b200 import ops  # noqa: E402


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


def call_bytes(N, d, self_adversarial):
    row = 3 * d * 4
    fwd = N * (row + 12 + 4) + (N * 8 if self_adversarial else N * 4)   # + coef write and read-back, or Y
    bwd = N * (row + 12 + 4) + N * row * 2
    return fwd + bwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--V", type=int, default=14541)
    ap.add_argument("--R", type=int, default=237)
    ap.add_argument("--d", type=int, default=500)
    ap.add_argument("--n", type=int, default=30000, help="positives per step (GraphBatchSize)")
    ap.add_argument("--K", type=int, default=10, help="NegativeSampleRate")
    ap.add_argument("--alpha", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_self_adversarial: no CUDA device")
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
    out = {"gpu": name, "power_limit": power, "V": V, "R": R, "d": d, "n": n, "K": K, "N": N, "alpha": args.alpha,
           "results": []}
    scorers = {"distmult": ops.distmult, "complex": ops.complex_score}
    for decoder in ("distmult", "complex"):
        def self_adversarial():
            loss, reg, _ = ops.self_adversarial_loss(codes, rel, X, K, args.alpha, decoder)
            torch.autograd.grad(loss + 0.01 * reg, [codes, rel])

        def negative_sampling():
            _, loss, reg = scorers[decoder](codes, rel, X, Y)
            torch.autograd.grad(loss + 0.01 * reg, [codes, rel])

        times = {"self_adversarial": [], "negative_sampling": []}
        for _ in range(args.rounds):
            times["self_adversarial"].append(timed(self_adversarial, args.warmup, args.iters))
            times["negative_sampling"].append(timed(negative_sampling, args.warmup, args.iters))
        row = {"decoder": decoder}
        for path, ts in times.items():
            ms = float(np.median(ts))
            nbytes = call_bytes(N, d, path == "self_adversarial")
            row[path] = {"fwd_bwd_ms": round(ms, 4), "spread_ms": [round(min(ts), 4), round(max(ts), 4)],
                         "bytes_per_call": nbytes, "gather_rate_GBps": round(nbytes / (ms * 1e-3) / 1e9, 1)}
        row["ratio"] = round(row["self_adversarial"]["fwd_bwd_ms"] / row["negative_sampling"]["fwd_bwd_ms"], 3)
        out["results"].append(row)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
