"""The RotatE decoder on the GPU: scorer forward + backward beside ComplEx, the self-adversarial step, and filtered
all-entity ranking beside a chunked torch restatement.

The shipped training shape: N = 330 000 fed triples (30 000 positives, NegativeSampleRate K = 10), d = 500, FB15k-237's
V = 14 541 entities and R = 237 relations; random codes, phases uniform in [-pi, pi], random corruptions in the
sampler's layout.  A training call is the loss and the gradient of loss + 0.01 reg with the relation slice norm on.
ops.rotate_score and ops.complex_score (both NegativeSampling) alternate --rounds times in this one process, each round
timing --iters calls with CUDA events after --warmup; the median round is reported, and likewise for the
self-adversarial step (ops.self_adversarial_loss, decoder "rotate").

Ranking: an FB15k-237-sized test set (--n-test = 20 466 random triples, both sides, random known masks with the gold
set) through ops.RotateRanker, and the same ranks from a torch restatement on the same GPU that materialises D for
chunks of queries (float32, torch.hypot summed over k).  The ranks of the two are compared: the fraction identical and
the two MRRs.  Achieved moduli per second count 2 n_test V d/2 moduli.

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


def torch_ranks(codes, rel, X, side, mask_bits, chunk=256):
    """the restatement: D [chunk, V] in float32 for each chunk of queries, then the counting rules"""
    V, d = codes.shape
    h = d // 2
    Xl = X.long()
    kept, gold = (Xl[:, 2], Xl[:, 0]) if side == 0 else (Xl[:, 0], Xl[:, 2])
    theta = rel[Xl[:, 1], :h] * (-1.0 if side == 0 else 1.0)
    cs, sn = torch.cos(theta), torch.sin(theta)
    qr = codes[kept, :h] * cs - codes[kept, h:] * sn
    qi = codes[kept, :h] * sn + codes[kept, h:] * cs
    cols = torch.arange(V, device=codes.device)
    raw, filt = [], []
    for c0 in range(0, len(X), chunk):
        c1 = min(len(X), c0 + chunk)
        D = torch.zeros((c1 - c0, V), device=codes.device)
        for k in range(h):
            D += torch.hypot(qr[c0:c1, k, None] - codes[None, :, k], qi[c0:c1, k, None] - codes[None, :, h + k])
        hit = D <= D[torch.arange(c1 - c0), gold[c0:c1]][:, None]
        known = ((mask_bits[c0:c1, cols >> 5] >> (cols & 31)) & 1).bool()
        r = hit.sum(1)
        raw.append(r)
        filt.append(r - (hit & known).sum(1) + 1)
    return torch.cat(raw), torch.cat(filt)


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
        raise SystemExit("bench_rotate: no CUDA device")
    dev = torch.device("cuda:0")
    ops.set_slice_norms(True)
    g = torch.Generator(device=dev).manual_seed(0)
    V, R, d, n, K = args.V, args.R, args.d, args.n, args.K
    N = n * (K + 1)
    codes = (torch.randn(V, d, device=dev, generator=g) * 0.1).requires_grad_(True)
    rel = ((torch.rand(R, d, device=dev, generator=g) * 2 - 1) * np.pi).requires_grad_(True)
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
    paths = {"rotate": step(lambda: ops.rotate_score(codes, rel, X, Y, gamma=12.0)[1:]),
             "complex": step(lambda: ops.complex_score(codes, rel, X, Y)[1:]),
             "rotate_self_adversarial": step(lambda: ops.self_adversarial_loss(codes, rel, X, K, 1.0, "rotate",
                                                                               gamma=12.0)[:2])}
    times = {p: [] for p in paths}
    for _ in range(args.rounds):
        for p, fn in paths.items():
            times[p].append(timed(fn, args.warmup, args.iters))
    out["scorer_fwd_bwd_ms"] = {p: {"median": round(float(np.median(ts)), 4),
                                    "spread": [round(min(ts), 4), round(max(ts), 4)]} for p, ts in times.items()}

    # filtered ranking of an FB15k-237-sized test set, both sides
    c = (torch.randn(V, d, device=dev, generator=g)).contiguous()
    r = ((torch.rand(R, d, device=dev, generator=g) * 2 - 1) * np.pi).contiguous()
    nt = args.n_test
    T = np.stack([rng.integers(0, V, nt), rng.integers(0, R, nt), rng.integers(0, V, nt)], 1).astype(np.int32)
    Xt = torch.as_tensor(T, device=dev)
    ranker = ops.RotateRanker(c, r)
    masks = []
    for side in (0, 1):
        gold = T[:, 0] if side == 0 else T[:, 2]
        lists = [[int(x)] + rng.integers(0, V, 3).tolist() for x in gold]
        masks.append(torch.as_tensor(BilinearDiag.known_bit_mask(lists, V), device=dev))

    def fused():
        return [ranker.rank(Xt, side, masks[side]) for side in (0, 1)]

    def restated():
        return [torch_ranks(c, r, Xt, side, masks[side]) for side in (0, 1)]
    fused_ms = [timed(fused, 1, 3) for _ in range(3)]
    torch_ms = [timed(restated, 0, 1) for _ in range(2)]
    a, b = fused(), restated()
    raw_a = torch.cat([x[0] for x in a]).double()
    raw_b = torch.cat([x[0] for x in b]).double()
    filt_a = torch.cat([x[1] for x in a]).double()
    filt_b = torch.cat([x[1] for x in b]).double()
    moduli = 2 * nt * V * (d // 2)
    ms = float(np.median(fused_ms))
    out["ranking"] = {"n_test": nt, "both_sides": True, "moduli": moduli,
                      "fused_ms": round(ms, 2), "fused_spread_ms": [round(min(fused_ms), 2), round(max(fused_ms), 2)],
                      "fused_moduli_per_s": float("%.3g" % (moduli / (ms * 1e-3))),
                      "torch_restatement_ms": round(float(np.median(torch_ms)), 1),
                      "raw_identical": round(float((raw_a == raw_b).double().mean()), 5),
                      "filtered_identical": round(float((filt_a == filt_b).double().mean()), 5),
                      "filtered_mrr": [round(float((1 / filt_a).mean()), 6), round(float((1 / filt_b).mean()), 6)]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
