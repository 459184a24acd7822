"""1-N training step: the fused library call (ops.one_to_n_loss) against the torch composition, on an H100.

Random codes at the FB15k-237 shape (V = 14 541, d = 500, R = 237), n queries with ~1 % positive labels, label
smoothing 0.1.  For each decoder and n it times the loss alone (no gradient wanted), the forward of a training step
(which also forms the gradient of the loss) and the forward + backward, with CUDA events
over --iters calls after --warmup, and records the peak device memory of one forward + backward.  The torch
composition is: the query rows in torch, q @ codes.T, binary_cross_entropy_with_logits against the dense smoothed
targets, autograd.  Prints one JSON line; writes nothing.

--driver-step instead times whole training steps of the driver (train.py --profile-iterations: sample wait,
forward + loss with the host query de-duplication and label rows, backward, optimizer) on a random graph of the
FB15k-237 size (272 115 training triples), for the embedding encoder (every step the whole split: about 540 000
queries, de-duplicated once) and for a 2-layer basis R-GCN with GraphBatchSize = 30 000 (about 60 000 fresh queries
per step).  Its dataset and settings go to a temporary directory."""
import argparse
import contextlib
import io
import json
import os
import sys
import tempfile

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, ".")
from relationprediction_b200 import ops  # noqa: E402


def torch_rows(codes, rel, q, decoder):
    a, r = codes[q[:, 0]], rel[q[:, 1]]
    if decoder == "distmult":
        return a * r
    h = codes.shape[1] // 2
    side = q[:, 2:3].float()
    kr, ki, br, bi = a[:, :h], a[:, h:], r[:, :h], r[:, h:]
    return side * torch.cat([kr * br - ki * bi, ki * br + kr * bi], 1) + \
        (1 - side) * torch.cat([br * kr + bi * ki, br * ki - bi * kr], 1)


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


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


DRIVER_EXP = """[Encoder]
\tName={encoder}
\tDropoutKeepProbability=0.8
\tInternalEncoderDimension=500
\tNumberOfBasisFunctions=2
\tNumberOfLayers=2
\tUseInputTransform=Yes
\tUseOutputTransform=No
\tAddDiagonal=No
\tDiagonalCoefficients=No
\tSkipConnections=None
\tStoreEdgeData=No
\tRandomInput=No
\tPartiallyRandomInput=No
\tConcatenation=No

[Decoder]
\tName={decoder}
\tRegularizationParameter=0.01

[Shared]
\tCodeDimension=500

[Optimizer]
\tMaxGradientNorm=1
\tReportTrainLossEvery=100

\t[Algorithm]
\t\tName=Adam
\t\tlearning_rate=0.01

[General]
\tNegativeSampleRate=10
\tGraphSplitSize=0.5
\tTrainingObjective=1-N
\tLabelSmoothing=0.1
{graph_batch}\tExperimentName=models/bench

[Evaluation]
\tMetric=MRR
"""


def driver_step(iters):
    from relationprediction_b200 import train as driver
    rng = np.random.default_rng(0)
    V, R = 14541, 237
    split = lambda m: np.stack([rng.integers(0, V, m), rng.integers(0, R, m), rng.integers(0, V, m)], 1).astype(np.int32)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        npz = os.path.join(tmp, "kg.npz")
        np.savez(npz, train=split(272115), valid=split(1000), test=split(1000), V=V, R=R)
        for encoder, batch in (("embedding", ""), ("gcn_basis", "\tGraphBatchSize=30000\n")):
            for decoder in ("bilinear-diag", "complex"):
                exp = os.path.join(tmp, "bench.exp")
                with open(exp, "w") as fh:
                    fh.write(DRIVER_EXP.format(encoder=encoder, decoder=decoder, graph_batch=batch))
                out = io.StringIO()
                with contextlib.redirect_stdout(out):
                    driver.main(["--settings", exp, "--dataset-npz", npz, "--no-save", "--no-periodic-eval",
                                 "--profile-iterations", str(iters)])
                prof = json.loads([l for l in out.getvalue().splitlines() if l.startswith("{")][-1])
                rows.append({"encoder": encoder, "decoder": decoder, "graph_batch": batch.strip() or "whole split",
                             "phase_ms": prof["phase_ms"],
                             "free_running_ms_per_iteration": prof["free_running_ms_per_iteration"]})
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "driver_step": rows}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--V", type=int, default=14541)
    ap.add_argument("--d", type=int, default=500)
    ap.add_argument("--R", type=int, default=237)
    ap.add_argument("--n", type=int, nargs="+", default=[4096, 60000])
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--driver-step", action="store_true", help="time whole driver steps instead (see above)")
    args = ap.parse_args()
    if args.driver_step:
        return driver_step(args.iters)
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    V, d, R = args.V, args.d, args.R
    codes = (torch.randn(V, d, device=dev, generator=g) * 0.1).requires_grad_(True)
    rel = (torch.randn(R, d, device=dev, generator=g) * 0.1).requires_grad_(True)
    rng = np.random.default_rng(0)
    out = {"gpu": torch.cuda.get_device_name(0), "V": V, "d": d, "results": []}
    for n in args.n:
        q = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, 2, n)], 1).astype(np.int32)
        q = q[np.lexsort((q[:, 0], q[:, 1], q[:, 2]))]
        dense = torch.rand(n, V, device=dev, generator=g) < 0.01
        bits = torch.zeros(n, (V + 31) // 32 * 32, dtype=torch.int64, device=dev)
        bits[:, :V] = dense.long()
        words = (bits.view(n, -1, 32) << torch.arange(32, device=dev)).sum(2)
        labels = torch.as_tensor(words.cpu().numpy().astype(np.uint32).view(np.int32), device=dev)
        qt = torch.as_tensor(q, device=dev).long()
        target = dense.float() * 0.9 + 0.1 / V
        for decoder in ("distmult", "complex"):
            fused_f = lambda: ops.one_to_n_loss(codes, rel, q, labels, 0.1, decoder, R)

            def fused_fb():
                loss, reg = ops.one_to_n_loss(codes, rel, q, labels, 0.1, decoder, R)
                torch.autograd.grad(loss + 0.01 * reg, [codes, rel])

            def torch_f():
                z = torch_rows(codes, rel, qt, decoder) @ codes.T
                return F.binary_cross_entropy_with_logits(z, target)

            def torch_fb():
                torch.autograd.grad(torch_f(), [codes, rel])

            def fused_loss_only():
                with torch.no_grad():
                    fused_f()

            with torch.no_grad():
                lf = float(fused_f()[0])
                lt = float(torch_f())
            row = {"decoder": decoder, "n": n, "loss_fused": lf, "loss_torch": lt,
                   "fused_loss_only_ms": timed(fused_loss_only, args.warmup, args.iters),
                   "fused_fwd_ms": timed(lambda: fused_f(), args.warmup, args.iters),
                   "fused_fwd_bwd_ms": timed(fused_fb, args.warmup, args.iters),
                   "fused_peak_mib": peak(fused_fb)}
            try:
                row.update({"torch_fwd_ms": timed(torch_f, args.warmup, args.iters),
                            "torch_fwd_bwd_ms": timed(torch_fb, args.warmup, args.iters),
                            "torch_peak_mib": peak(torch_fb)})
            except torch.cuda.OutOfMemoryError:
                row["torch"] = "out of memory"
                torch.cuda.empty_cache()
            out["results"].append({k: round(v, 4) if isinstance(v, float) else v for k, v in row.items()})
        del dense, bits, words, labels, target
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
