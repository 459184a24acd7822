"""GPU graph preparation, canonical against per-relation normalisation (NormalizationMode=relation), on an H100.

The half-size synthetic workload of bench.py (5 M nodes, 1 000 relations, 50 M edges = 100 M messages, uniform and
skewed endpoints, SURVEY.md 8(d) generator) is copied to the GPU once; then rgcn_graph_create_device builds the graph
from the device edge list with graph_views 2 and 3, the two norm modes alternating, --warmup untimed builds and
--repeat timed ones per configuration.  A build is timed with a host clock between two device synchronisations (the
build itself ends in one), and the graph is destroyed outside the timed window.  Reported per configuration: median
and min milliseconds, resident device bytes of the graph (info[11]), and the relation / canonical time ratio.
Prints the GPU name and power limit, then one JSON line; writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from relationprediction_b200 import _lib, ops  # noqa: E402


def synthetic_kg(V, R, E, seed, skewed):
    """bench.py's generator: uniform, or skewed s,o = floor(V*u^3) under a fixed permutation, r = floor(R*u^2)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    if not skewed:
        s, o, r = rng.integers(0, V, E), rng.integers(0, V, E), rng.integers(0, R, E)
    else:
        perm = rng.permutation(V)
        s = perm[np.minimum((V * rng.random(E) ** 3).astype(np.int64), V - 1)]
        o = perm[np.minimum((V * rng.random(E) ** 3).astype(np.int64), V - 1)]
        r = np.minimum((R * rng.random(E) ** 2).astype(np.int64), R - 1)
    return np.stack([s, r, o], 1).astype(np.int32)


def gpu_description():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def build_ms(t, V, R, mode):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    g = ops.Graph.from_device_triples(t, V, R, norm_mode=mode)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    info = g.info()
    del g
    torch.cuda.synchronize()
    return ms, info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=5_000_000)
    ap.add_argument("--relations", type=int, default=1000)
    ap.add_argument("--edges", type=int, default=50_000_000)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--views", default="2,3")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph_prep.py needs a CUDA device")
    print("gpu:", gpu_description(), flush=True)
    V, R, E = args.nodes, args.relations, args.edges
    results = []
    for skewed in (False, True):
        t = torch.from_numpy(synthetic_kg(V, R, E, seed=1234, skewed=skewed)).cuda()
        for views in [int(v) for v in args.views.split(",")]:
            _lib.set_option("graph_views", views)
            times = {"canonical": [], "relation": []}
            info = {}
            for it in range(args.warmup + args.repeat):
                for mode in (("canonical", "relation") if it % 2 == 0 else ("relation", "canonical")):
                    ms, info[mode] = build_ms(t, V, R, mode)
                    if it >= args.warmup:
                        times[mode].append(ms)
            row = {"graph": "skewed" if skewed else "uniform", "graph_views": views, "V": V, "R": R, "E": E}
            for mode in ("canonical", "relation"):
                row[mode] = {"median_ms": float(np.median(times[mode])), "min_ms": float(np.min(times[mode])),
                             "resident_bytes": int(info[mode][11]), "n_groups": int(info[mode][9])}
            row["relation_over_canonical"] = row["relation"]["median_ms"] / row["canonical"]["median_ms"]
            print(json.dumps(row), flush=True)
            results.append(row)
        del t
        torch.cuda.empty_cache()
    _lib.set_option("graph_views", 3)
    print(json.dumps({"what": "GPU graph preparation from a device edge list, canonical vs relation norms",
                      "gpu": gpu_description(), "results": results}))


if __name__ == "__main__":
    main()
