"""CompGCN layer (Encoder Name=compgcn) measurements, next to the diagonal R-GCN layer (Name=gcn_diag) at the same
graph and width.  Per shape: ops.compgcn_layer forward and forward + backward (ReLU on, no dropout mask, L2 flushed
between calls) alternated with ops.diag_layer, medians over rounds of CUDA-event timings; the library's per-stage event
marks in a separate profiled pass; the achieved walk bytes/s from the DESIGN §3 formulas; and the output difference
against a chunked float64 torch restatement of the layer.  Prints the card's name and power limit, then one JSON line.

    python scripts/bench_compgcn.py [--small]      (--small: the FB15k-237 shape only)"""
import json
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from bench import synthetic_kg  # noqa: E402
from relationprediction_b200 import _lib, ops  # noqa: E402

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


def walk_bytes(tr, V, R, d):
    """Algorithmic bytes of the two CompGCN walks (DESIGN §3).  Forward: per message the gathered H row and its index,
    weight id and norm, M (4d + 12), plus the loop row of H read and the Cat row (3d) written, 16 V d.  Backward: per
    message the gathered dCat slab row and the same 12 bytes, M (4d + 12), plus H read and dH written, 8 V d, the loop
    slab of dCat read, 4 V d, and one d-wide vector reduction into dZ per (source, weight id) run, 4 d each."""
    t = torch.as_tensor(tr, device=dev).long()
    s, r, o = t[:, 0], t[:, 1], t[:, 2]
    runs = torch.unique(torch.cat([s * (2 * R) + r, o * (2 * R) + R + r])).numel()
    M = 2 * len(tr)
    return M * (4 * d + 12) + 16 * V * d, M * (4 * d + 12) + 12 * V * d + runs * 4 * d, runs


@torch.no_grad()
def restated_forward(tr, V, R, H, Z, zl, W_cat, W_rel, b, chunk=1 << 21):
    """the layer in float64 torch, messages in chunks (mult composition, ReLU, no mask)"""
    t = torch.as_tensor(tr, device=dev).long()
    s, r, o = t[:, 0], t[:, 1], t[:, 2]
    deg_o = torch.bincount(o, minlength=V).double()
    deg_s = torch.bincount(s, minlength=V).double()
    Hd, Zd = H.double(), Z.double()
    A = torch.zeros(V, 2 * H.shape[1], dtype=torch.float64, device=dev)
    d = H.shape[1]
    for c0 in range(0, len(t), chunk):
        sl = slice(c0, c0 + chunk)
        A[:, :d].index_add_(0, o[sl], Hd[s[sl]] * Zd[r[sl]] / deg_o[o[sl]][:, None])
        A[:, d:].index_add_(0, s[sl], Hd[o[sl]] * Zd[R + r[sl]] / deg_s[s[sl]][:, None])
    Cat = torch.cat([A, Hd * zl.double()], 1) / 3
    return torch.relu(Cat @ W_cat.double() + b.double()), Zd @ W_rel.double()


def case(name, V, R, E, d, rounds=3):
    g = torch.Generator(device=dev).manual_seed(0)
    tr = synthetic_kg(V, R, E, seed=1234, skewed=False)
    _lib.set_option("graph_views", 1)         # both layers walk the CSR views only
    try:
        gr = ops.Graph.from_device_triples(torch.as_tensor(tr, device=dev), V, R)
    finally:
        _lib.set_option("graph_views", 3)
    H = torch.randn(V, d, device=dev, generator=g).requires_grad_(True)
    dOut = torch.randn(V, d, device=dev, generator=g)
    dZn = torch.randn(2 * R, d, device=dev, generator=g)
    std = 1.0 / np.sqrt(d)
    wc = [torch.randn(2 * R, d, device=dev, generator=g), torch.randn(d, device=dev, generator=g),
          torch.randn(3 * d, d, device=dev, generator=g) * std, torch.randn(d, d, device=dev, generator=g) * std,
          torch.zeros(d, device=dev)]
    wc = [w.requires_grad_(True) for w in wc]
    wd = [torch.randn(R, d, device=dev, generator=g).requires_grad_(True) for _ in range(2)]
    wd.append((torch.randn(d, d, device=dev, generator=g) * std).requires_grad_(True))
    wd.append(torch.zeros(d, device=dev).requires_grad_(True))
    fns = {"compgcn": lambda: ops.compgcn_layer(H, *wc, gr, "mult", None, 1.0, True),
           "gcn_diag": lambda: (ops.diag_layer(H, wd[0], wd[1], wd[2], wd[3], gr, None, 1.0, True),)}

    def step(k):
        H.grad = None
        outs = fns[k]()
        torch.autograd.backward(list(outs), [dOut, dZn][:len(outs)])

    def fwd(k):
        with torch.no_grad():
            fns[k]()
    ms = {k: {"fwd": [], "fwd_bwd": []} for k in fns}
    for _ in range(rounds):
        for k in fns:
            ms[k]["fwd"].append(timeit(lambda: fwd(k)))
            ms[k]["fwd_bwd"].append(timeit(lambda: step(k)))
    med = {k: {p: float(np.median(v[p])) for p in v} for k, v in ms.items()}
    stages = {}
    for k in fns:
        _lib.profile_enable(True)
        acc = {}
        for _ in range(5):
            flush.zero_()
            step(k)
            torch.cuda.synchronize()
            for nm, v in _lib.profile_read():
                acc[nm] = acc.get(nm, 0.0) + v / 5
        _lib.profile_enable(False)
        stages[k] = {nm: round(v, 4) for nm, v in acc.items()}
    by_f, by_b, runs = walk_bytes(tr, V, R, d)
    t_f, t_b = stages["compgcn"].get("compgcn_walk_fwd", 0.0), stages["compgcn"].get("compgcn_walk_bwd", 0.0)
    with torch.no_grad():
        out, Zn = fns["compgcn"]()
        ref_out, ref_Zn = restated_forward(tr, V, R, H.detach(), *[w.detach() for w in wc])
        diff = {"out": float((out.double() - ref_out).abs().max() / ref_out.abs().max()),
                "Z_next": float((Zn.double() - ref_Zn).abs().max() / ref_Zn.abs().max())}
    del out, Zn, ref_out, ref_Zn
    res = {"V": V, "R": R, "E": E, "M": 2 * E, "d": d, "medians_ms": med, "runs_ms": ms, "stages_ms": stages,
           "bwd_source_weight_runs": runs, "fwd_walk_bytes": by_f, "bwd_walk_bytes": by_b,
           "fwd_walk_GBps": by_f / t_f / 1e6 if t_f > 0 else None, "bwd_walk_GBps": by_b / t_b / 1e6 if t_b > 0 else None,
           "frac_of_3350_GBps": {"fwd_walk": by_f / t_f / 1e6 / 3350 if t_f > 0 else None,
                                 "bwd_walk": by_b / t_b / 1e6 / 3350 if t_b > 0 else None},
           "max_rel_diff_vs_float64_torch": diff}
    del H, dOut, dZn, wc, wd, fns, gr
    torch.cuda.empty_cache()
    return res


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print("GPU:", card, flush=True)
    out = {"gpu": card}
    out["fb15k237_d200"] = case("fb15k237_d200", 14541, 237, 272115, 200)
    if "--small" not in sys.argv:
        out["synthetic_V1M_E10M_d256"] = case("synthetic_V1M_E10M_d256", 1_000_000, 237, 10_000_000, 256, rounds=2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
