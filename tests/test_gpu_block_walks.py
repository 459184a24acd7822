"""GPU: every walk-table row (tests/block_walks.py) against a float64 restatement, on graphs whose run structure is
set by construction.

Within one (supertile, weight id) the weight-id-major walks take messages sorted by row, so the number of messages a
row receives from one weight id is the length of a run.  The graph holds one run-length pattern per weight id: all
singletons, one long run, and mixed patterns whose runs straddle every group (8 or 4 messages), index-batch (32) and
work-item (RGCN_ITEM_MAX) boundary.  A second message family gives the backward walk over sources the same patterns.

Error bound: besides the suite's global max|a-b| / max|b| < 1e-4, every element must satisfy
|got - ref| <= TOL * ref_abs, where ref_abs is the same float64 computation on |H|, |W|, |norm|, |W_self| and |dOut|
(the sum of the absolute values of the terms).  The ReLU gate of the backward reference is taken from the kernel's
own `out`, which is exactly what the backward computes; a pre-activation within its bound of zero may flip the gate,
and the forward bound already limits such flips to those elements."""
import os

import numpy as np
import pytest
import torch

import block_walks as bw
from relationprediction_b200 import _lib, ops
from test_gpu_parity import assert_close

pytestmark = pytest.mark.gpu

TOL = 1e-5
DEV = "cuda:0"
V, R = 420, 32                      # 2R = 64 weight ids
PATTERNS = ([[1] * n for n in (1, 7, 8, 9, 31, 32, 33, 63, 64, 65, 127, 128, 129, 300)]
            + [[L] for L in (1, 8, 32, 33, 128, 129, 300)]
            + [[7, 2, 30, 1, 24, 64], [31, 1, 32], [33, 31], [8] * 16, [4] * 32])
# weight ids [0, 26): runs over destinations (forward walk); [26, 52): runs over sources (backward walk);
# [52, 64): empty (their dW must come back exactly zero)
FWD_IDS = range(0, len(PATTERNS))
BWD_IDS = range(len(PATTERNS), 2 * len(PATTERNS))


def pattern_messages(seed=0):
    rng = np.random.RandomState(seed)
    rows = np.array([r for r in range(V) if r % 10 != 3])   # rows = 3 (mod 10) never send or receive
    dst, src, relw = [], [], []
    for fam, ids in ((0, FWD_IDS), (1, BWD_IDS)):
        for w, pat in zip(ids, PATTERNS):
            runs = np.sort(rng.choice(rows, len(pat), replace=False))
            if len(pat) > 1 and w % 2 == 0:                  # rows 0 and V-1 in use
                runs[0], runs[-1] = 0, V - 1
            key = np.repeat(runs, pat)
            other = rng.choice(rows, len(key))
            dst.append(key if fam == 0 else other)
            src.append(other if fam == 0 else key)
            relw.append(np.full(len(key), w))
    dst, src, relw = (np.concatenate(a).astype(np.int32) for a in (dst, src, relw))
    perm = rng.permutation(len(dst))                         # the graph builder, not the input order, makes the runs
    norm = rng.uniform(0.1, 1.0, len(dst)).astype(np.float32)
    return dst[perm], src[perm], relw[perm], norm


MSGS = pattern_messages()


def layer_inputs(d, B, seed=1):
    rng = np.random.RandomState(seed + d * 7 + B)
    s = d // B
    H = rng.normal(0, 1, (V, d)).astype(np.float32)
    W = rng.normal(0, 0.3, (2 * R, B, s, s)).astype(np.float32)
    Ws = rng.normal(0, 1.0 / np.sqrt(d), (d, d)).astype(np.float32)
    dOut = rng.normal(0, 1, (V, d)).astype(np.float32)
    mask = (rng.uniform(size=(V, d)) < 0.8).astype(np.uint8)
    return H, W, Ws, dOut, mask


def add_messages(acc, X, W, msgs, B):
    """acc[dst_m] += norm_m W[relw_m] X[src_m] (blocks of s), one weight id at a time, differentiable in X and W"""
    dst, src, relw, norm = msgs
    d = X.shape[1]
    s = d // B
    nm = torch.tensor(norm, dtype=torch.float64)
    for w in np.unique(relw):
        sel = np.nonzero(relw == w)[0]
        x = X[torch.tensor(src[sel].astype(np.int64))].reshape(-1, B, s) * nm[sel][:, None, None]
        y = torch.einsum("bij,mbj->mbi", W[int(w)], x).reshape(-1, d)
        acc = acc.index_add(0, torch.tensor(dst[sel].astype(np.int64)), y)
    return acc


def reference(d, B, H, W, Ws, mask, keep, gate, dOut, absolute=False):
    """float64 autograd restatement over the messages: pre = dropout(H W_self) + sum_m norm_m W[relw_m] H[src_m] at
    dst_m, gradients of sum(pre * gate * dOut).  absolute=True runs it on the absolute values (the error scale)."""
    f = np.abs if absolute else (lambda x: x)
    Ht = torch.tensor(f(H), dtype=torch.float64, requires_grad=True)
    Wt = torch.tensor(f(W), dtype=torch.float64, requires_grad=True)
    Wst = torch.tensor(f(Ws), dtype=torch.float64, requires_grad=True)
    pre = Ht @ Wst
    if mask is not None:
        pre = pre * torch.tensor(mask, dtype=torch.float64) / keep
    dst, src, relw, norm = MSGS
    pre = add_messages(pre, Ht, Wt, (dst, src, relw, f(norm)), B)
    up = torch.tensor(f(dOut), dtype=torch.float64) * torch.tensor(gate, dtype=torch.float64)
    pre.backward(up)
    return {"out": pre.detach().numpy(), "dH": Ht.grad.numpy(), "dW": Wt.grad.numpy(), "dW_self": Wst.grad.numpy()}


_REF = {}


def references(d, B, H, W, Ws, mask, keep, gate, dOut):
    """(reference, error scale) for one layer shape and ReLU gate; the cases of one table row share them"""
    key = (d, B, mask is not None, hash(gate.tobytes()))
    if key not in _REF:
        if any(k[:2] != (d, B) for k in _REF):
            _REF.clear()
        _REF[key] = (reference(d, B, H, W, Ws, mask, keep, gate, dOut),
                     reference(d, B, H, W, Ws, mask, keep, gate, dOut, absolute=True))
    return _REF[key]


def run_layer(row, H, W, Ws, dOut, mask, keep, relu):
    g = ops.Graph.from_messages(*MSGS, V, V, 2 * R, device=0)
    Ht = torch.tensor(H, device=DEV, requires_grad=True)
    Wf = torch.tensor(W[:R], device=DEV, requires_grad=True)
    Wb = torch.tensor(W[R:], device=DEV, requires_grad=True)
    Wst = torch.tensor(Ws, device=DEV, requires_grad=True)
    m = None if mask is None else torch.tensor(mask, device=DEV)
    out = ops.block_layer(Ht, Wf, Wb, Wst, g, row.B, m, keep, relu)
    out.backward(torch.tensor(dOut, device=DEV))
    torch.cuda.synchronize()
    return {"out": out.detach().cpu().numpy(), "dH": Ht.grad.cpu().numpy(),
            "dW": np.concatenate([Wf.grad.cpu().numpy(), Wb.grad.cpu().numpy()]), "dW_self": Wst.grad.cpu().numpy()}


def assert_elementwise(name, got, ref, scale, tol=TOL):
    assert np.isfinite(got).all(), name + " has non-finite values"
    err = np.abs(got.astype(np.float64) - ref)
    bad = err > tol * scale
    if bad.any():
        i = np.unravel_index(np.argmax(err - tol * scale), err.shape)
        raise AssertionError("%s: %d elements over %.0e * sum|terms|; worst at %s: got %.9g ref %.9g scale %.3g "
                             "(|err| / scale = %.3g)" % (name, int(bad.sum()), tol, i, got[i], ref[i], scale[i],
                                                         err[i] / max(scale[i], 1e-300)))


@pytest.fixture
def walk_row(request, monkeypatch):
    row = request.param
    for k in ("RGCN_STG_FWD", "RGCN_STG_BWD", "RGCN_STG_TEAM", "RGCN_REL_GROUP", "RGCN_REL_NV", "RGCN_FUSE_DW_S5",
              "RGCN_NO_FUSE_DW", "RGCN_BLOCK_ALGO", "RGCN_STG_SMS", "RGCN_ITEM_MAX", "RGCN_SUPERTILE_ROWS"):
        monkeypatch.delenv(k, raising=False)
    for k, v in row.env.items():
        monkeypatch.setenv(k, v)
    slice_norms = ops._SLICE_NORMS          # the training tests may leave the slice-norm pass switched on
    ops.set_slice_norms(False)
    _lib.set_option("block_algo", row.algo)
    yield row
    _lib.set_option("block_algo", -1)
    ops.set_slice_norms(slice_norms)


# (name, RGCN_ITEM_MAX, RGCN_STG_SMS, RGCN_SUPERTILE_ROWS, relu and dropout)
SETTINGS = [("item%d-%s-%s" % (im, "sms1" if sms else "allsms", act), im, sms, None, act == "relu-mask")
            for im in (8, 128, 1000) for sms in (None, 1) for act in ("plain", "relu-mask")]
SETTINGS.append(("item128-supertile7-relu-mask", 128, None, 7, True))


def _cases():
    out = []
    for row in bw.ROWS:
        for st in SETTINGS:
            if st[2] and not row.staged:    # RGCN_STG_SMS only sizes the persistent grids of the staged kernels
                continue
            out.append(pytest.param(row, st, id="%s-%s" % (row.name, st[0])))
    return out


@pytest.mark.parametrize("walk_row,setting", _cases(), indirect=["walk_row"])
def test_walk_boundaries_vs_float64(walk_row, setting, monkeypatch):
    row = walk_row
    _, item_max, sms, supertile, act = setting
    monkeypatch.setenv("RGCN_ITEM_MAX", str(item_max))
    if sms:
        monkeypatch.setenv("RGCN_STG_SMS", str(sms))
    if supertile:
        monkeypatch.setenv("RGCN_SUPERTILE_ROWS", str(supertile))
    d, B = row.d, row.B
    H, W, Ws, dOut, mask = layer_inputs(d, B)
    mask, keep = (mask, 0.8) if act else (None, 1.0)
    got = run_layer(row, H, W, Ws, dOut, mask, keep, act)
    gate = (got["out"] > 0) if act else np.ones_like(got["out"], dtype=bool)
    ref, scale = references(d, B, H, W, Ws, mask, keep, gate, dOut)
    ref_out = np.maximum(ref["out"], 0) if act else ref["out"]
    assert_close("out", got["out"], ref_out)
    assert_elementwise("out", got["out"], ref_out, scale["out"])
    if act:   # gate flips are only allowed where the pre-activation is within its own bound of zero
        flips = gate != (ref["out"] > 0)
        assert (np.abs(ref["out"][flips]) <= TOL * scale["out"][flips]).all()
    for k in ("dH", "dW", "dW_self"):
        assert_close(k, got[k], ref[k])
        assert_elementwise(k, got[k], ref[k], scale[k])
    assert np.abs(got["dW"][52:]).max() == 0, "weight ids without messages got a gradient"
    if row.staged:   # dynamic work distribution: a second run may hand the items to other warps
        again = run_layer(row, H, W, Ws, dOut, mask, keep, act)
        for k in ("out", "dH", "dW", "dW_self"):
            assert_elementwise(k + " (second run)", again[k], got[k].astype(np.float64), scale[k])


@pytest.mark.parametrize("walk_row", [pytest.param(r, id=r.name) for r in bw.ROWS], indirect=True)
def test_walk_row_launches_exactly_its_kernels(walk_row):
    """Run one forward + backward under torch.profiler (CUPTI activity tracing) and compare the block-layer kernels
    launched with the row: the table says which walk each configuration really takes."""
    from torch.profiler import ProfilerActivity, profile
    row = walk_row
    H, W, Ws, dOut, mask = layer_inputs(row.d, row.B)
    run_layer(row, H, W, Ws, dOut, None, 1.0, True)       # first launch outside the trace (attribute setup)
    # the dispatch is deterministic, so the union of several traces adds no kernel; it only covers a trace whose
    # activity records were not all delivered.  A trace holding both re-layouts (the first kernel of the forward,
    # the last of the backward) is complete.
    launched = set()
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            run_layer(row, H, W, Ws, dOut, None, 1.0, True)
        traced = {c for c in map(bw.canonical, {e.name for e in prof.events()}) if c is not None}
        launched |= traced
        if set(bw.LAYOUT) <= traced:
            break
    assert set(bw.LAYOUT) <= launched, ("no weight-table re-layout traced: is kernel tracing working?", launched)
    walks = launched - set(bw.NON_WALK)
    assert walks == row.kernels, (sorted(walks), sorted(row.kernels))


MO_V_DST, MO_V_SRC = 300, 500


@pytest.mark.parametrize("algo", [-1, 1, 0], ids=["default", "rel-major", "dst-major"])
@pytest.mark.parametrize("d,B", [(512, 64), (400, 50)])
def test_messages_only_entry_points(d, B, algo):
    """rgcn_block_aggregate / _backward (the halo messages of the node-sharded layers): V_src > V_dst, `out` and
    dW_forward / dW_backward accumulated into non-zero tensors."""
    rng = np.random.RandomState(d + algo)
    s, M = d // B, 9000
    dst = rng.randint(0, MO_V_DST, M).astype(np.int32)
    src = rng.randint(0, MO_V_SRC, M).astype(np.int32)
    relw = rng.randint(0, 2 * R, M).astype(np.int32)
    norm = rng.uniform(0.1, 1.0, M).astype(np.float32)
    X = rng.normal(0, 1, (MO_V_SRC, d)).astype(np.float32)
    G = rng.normal(0, 1, (MO_V_DST, d)).astype(np.float32)
    W = rng.normal(0, 0.3, (2 * R, B, s, s)).astype(np.float32)
    out0 = rng.normal(0, 1, (MO_V_DST, d)).astype(np.float32)
    dW0 = rng.normal(0, 1, W.shape).astype(np.float32)
    _lib.set_option("block_algo", algo)
    try:
        g = ops.Graph.from_messages(dst, src, relw, norm, MO_V_DST, MO_V_SRC, 2 * R, device=0)
        cu = lambda a: torch.tensor(a, device=DEV)
        out = cu(out0)
        ops.block_aggregate_(out, cu(X), cu(W[:R]), cu(W[R:]), g, B)
        dWf, dWb = cu(dW0[:R]), cu(dW0[R:])
        dX, _, _ = ops.block_aggregate_backward(cu(X), cu(W[:R]), cu(W[R:]), cu(G), g, B, dWf, dWb)
        torch.cuda.synchronize()
    finally:
        _lib.set_option("block_algo", -1)

    def restate(Xa, Wa, Ga, out_init, dW_init):
        Xt = torch.tensor(Xa, dtype=torch.float64, requires_grad=True)
        Wt = torch.tensor(Wa, dtype=torch.float64, requires_grad=True)
        agg = add_messages(torch.zeros(MO_V_DST, d, dtype=torch.float64), Xt, Wt, (dst, src, relw, norm), B)
        agg.backward(torch.tensor(Ga, dtype=torch.float64))
        return agg.detach().numpy() + out_init, Xt.grad.numpy(), Wt.grad.numpy() + dW_init

    f64 = lambda a: a.astype(np.float64)
    ref = restate(X, W, G, f64(out0), f64(dW0))
    scale = restate(np.abs(X), np.abs(W), np.abs(G), np.abs(f64(out0)), np.abs(f64(dW0)))
    got = (out.cpu().numpy(), dX.cpu().numpy(), np.concatenate([dWf.cpu().numpy(), dWb.cpu().numpy()]))
    for name, a, r, sc in zip(("out", "dX", "dW"), got, ref, scale):
        assert_close(name, a, r)
        assert_elementwise(name, a, r, sc)
