"""GPU: every basis walk-table row (tests/basis_walks.py) against a float64 restatement, on a graph whose run
structure is set by construction.

The basis walks take a row's messages from a CSR view sorted by weight id, so a row's messages come as runs, one per
weight id, in increasing weight-id order; the direction switches where the weight id reaches R.  Family A prescribes
the runs of destination rows (the forward walk and the dC walk), family B those of source rows (the backward walk that
builds P, and the one-hot layer's dW walk).  A's sources stay in A and B's destinations in B, so each family's rows
hold exactly their pattern in their own view; tests assert that through the graph export.  The patterns cover a single
message, all-singleton rows, single long runs, forward-only and backward-only rows, direction switches inside and at
the edges of the 4-message unroll and the 32-message index batch, and a long mixed row that the default item size
splits.  One row of a 129-singleton pattern needs more than 128 weight ids, hence R = 80.

Error bound: besides the suite's global max|a-b| / max|b| < 1e-4, every element must satisfy
|got - ref| <= TOL * ref_abs, where ref_abs is the same float64 computation on the absolute values of every input
(the sum of the absolute values of the terms).  The ReLU gate of the backward reference is taken from the kernel's
own `out`; a gate may differ from the float64 pre-activation's sign only where that pre-activation is within its
own bound of zero."""
import numpy as np
import pytest
import torch

import basis_walks as bw
import fresh_process
from relationprediction_b200 import _lib, ops
from test_gpu_block_walks import assert_elementwise
from test_gpu_parity import assert_close

pytestmark = pytest.mark.gpu

TOL = 1e-5
DEV = "cuda:0"
V, R = 420, 80                 # 2R = 160 weight ids
V_HALO = 300                   # V_dst of the halo variant (V_src stays V)
RGCN_ERR_INVALID = -1
KEEP = 0.8

# (forward run lengths, backward run lengths) of one row; the direction switches after sum(forward) messages
PATTERNS = ([([1], []), ([], [1]),                                            # a single message
             ([1] * 17, [1] * 16), ([1] * 40, [1] * 25), ([1] * 64, [1] * 65)]  # 33, 65, 129 singleton runs
            + [([L], []) for L in (31, 32, 33, 64, 65, 129, 300)]            # one run, forward only
            + [([], [L]) for L in (31, 32, 33, 64, 65, 129, 300)]            # one run, backward only
            + [([1], [40]), ([3, 1], [5, 30]), ([31], [2]), ([30, 2], [1, 1, 7]), ([33], [33]),  # switch at 1..33
               ([7, 1, 40, 3, 12, 33, 1, 2, 25, 9, 17], [1, 38, 5, 11, 4, 29, 1, 8, 20])])     # 20 runs, 267 msgs
SWITCHES = (1, 4, 31, 32, 33)
FWD_POOL, BWD_POOL = np.arange(0, R - 2), np.arange(R, 2 * R - 2)   # ids R-2, R-1, 2R-2, 2R-1 never used


def _rows(lo, hi, parity):
    return np.array([r for r in range(lo, hi) if r % 2 == parity and r % 10 != 3])   # r = 3 (mod 10): isolated


def pattern_messages(seed=0):
    """Messages of both families.  Every destination is below V_HALO, so the same messages serve the square graph and
    the halo graph (V_dst = V_HALO < V_src = V); family B's source rows include halo rows, and most halo rows send
    nothing.  Returns (dst, src, relw, norm) and {family: [(row, [(weight id, run length), ...]), ...]}."""
    rng = np.random.RandomState(seed)
    rows_a, rows_b = _rows(0, V_HALO, 0), _rows(0, V, 1)
    dst_b = rows_b[rows_b < V_HALO]
    runs = {}
    dst, src, relw = [], [], []
    for fam, rows, others in (("A", rows_a, rows_a), ("B", rows_b, dst_b)):
        keys = np.sort(rng.choice(rows, len(PATTERNS), replace=False))
        keys[0], keys[-1] = rows[0], rows[-1]                   # the first and last row of the family in use
        runs[fam] = []
        for key, (fl, bl) in zip(keys, PATTERNS):
            ids = np.concatenate([np.sort(rng.choice(FWD_POOL, len(fl), replace=False)),
                                  np.sort(rng.choice(BWD_POOL, len(bl), replace=False))]).astype(np.int64)
            lens = list(fl) + list(bl)
            runs[fam].append((int(key), list(zip(ids.tolist(), lens))))
            n = sum(lens)
            k = np.full(n, key)
            o = rng.choice(others, n)
            dst.append(k if fam == "A" else o)
            src.append(o if fam == "A" else k)
            relw.append(np.repeat(ids, lens))
    dst, src, relw = (np.concatenate(a).astype(np.int32) for a in (dst, src, relw))
    perm = rng.permutation(len(dst))                              # the graph builder, not the input order, makes runs
    norm = rng.uniform(0.1, 1.0, len(dst)).astype(np.float32)
    return (dst[perm], src[perm], relw[perm], norm), runs


MSGS, RUNS = pattern_messages()
UNUSED_IDS = np.setdiff1d(np.arange(2 * R), MSGS[2])
SILENT_HALO = np.setdiff1d(np.arange(V_HALO, V), MSGS[1])        # halo rows that send nothing


def make_graph(halo):
    return ops.Graph.from_messages(*MSGS, V_HALO if halo else V, V, 2 * R, device=0)


def run_length_encoding(a):
    if len(a) == 0:
        return []
    cut = np.flatnonzero(np.diff(a)) + 1
    starts = np.concatenate([[0], cut])
    ends = np.concatenate([cut, [len(a)]])
    return [(int(a[s]), int(e - s)) for s, e in zip(starts, ends)]


# ---- inputs and float64 references ------------------------------------------------------------------------------------
def layer_inputs(row, seed=1):
    """float32 numpy inputs for one table row (the feature layer: H, Vf, Vb; the one-hot layer: Wf, Wb)"""
    rng = np.random.RandomState(seed + row.d * 7 + row.B)
    d, B = row.d, row.B
    inp = {"Cf": rng.normal(0, 1, (R, B)), "Cb": rng.normal(0, 1, (R, B))}
    if row.onehot:
        inp.update(Wf=rng.normal(0, 0.3, (V, B, d)), Wb=rng.normal(0, 0.3, (V, B, d)),
                   Ws=rng.normal(0, 0.3, (V, d)))
    else:
        inp.update(H=rng.normal(0, 1, (V, d)), Vf=rng.normal(0, 1 / np.sqrt(d * B), (d, B, d)),
                   Vb=rng.normal(0, 1 / np.sqrt(d * B), (d, B, d)), Ws=rng.normal(0, 1 / np.sqrt(d), (d, d)))
    inp = {k: v.astype(np.float32) for k, v in inp.items()}
    dOut = rng.normal(0, 1, (V, d)).astype(np.float32)
    mask = (rng.uniform(size=(V, d)) < KEEP).astype(np.uint8)
    return inp, dOut, mask


def grad_names(row):
    return ("dWf", "dWb", "dCf", "dCb", "dWs") if row.onehot else ("dH", "dVf", "dVb", "dCf", "dCb", "dWs")


def reference(row, V_dst, inp, mask, keep, gate, dOut, absolute=False):
    """float64 autograd restatement over the messages, on the GPU, re-associated as the kernels compute it:
    feature layer  Agg_dir[v, k, b] = sum_m norm_m C_dir[w_m, b] H[src_m, k];
                   pre = mask / keep * (H[:V_dst] W_self) + Agg_f.reshape(V_dst, d B) @ Vf.reshape(d B, d) + (b);
    one-hot layer  pre = mask / keep * W_self + sum_m norm_m sum_b C_dir[w_m, b] W_dir[src_m, b, :] at dst_m;
    gradients of sum(pre * gate * dOut).  absolute=True runs it on the absolute values (the error scale)."""
    f = torch.abs if absolute else (lambda x: x)
    t = {k: f(torch.tensor(v, dtype=torch.float64, device=DEV)).requires_grad_(True) for k, v in inp.items()}
    dst, src, relw, norm = (torch.tensor(a, device=DEV) for a in MSGS)
    dst, src, relw = dst.long(), src.long(), relw.long()
    norm = f(norm.double())
    d, B = row.d, row.B
    fwd = relw < R
    C = torch.cat([t["Cf"], t["Cb"]])
    coef = norm[:, None] * C[relw]                                      # [M, B]
    drop = 1.0 if mask is None else torch.tensor(mask[:V_dst], dtype=torch.float64, device=DEV) / keep
    res = {}
    if row.onehot:
        Wsrc = torch.where(fwd[:, None, None], t["Wf"][src], t["Wb"][src])  # [M, B, d]
        msg = (coef[:, :, None] * Wsrc).sum(1)
        pre = (t["Ws"][:V_dst] * drop).index_add(0, dst, msg)
        pairs = (("dWf", "Wf"), ("dWb", "Wb"), ("dCf", "Cf"), ("dCb", "Cb"), ("dWs", "Ws"))
    else:
        contrib = t["H"][src][:, :, None] * coef[:, None, :]             # [M, d, B]
        zero = torch.zeros(V_dst, d, B, dtype=torch.float64, device=DEV)
        agg_f = zero.index_add(0, dst[fwd], contrib[fwd]).reshape(V_dst, d * B)
        agg_b = zero.index_add(0, dst[~fwd], contrib[~fwd]).reshape(V_dst, d * B)
        pre = (t["H"][:V_dst] @ t["Ws"]) * drop
        pre = pre + agg_f @ t["Vf"].reshape(d * B, d) + agg_b @ t["Vb"].reshape(d * B, d)
        res["saved"] = torch.cat([agg_f, agg_b], 1).detach().cpu().numpy()
        pairs = (("dH", "H"), ("dVf", "Vf"), ("dVb", "Vb"), ("dCf", "Cf"), ("dCb", "Cb"), ("dWs", "Ws"))
    up = f(torch.tensor(dOut[:V_dst], dtype=torch.float64, device=DEV)) * torch.tensor(gate, device=DEV)
    pre.backward(up)
    res["out"] = pre.detach().cpu().numpy()
    res.update({g: t[k].grad.cpu().numpy() for g, k in pairs})
    return res


_REF = {}


def references(row, V_dst, inp, mask, keep, gate, dOut):
    """(reference, error scale) for one row, graph and ReLU gate; the cases of one table row share them"""
    key = (row.name, V_dst, mask is not None, hash(gate.tobytes()))
    if key not in _REF:
        if any(k[0] != row.name for k in _REF):
            _REF.clear()
        _REF[key] = (reference(row, V_dst, inp, mask, keep, gate, dOut),
                     reference(row, V_dst, inp, mask, keep, gate, dOut, absolute=True))
    return _REF[key]


# ---- the product layer -----------------------------------------------------------------------------------------------
def run_layer(row, g, inp, dOut, mask, keep, relu):
    """ops.basis_layer / ops.basis_onehot_layer forward + backward: numpy out and gradients"""
    t = {k: torch.tensor(v, device=DEV).requires_grad_(True) for k, v in inp.items()}
    Vd = g.V_dst
    m = None if mask is None else torch.tensor(mask[:Vd], device=DEV)
    if row.onehot:
        Ws = t["Ws"] if Vd == V else torch.tensor(inp["Ws"][:Vd], device=DEV).requires_grad_(True)
        out = ops.basis_onehot_layer(t["Wf"], t["Wb"], t["Cf"], t["Cb"], Ws, g, m, keep, relu)
        leaves = (("dWf", t["Wf"]), ("dWb", t["Wb"]), ("dCf", t["Cf"]), ("dCb", t["Cb"]), ("dWs", Ws))
    else:
        out = ops.basis_layer(t["H"], t["Vf"], t["Vb"], t["Cf"], t["Cb"], t["Ws"], g, m, keep, relu)
        leaves = (("dH", t["H"]), ("dVf", t["Vf"]), ("dVb", t["Vb"]), ("dCf", t["Cf"]), ("dCb", t["Cb"]),
                  ("dWs", t["Ws"]))
    out.backward(torch.tensor(dOut[:Vd], device=DEV))
    torch.cuda.synchronize()
    res = {"out": out.detach().cpu().numpy()}
    res.update({k: v.grad.cpu().numpy() for k, v in leaves})
    return res


def onehot_inputs_for(inp, V_dst):
    """the one-hot layer's W_self has V_dst rows"""
    return dict(inp, Ws=inp["Ws"][:V_dst]) if "Wf" in inp else inp


@pytest.fixture
def basis_env(monkeypatch):
    """environment knobs cleared, slice-norm pass off, library options at their defaults; all restored after"""
    for k in ("RGCN_ITEM_MAX", "RGCN_SUPERTILE_ROWS", "RGCN_PREP", "RGCN_KEEP_MID", "RGCN_BLOCK_ALGO"):
        monkeypatch.delenv(k, raising=False)
    slice_norms = ops._SLICE_NORMS
    ops.set_slice_norms(False)
    _lib.set_option("block_algo", -1)
    _lib.set_option("graph_views", 3)
    yield monkeypatch
    _lib.set_option("block_algo", -1)
    _lib.set_option("graph_views", 3)
    ops.set_slice_norms(slice_norms)


# ---- the pattern graph holds the intended runs ------------------------------------------------------------------------
@pytest.mark.parametrize("halo", [False, True], ids=["square", "halo"])
def test_pattern_graph_holds_the_intended_runs(basis_env, halo):
    g = make_graph(halo)
    Vd = V_HALO if halo else V
    assert (g.V_dst, g.V_src, g.n_relw) == (Vd, V, 2 * R)
    for fam, ptr_x, relw_x, n_rows in (("A", _lib.X_DST_ROWPTR, _lib.X_DST_RELW, Vd),
                                       ("B", _lib.X_SRC_ROWPTR, _lib.X_SRC_RELW, V)):
        ptr, relw = g.export(ptr_x), g.export(relw_x)
        assert len(ptr) == n_rows + 1
        for row, runs in RUNS[fam]:
            assert run_length_encoding(relw[ptr[row]:ptr[row + 1]]) == runs, (fam, row)
    # every boundary the patterns were written for is present
    switches = {sum(n for w, n in runs if w < R) for _, runs in RUNS["A"] if runs[0][0] < R <= runs[-1][0]}
    assert switches >= set(SWITCHES)
    lens = {n for _, runs in RUNS["A"] for _, n in runs}
    assert lens >= {1, 31, 32, 33, 64, 65, 129, 300}
    assert {len(runs) for _, runs in RUNS["A"]} >= {1, 20, 33, 65, 129}
    assert max(sum(n for _, n in runs) for _, runs in RUNS["A"] if len(runs) == 20) > 128
    src = g.export(_lib.X_SRC_ROWPTR)
    assert any(row >= V_HALO for row, _ in RUNS["B"]) and len(SILENT_HALO) > 0
    assert all(src[r + 1] == src[r] for r in SILENT_HALO)
    assert len(UNUSED_IDS) >= 4
    # the weight ids on either side of the direction switch carry messages in both families
    for fam in ("A", "B"):
        ids = {w for _, runs in RUNS[fam] for w, _ in runs}
        assert {R - 3, R} <= ids, fam
    dst = g.export(_lib.X_DST_ROWPTR)
    isolated = np.arange(3, V, 10)
    assert all(src[r + 1] == src[r] for r in isolated) and all(dst[r + 1] == dst[r] for r in isolated if r < Vd)


@pytest.mark.parametrize("item_max,split", [(8, True), (128, True), (1000, False)])
def test_item_sizes_split_the_intended_rows(basis_env, item_max, split):
    basis_env.setenv("RGCN_ITEM_MAX", str(item_max))
    info = make_graph(False).info()
    assert info[12] == item_max
    assert (info[7] > 0 and info[8] > 0) == split and (info[7] == 0 and info[8] == 0) == (not split)


# ---- every row against float64 ----------------------------------------------------------------------------------------
# (name, RGCN_ITEM_MAX, relu and dropout, halo graph)
SETTINGS = [("item%d-%s" % (im, act), im, act == "relu-mask", False)
            for im in (8, 128, 1000) for act in ("plain", "relu-mask")]
SETTINGS.append(("item128-relu-mask-halo", 128, True, True))


def check_case(row, got, ref, scale, relu):
    ref_out = np.maximum(ref["out"], 0) if relu else ref["out"]
    assert_close("out", got["out"], ref_out)
    assert_elementwise("out", got["out"], ref_out, scale["out"], TOL)
    if relu:   # gate flips are only allowed where the pre-activation is within its own bound of zero
        gate = got["out"] > 0
        flips = gate != (ref["out"] > 0)
        assert (np.abs(ref["out"][flips]) <= TOL * scale["out"][flips]).all()
    for k in grad_names(row):
        assert_close(k, got[k], ref[k])
        assert_elementwise(k, got[k], ref[k], scale[k], TOL)


@pytest.mark.parametrize("setting", SETTINGS, ids=[s[0] for s in SETTINGS])
@pytest.mark.parametrize("row", bw.ROWS, ids=[r.name for r in bw.ROWS])
def test_walk_boundaries_vs_float64(basis_env, row, setting):
    _, item_max, act, halo = setting
    basis_env.setenv("RGCN_ITEM_MAX", str(item_max))
    g = make_graph(halo)
    Vd = g.V_dst
    inp, dOut, mask = layer_inputs(row)
    mask, keep = (mask, KEEP) if act else (None, 1.0)
    got = run_layer(row, g, inp, dOut, mask, keep, act)
    gate = (got["out"] > 0) if act else np.ones_like(got["out"], dtype=bool)
    ref, scale = references(row, Vd, onehot_inputs_for(inp, Vd), mask, keep, gate, dOut)
    check_case(row, got, ref, scale, act)
    # exact zeros: the coefficients of weight ids without messages, the input rows of halo rows that send nothing
    assert np.abs(got["dCf"][UNUSED_IDS[UNUSED_IDS < R]]).max() == 0
    assert np.abs(got["dCb"][UNUSED_IDS[UNUSED_IDS >= R] - R]).max() == 0
    if halo:
        silent = ("dWf", "dWb") if row.onehot else ("dH",)
        for k in silent:
            assert np.abs(got[k][SILENT_HALO]).max() == 0, k
    # the walks reduce with atomics: a second run agrees within the bound
    again = run_layer(row, g, inp, dOut, mask, keep, act)
    for k in ("out",) + grad_names(row):
        assert_elementwise(k + " (second run)", again[k], got[k].astype(np.float64), scale[k], TOL)


# ---- every output is written ------------------------------------------------------------------------------------------
def _nan(*shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device=DEV)


def _workspace(nbytes, fill):
    """workspace bytes pre-filled with 0xff (every float NaN) or zero"""
    return torch.full((max(int(nbytes), 256),), 255 if fill else 0, dtype=torch.uint8, device=DEV)


def cabi_feature_layer(g, row, inp, dOut, mask, poison):
    """rgcn_basis_forward / _backward called directly, as ops does, with every output and workspace pre-filled with
    NaN (poison=True) or zero"""
    lib = _lib.load()
    P = ops._ptr
    d, B, Vd = row.d, row.B, g.V_dst
    fill = _nan if poison else (lambda *s: torch.zeros(s, dtype=torch.float32, device=DEV))
    t = {k: torch.tensor(v, device=DEV) for k, v in inp.items()}
    m = torch.tensor(mask[:Vd], device=DEV)
    st = ops._stream(DEV)
    out, saved = fill(Vd, d), fill(Vd, 2 * d * B)
    ws = _workspace(lib.rgcn_basis_workspace_bytes(g.handle, d, B, 0), poison)
    _lib.check(lib.rgcn_basis_forward(g.handle, d, B, P(t["H"]), P(t["Vf"]), P(t["Vb"]), P(t["Cf"]), P(t["Cb"]),
                                      P(t["Ws"]), P(m), KEEP, 1, P(out), P(saved), P(ws), ws.numel(), st),
               "rgcn_basis_forward")
    grads = {"dH": fill(V, d), "dVf": fill(d, B, d), "dVb": fill(d, B, d), "dCf": fill(R, B), "dCb": fill(R, B),
             "dWs": fill(d, d)}
    ws = _workspace(lib.rgcn_basis_workspace_bytes(g.handle, d, B, 1), poison)
    dO = torch.tensor(dOut[:Vd], device=DEV)
    _lib.check(lib.rgcn_basis_backward(g.handle, d, B, P(t["H"]), P(t["Vf"]), P(t["Vb"]), P(t["Cf"]), P(t["Cb"]),
                                       P(t["Ws"]), P(m), KEEP, 1, P(out), P(saved), P(dO), P(grads["dH"]),
                                       P(grads["dVf"]), P(grads["dVb"]), P(grads["dCf"]), P(grads["dCb"]),
                                       P(grads["dWs"]), P(ws), ws.numel(), st), "rgcn_basis_backward")
    torch.cuda.synchronize()
    res = {"out": out.cpu().numpy(), "saved": saved.cpu().numpy()}
    res.update({k: v.cpu().numpy() for k, v in grads.items()})
    return res


def cabi_onehot_layer(g, row, inp, dOut, mask, poison):
    """rgcn_basis_onehot_forward / _backward called directly with outputs and workspaces pre-filled"""
    lib = _lib.load()
    P = ops._ptr
    d, B, Vd = row.d, row.B, g.V_dst
    fill = _nan if poison else (lambda *s: torch.zeros(s, dtype=torch.float32, device=DEV))
    t = {k: torch.tensor(v, device=DEV) for k, v in onehot_inputs_for(inp, Vd).items()}
    m = torch.tensor(mask[:Vd], device=DEV)
    st = ops._stream(DEV)
    out = fill(Vd, d)
    ws = _workspace(lib.rgcn_basis_onehot_workspace_bytes(g.handle, d, B, 0), poison)
    _lib.check(lib.rgcn_basis_onehot_forward(g.handle, d, B, P(t["Wf"]), P(t["Wb"]), P(t["Cf"]), P(t["Cb"]),
                                             P(t["Ws"]), P(m), KEEP, 1, P(out), P(ws), ws.numel(), st),
               "rgcn_basis_onehot_forward")
    grads = {"dWf": fill(V, B, d), "dWb": fill(V, B, d), "dCf": fill(R, B), "dCb": fill(R, B), "dWs": fill(Vd, d)}
    ws = _workspace(lib.rgcn_basis_onehot_workspace_bytes(g.handle, d, B, 1), poison)
    dO = torch.tensor(dOut[:Vd], device=DEV)
    _lib.check(lib.rgcn_basis_onehot_backward(g.handle, d, B, P(t["Wf"]), P(t["Wb"]), P(t["Cf"]), P(t["Cb"]), P(m),
                                              KEEP, 1, P(out), P(dO), P(grads["dWf"]), P(grads["dWb"]),
                                              P(grads["dCf"]), P(grads["dCb"]), P(grads["dWs"]), P(ws), ws.numel(),
                                              st), "rgcn_basis_onehot_backward")
    torch.cuda.synchronize()
    res = {"out": out.cpu().numpy()}
    res.update({k: v.cpu().numpy() for k, v in grads.items()})
    return res


def _written_case(basis_env, row, halo):
    """Split rows (RGCN_ITEM_MAX = 8: their rows are cleared by zero_rows, then reduced into) and unsplit rows with
    one direction only (explicit zeros) on the poisoned run must match the zero-filled run and float64."""
    basis_env.setenv("RGCN_ITEM_MAX", "8")
    g = make_graph(halo)
    Vd = g.V_dst
    inp, dOut, mask = layer_inputs(row)
    call = cabi_onehot_layer if row.onehot else cabi_feature_layer
    clean = call(g, row, inp, dOut, mask, poison=False)
    poisoned = call(g, row, inp, dOut, mask, poison=True)
    ref, scale = references(row, Vd, onehot_inputs_for(inp, Vd), mask, KEEP, clean["out"] > 0, dOut)
    check_case(row, clean, ref, scale, True)
    for k in clean:
        assert np.isfinite(poisoned[k]).all(), k + " has entries the kernels never wrote"
        assert_elementwise(k + " (poisoned run)", poisoned[k], clean[k].astype(np.float64), scale[k], TOL)


FEAT_ROWS = [r for r in bw.ROWS if not r.onehot]
ONEHOT_ROWS = [r for r in bw.ROWS if r.onehot]


@pytest.mark.parametrize("halo", [False, True], ids=["square", "halo"])
@pytest.mark.parametrize("row", FEAT_ROWS, ids=[r.name for r in FEAT_ROWS])
def test_feature_layer_writes_every_output(basis_env, row, halo):
    _written_case(basis_env, row, halo)


@pytest.mark.parametrize("halo", [False, True], ids=["square", "halo"])
@pytest.mark.parametrize("row", ONEHOT_ROWS, ids=[r.name for r in ONEHOT_ROWS])
def test_onehot_layer_writes_every_output(basis_env, row, halo):
    _written_case(basis_env, row, halo)


# ---- the dispatch ----------------------------------------------------------------------------------------------------
ROW_RANGE = "basis-walk-row:"


def trace_rows(rows, g):
    """{row name: canonical k_basis_* kernels} of one forward + backward per row, all rows in ONE torch.profiler
    (CUPTI activity) session: each row runs inside its own record_function range and synchronizes before the range
    closes, so a kernel belongs to the range that holds the midpoint of its execution."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile, record_function
    inputs = {r.name: layer_inputs(r) for r in rows}
    for r in rows:                                          # first launches outside the trace (attribute setup)
        inp, dOut, _ = inputs[r.name]
        run_layer(r, g, inp, dOut, None, 1.0, True)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for r in rows:
            inp, dOut, _ = inputs[r.name]
            with record_function(ROW_RANGE + r.name):
                run_layer(r, g, inp, dOut, None, 1.0, True)
    events = list(prof.events())
    ranges = [(e.time_range.start, e.time_range.end, e.name[len(ROW_RANGE):]) for e in events
              if e.name.startswith(ROW_RANGE) and e.device_type == DeviceType.CPU]
    launched = {r.name: set() for r in rows}
    for e in events:
        c = bw.canonical(e.name)
        if c is None or e.device_type != DeviceType.CUDA:
            continue
        mid = 0.5 * (e.time_range.start + e.time_range.end)
        owners = [n for s, t, n in ranges if s <= mid <= t]
        assert len(owners) == 1, (c, mid, owners)
        launched[owners[0]].add(c)
    return launched


_CHILD = """
import json
import basis_walks as bw
import test_gpu_basis_walks as t
rows = [bw.BY_NAME[n] for n in sys.argv[1:]]
print("RESULT " + json.dumps({k: sorted(v) for k, v in t.trace_rows(rows, t.make_graph(False)).items()}))
"""


def trace_in_child(rows):
    """trace_rows in a fresh interpreter (tests/fresh_process.py says why)"""
    return {k: set(v) for k, v in fresh_process.run_json(_CHILD, *[r.name for r in rows]).items()}


@pytest.fixture(scope="module")
def traced_walks():
    return trace_in_child(bw.ROWS)


@pytest.mark.parametrize("row", bw.ROWS, ids=[r.name for r in bw.ROWS])
def test_walk_row_launches_exactly_its_kernels(traced_walks, row):
    """Compare the basis walk kernels one forward + backward launched (traced with torch.profiler) with the row: the
    table says which walk each (B, d) really takes."""
    launched = set(traced_walks[row.name])
    # the dispatch is deterministic: the union with more traces adds no kernel, it only covers a trace whose
    # activity records were not all delivered
    for _ in range(2):
        if launched == row.kernels:
            break
        launched |= trace_in_child([row])[row.name]
    assert launched == row.kernels, (sorted(launched), sorted(row.kernels))


# ---- argument checks --------------------------------------------------------------------------------------------------
def test_graphs_without_csr_views_are_rejected(basis_env):
    """the basis walks need the CSR views: a graph prepared with graph_views = 2 (weight-id-major views only)"""
    lib = _lib.load()
    row = bw.BY_NAME["feat-B2-d8"]
    d, B = row.d, row.B
    _lib.set_option("graph_views", 2)
    g = ops.Graph.from_device_messages(*(torch.tensor(a, device=DEV) for a in MSGS), V, V, 2 * R)
    _lib.set_option("graph_views", 3)
    inp, dOut, _ = layer_inputs(row)
    t = {k: torch.tensor(v, device=DEV) for k, v in inp.items()}
    P = ops._ptr
    buf = torch.zeros(V * 2 * d * B + 4 * d * d * B + 2 * V * d, dtype=torch.float32, device=DEV)
    ws = torch.zeros(int(lib.rgcn_basis_workspace_bytes(g.handle, d, B, 1)), dtype=torch.uint8, device=DEV)
    st = ops._stream(DEV)
    rc = lib.rgcn_basis_forward(g.handle, d, B, P(t["H"]), P(t["Vf"]), P(t["Vb"]), P(t["Cf"]), P(t["Cb"]),
                                P(t["Ws"]), None, 1.0, 1, P(buf), P(buf), P(ws), ws.numel(), st)
    assert rc == RGCN_ERR_INVALID and b"CSR" in lib.rgcn_last_error()
    rc = lib.rgcn_basis_backward(g.handle, d, B, P(t["H"]), P(t["Vf"]), P(t["Vb"]), P(t["Cf"]), P(t["Cb"]),
                                 P(t["Ws"]), None, 1.0, 1, P(buf), P(buf), P(buf), P(buf), P(buf), P(buf), P(buf),
                                 P(buf), P(buf), P(ws), ws.numel(), st)
    assert rc == RGCN_ERR_INVALID and b"CSR" in lib.rgcn_last_error()
    torch.cuda.synchronize()
    assert torch.count_nonzero(buf).item() == 0 and torch.count_nonzero(ws).item() == 0


def test_fewer_sources_than_destinations_is_rejected(basis_env):
    """the self loop reads H rows [0, V_dst): V_src < V_dst is an argument error of both basis layers"""
    dst, src, relw, norm = MSGS        # every destination is below V_HALO: reversed, the messages fit V_src = V_HALO
    g = ops.Graph.from_messages(src, dst, relw, norm, V, V_HALO, 2 * R, device=0)
    assert (g.V_dst, g.V_src) == (V, V_HALO)
    d, B = 8, 2
    H = torch.zeros(V_HALO, d, device=DEV)
    Vf, Vb = torch.zeros(d, B, d, device=DEV), torch.zeros(d, B, d, device=DEV)
    C = torch.zeros(R, B, device=DEV)
    with pytest.raises(_lib.RgcnError, match="V_src >= V_dst"):
        ops.basis_layer(H, Vf, Vb, C, C, torch.zeros(d, d, device=DEV), g)
    W = torch.zeros(V_HALO, B, d, device=DEV)
    with pytest.raises(_lib.RgcnError, match="V_src >= V_dst"):
        ops.basis_onehot_layer(W, W, C, C, torch.zeros(V, d, device=DEV), g)
