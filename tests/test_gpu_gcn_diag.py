"""GPU: the diagonal R-GCN layer (Encoder Name=gcn_diag), ops.diag_layer over rgcn_diag_forward / _backward, against a
float64 gather restatement of the reference layer (gcn_diag.py), the IndexedSlices sum of squares against float64 and
against rgcn_block_slice_sumsq with blocks of size 1, the reference-code goldens of tests/golden/make_gcn_diag_golden.py,
and a driver run.  Tolerance 1e-4 relative (max |error| / max |reference|): fp32 kernels with non-deterministic
reduction order."""
import ctypes

import numpy as np
import pytest
import torch

import fresh_process
import gcn_diag_walks as gw
from relationprediction_b200 import _lib, ops
from relationprediction_b200 import train as driver
from test_gcn_diag_cpu import CASES, build_model, case_shape, load_case
from test_gpu_reference_golden import layers_of
from test_gpu_train import TOY_EXP, write_toy
import gcn_diag_oracle as gd

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KEEP = 0.8
NAMES = ("H", "D_forward", "D_backward", "W_self", "b")


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def make_messages(V_dst, V_src, R, M, seed, dominant=None, empty_dst=()):
    """Random messages (dst < V_dst, src < V_src, weight id < 2R, positive norms); `dominant`: share of the messages
    that carry weight id 0; rows in `empty_dst` receive nothing."""
    rng = np.random.RandomState(seed)
    dst = rng.randint(0, V_dst, M)
    src = rng.randint(0, V_src, M)
    relw = rng.randint(0, 2 * R, M)
    if dominant is not None:
        relw[rng.rand(M) < dominant] = 0
    norm = rng.uniform(0.1, 1.0, M)
    keep = ~np.isin(dst, np.asarray(empty_dst, dtype=np.int64))
    return tuple(a[keep] for a in (dst.astype(np.int32), src.astype(np.int32), relw.astype(np.int32),
                                   norm.astype(np.float32)))


def make_inputs(V_dst, V_src, R, d, seed, mask):
    g = torch.Generator().manual_seed(seed)
    std = 3 / np.sqrt(2 * d)
    w = {"H": torch.randn(V_src, d, generator=g), "D_forward": torch.randn(R, d, generator=g),
         "D_backward": torch.randn(R, d, generator=g), "W_self": torch.randn(d, d, generator=g) * std,
         "b": 0.1 * torch.randn(d, generator=g)}
    m = (torch.rand(V_dst, d, generator=g) < KEEP).to(torch.uint8) if mask else None
    return w, m


def reference(msgs, V_dst, R, w, mask, relu, dOut=None):
    """gcn_diag.py restated over explicit messages, float64 on the GPU (autograd): message m adds
    norm * D_dir[r] * H[src] into dst.  Returns (out, grads, aggregate, slice sums of squares per direction)."""
    dst, src, relw, norm = (torch.as_tensor(a, device=DEV) for a in msgs)
    t = {k: v.to(DEV).double().requires_grad_(True) for k, v in w.items()}
    H = t["H"]
    back = (relw >= R)[:, None]
    r = (relw % R).long()
    D = torch.where(back, t["D_backward"][r], t["D_forward"][r])
    Hs = H[src.long()]
    agg = torch.zeros(V_dst, H.shape[1], dtype=torch.float64, device=DEV).index_add(
        0, dst.long(), D * Hs * norm.double()[:, None])
    S = H[:V_dst] @ t["W_self"]
    if mask is not None:
        S = S * mask.to(DEV).double() / KEEP
    pre = S + agg + t["b"]
    out = torch.relu(pre) if relu else pre
    if dOut is None:
        return pre.detach().cpu(), None, agg.detach().cpu(), None
    out.backward(dOut.to(DEV).double())
    G = dOut.to(DEV).double() * (pre > 0).double() if relu else dOut.to(DEV).double()
    sl = ((norm.double()[:, None] * G[dst.long()] * Hs.detach()) ** 2).sum(1)
    ss = torch.stack([sl[relw < R].sum(), sl[relw >= R].sum()])
    return out.detach().cpu(), {k: v.grad.cpu() for k, v in t.items()}, agg.detach().cpu(), ss.cpu()


def run_layer(graph, w, mask, relu, dOut):
    t = {k: v.to(DEV).float().contiguous().requires_grad_(True) for k, v in w.items()}
    out = ops.diag_layer(*(t[k] for k in NAMES), graph, None if mask is None else mask.to(DEV),
                         KEEP if mask is not None else 1.0, relu)
    out.backward(dOut.to(DEV).float())
    torch.cuda.synchronize()
    return out.detach().double().cpu(), {k: v.grad.double().cpu() for k, v in t.items()}, t


def check_case(msgs, V_dst, V_src, R, d, seed, relu, mask, tol=1e-4):
    w, m = make_inputs(V_dst, V_src, R, d, seed, mask)
    dOut = torch.randn(V_dst, d, generator=torch.Generator().manual_seed(seed + 1), dtype=torch.float64)
    if relu:   # zeros where the pre-activation lies within rounding of the ReLU kink
        pre, _, _, _ = reference(msgs, V_dst, R, w, m, relu)
        dOut = torch.where(pre.abs() < 1e-5 * pre.abs().max(), torch.zeros_like(dOut), dOut)
    graph = ops.Graph.from_messages(*msgs, V_dst, V_src, 2 * R, device=0)
    got_out, got, _ = run_layer(graph, w, m, relu, dOut)
    ref_out, ref, agg, _ = reference(msgs, V_dst, R, w, m, relu, dOut)
    assert rel(got_out, ref_out) < tol
    for k in NAMES:
        assert rel(got[k], ref[k]) < tol, (k, rel(got[k], ref[k]))
    return got_out, got, ref, agg


@pytest.mark.parametrize("d", [4, 24, 200, 500, 512, 516])
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "linear"])
@pytest.mark.parametrize("mask", [True, False], ids=["mask", "nomask"])
def test_layer_matches_float64(d, relu, mask):
    V, R = 300, 7
    msgs = make_messages(V, V, R, 3000, seed=d * 10 + relu * 2 + mask)
    check_case(msgs, V, V, R, d, seed=d + relu, relu=relu, mask=mask)


def test_rows_without_messages_get_exactly_the_self_loop_and_bias():
    """destination rows 0..9 receive no message: their aggregate is exactly zero, so out = dropout(H W_self) + b"""
    V, R, d = 200, 4, 200
    msgs = make_messages(V, V, R, 2000, seed=3, empty_dst=range(10))
    w, _ = make_inputs(V, V, R, d, 4, False)
    g = ops.Graph.from_messages(*msgs, V, V, 2 * R, device=0)
    zero = {k: (torch.zeros_like(v) if k in ("W_self", "b") else v) for k, v in w.items()}
    out, _, _ = run_layer(g, zero, None, False, torch.zeros(V, d, dtype=torch.float64))
    assert float(out[:10].abs().max()) == 0.0 and float(out[10:].abs().max()) > 0
    check_case(msgs, V, V, R, d, seed=5, relu=True, mask=True)


def test_split_rows_on_both_views(monkeypatch):
    """RGCN_ITEM_MAX=8: most rows of both CSR views are cut into several items (scratch rows and the last-arriver
    epilogue forward, vector reductions into dH backward)"""
    monkeypatch.setenv("RGCN_ITEM_MAX", "8")
    V, R = 120, 4
    for d in (24, 500, 516):
        msgs = make_messages(V, V, R, 4000, seed=d)
        check_case(msgs, V, V, R, d, seed=d, relu=True, mask=True)


def test_one_relation_carries_most_messages():
    """90 % of the messages on weight id 0: thousands of runs reduce into one dD row"""
    V, R = 2000, 6
    msgs = make_messages(V, V, R, 60000, seed=5, dominant=0.9)
    _, _, ref, _ = check_case(msgs, V, V, R, 200, seed=6, relu=True, mask=False)
    assert float(ref["D_forward"][0].abs().max()) > 0


def test_halo_rows():
    """V_src > V_dst: rows [V_dst, V_src) of H only send; their dH comes from the messages alone, and a halo row that
    sends nothing gets exactly zero"""
    V_dst, V_src, R = 150, 260, 4
    msgs = make_messages(V_dst, V_src, R, 2500, seed=8)
    keep = msgs[1] != V_src - 1
    msgs = tuple(a[keep] for a in msgs)
    _, got, _, _ = check_case(msgs, V_dst, V_src, R, 200, seed=9, relu=True, mask=True)
    assert float(got["H"][V_src - 1].abs().max()) == 0.0


def test_graph_without_csr_views_is_rejected():
    V, R, d = 60, 3, 16
    msgs = make_messages(V, V, R, 300, seed=10)
    w, _ = make_inputs(V, V, R, d, 11, False)
    t = [w[k].to(DEV).contiguous() for k in NAMES]
    _lib.set_option("graph_views", 2)
    try:
        g2 = ops.Graph.from_device_messages(*(torch.as_tensor(a, device=DEV) for a in msgs), V, V, 2 * R)
    finally:
        _lib.set_option("graph_views", 3)
    with pytest.raises(_lib.RgcnError, match="CSR"):
        ops.diag_layer(*t, g2)
    g3 = ops.Graph.from_device_messages(*(torch.as_tensor(a, device=DEV) for a in msgs), V, V, 2 * R)
    ops.diag_layer(*t, g3)
    with pytest.raises(_lib.RgcnError, match="d % 4"):
        ops.diag_layer(torch.zeros(V, 18, device=DEV), torch.zeros(R, 18, device=DEV), torch.zeros(R, 18, device=DEV),
                       torch.zeros(18, 18, device=DEV), torch.zeros(18, device=DEV), g3)


@pytest.mark.parametrize("d", [24, 500, 516])
def test_slice_sumsq_matches_float64_and_the_block_path(d):
    """with set_slice_norms(True) the backward parks sum_m norm^2 |G[dst] * H[src]|^2 per direction on D_forward /
    D_backward; rgcn_block_slice_sumsq with B = d (blocks of size 1) computes the same quantity by another path"""
    V, R = 400, 5
    msgs = make_messages(V, V, R, 5000, seed=d + 1, dominant=0.3)
    w, m = make_inputs(V, V, R, d, 12, True)
    dOut = torch.randn(V, d, generator=torch.Generator().manual_seed(13), dtype=torch.float64)
    g = ops.Graph.from_messages(*msgs, V, V, 2 * R, device=0)
    ops.set_slice_norms(True)
    try:
        _, _, t = run_layer(g, w, m, False, dOut)
    finally:
        ops.set_slice_norms(False)
    got = torch.stack([t["D_forward"]._slice_sumsq, t["D_backward"]._slice_sumsq]).double().cpu()
    _, _, _, ref = reference(msgs, V, R, w, m, False, dOut)
    assert float((got - ref).abs().max() / ref.abs().max()) < 1e-4
    lib = _lib.load()
    H, G = t["H"].detach().contiguous(), dOut.to(DEV).float().contiguous()
    nb = lib.rgcn_block_slice_sumsq_workspace_bytes(g.handle, d, d)
    ws = torch.empty(int(nb), dtype=torch.uint8, device=DEV)
    ss = torch.empty(2, dtype=torch.float32, device=DEV)
    _lib.check(lib.rgcn_block_slice_sumsq(g.handle, d, d, ctypes.c_void_p(H.data_ptr()),
                                          ctypes.c_void_p(G.data_ptr()), ctypes.c_void_p(ss.data_ptr()),
                                          ctypes.c_void_p(ws.data_ptr()), ws.numel(),
                                          ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "rgcn_block_slice_sumsq")
    torch.cuda.synchronize()
    assert float((got - ss.double().cpu()).abs().max() / ref.abs().max()) < 1e-4


def test_second_run_agrees_with_the_first():
    V, R, d = 300, 5, 500
    msgs = make_messages(V, V, R, 4000, seed=14)
    w, m = make_inputs(V, V, R, d, 15, True)
    dOut = torch.randn(V, d, generator=torch.Generator().manual_seed(16), dtype=torch.float64)
    g = ops.Graph.from_messages(*msgs, V, V, 2 * R, device=0)
    o1, g1, _ = run_layer(g, w, m, True, dOut)
    o2, g2, _ = run_layer(g, w, m, True, dOut)
    assert torch.equal(o1, o2)       # the forward has no atomics on unsplit rows
    for k in NAMES:
        assert rel(g1[k], g2[k]) < 1e-6, k


# ---- the dispatch ----------------------------------------------------------------------------------------------------
_CHILD = """
import json
import numpy as np
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile, record_function
import gcn_diag_walks as gw
import test_gpu_gcn_diag as t
rows = [gw.BY_NAME[n] for n in sys.argv[1:]]
V, R = 100, 3
msgs = t.make_messages(V, V, R, 600, seed=1)
g = t.ops.Graph.from_messages(*msgs, V, V, 2 * R, device=0)
inputs = {r.name: t.make_inputs(V, V, R, r.d, 2, True) for r in rows}
dOut = {r.name: torch.randn(V, r.d, dtype=torch.float64) for r in rows}
for r in rows:
    t.run_layer(g, inputs[r.name][0], inputs[r.name][1], True, dOut[r.name])
with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    for r in rows:
        with record_function("gcn-diag-row:" + r.name):
            t.run_layer(g, inputs[r.name][0], inputs[r.name][1], True, dOut[r.name])
events = list(prof.events())
ranges = [(e.time_range.start, e.time_range.end, e.name[len("gcn-diag-row:"):]) for e in events
          if e.name.startswith("gcn-diag-row:") and e.device_type == DeviceType.CPU]
launched = {r.name: [] for r in rows}
for e in events:
    c = gw.canonical(e.name)
    if c is None or e.device_type != DeviceType.CUDA:
        continue
    mid = 0.5 * (e.time_range.start + e.time_range.end)
    owners = [n for s, u, n in ranges if s <= mid <= u]
    assert len(owners) == 1, (c, owners)
    launched[owners[0]].append(c)
print("RESULT " + json.dumps({k: sorted(set(v)) for k, v in launched.items()}))
"""


@pytest.fixture(scope="module")
def traced_rows():
    return {k: set(v) for k, v in fresh_process.run_json(_CHILD, *[r.name for r in gw.ROWS]).items()}


@pytest.mark.parametrize("row", gw.ROWS, ids=[r.name for r in gw.ROWS])
def test_walk_row_launches_exactly_its_kernels(traced_rows, row):
    launched = traced_rows[row.name]
    assert launched == row.kernels | set(gw.HELPERS), (sorted(launched), sorted(row.kernels))


@pytest.mark.parametrize("row", gw.ROWS, ids=[r.name for r in gw.ROWS])
def test_walk_row_matches_float64(row):
    V, R = 200, 5
    msgs = make_messages(V, V, R, 1500, seed=row.d)
    check_case(msgs, V, V, R, row.d, seed=row.d, relu=True, mask=True)


# ---- the reference's own outputs ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_product_matches_reference_gcn_diag_outputs(toy, name):
    c = load_case(name)
    _, _, _, n_layers, outproj = case_shape(name)
    model = build_model(toy, name, int(c["V"]), int(c["R"]), len(c["test_graph"]))
    model.set_device(DEV)
    model.initialize_train()
    names = gd.weight_names(n_layers, outproj)
    ws = model.get_weights()
    assert len(ws) == len(names)
    with torch.no_grad():
        for i, w in enumerate(ws):
            assert tuple(w.shape) == c["w%d" % i].shape, names[i]
            w.copy_(torch.tensor(c["w%d" % i], dtype=torch.float32, device=w.device))
    masks = [torch.tensor(c["mask%d" % i], dtype=torch.uint8, device=DEV) for i in range(int(c["n_masks"]))]
    for layer, m in zip(layers_of(model), masks):
        layer.make_drop_mask = (lambda rows, mode, m=m, k=layer.dropout_keep_probability:
                                (m, k) if mode == 'train' else (None, 1.0))
    total = model.train_loss(c["graph_split"], c["X"], c["Y"])
    total.backward()
    ref_total = float(c["loss"]) + float(c["reg"])
    assert abs(total.item() - ref_total) <= 1e-4 * abs(ref_total)
    for i, (nm, w) in enumerate(zip(names, ws)):
        assert rel(w.grad.cpu().numpy(), c["g%d" % i]) < 1e-4, nm
    model.preprocess(c["test_graph"])
    model.register_for_test(c["test_graph"])
    tX = c["test_X"]
    for got, ref in ((model.score(tX), c["predict"]), (model.score_all_objects(tX), c["all_objects"]),
                     (model.score_all_subjects(tX), c["all_subjects"])):
        got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
        assert got.shape == ref.shape and np.abs(got - ref).max() < 2e-4
        live = (ref > 1e-3) & (ref < 1 - 1e-3) & (got > 0) & (got < 1)
        if live.any():
            lg, lr = np.log(got[live] / (1 - got[live])), np.log(ref[live] / (1 - ref[live]))
            assert np.abs(lg - lr).max() / max(1.0, np.abs(lr).max()) < 1e-4


def test_toy_training_with_the_diagonal_encoder(toy, tmp_path, capsys):
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(TOY_EXP.format(layers=2, concat="No").replace("Name=gcn_basis", "Name=gcn_diag"))
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--save-path", str(tmp_path / "ckpt" / "Toy")])
    text = capsys.readouterr().out
    assert "Initial loss" in text and "Validation filtered MRR" in text
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and losses[-1] < losses[0]
    layers = layers_of(model)
    assert [type(l).__name__ for l in layers] == ["DiagGcn", "DiagGcn"]
    first = layers[0]
    assert tuple(first.D_types_forward.shape) == (toy["R"], 16)
    assert float(first.b.detach().abs().max()) > 0      # the bias trains
    summ = scorer.compute_scores(np.array(toy["train"])[:20]).get_summary()
    assert 0.0 < summ.results["Filtered"]["MRR"] <= 1.0
    # checkpoint round trip: reload the saved weights into the trained model after scrambling them
    X = np.array(toy["train"], np.int32)[:20]
    before = np.asarray(model.score(X), np.float64)
    it = model.save_iter
    model.save(str(tmp_path / "rt"))
    with torch.no_grad():
        for w in model.get_weights():
            w.zero_()
    model.load(str(tmp_path / ("rt-%d.pt" % it)))
    after = np.asarray(model.score(X), np.float64)
    assert np.array_equal(before, after)
