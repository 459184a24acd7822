"""GPU: the basis layer with per-channel sigmoid coefficients (DiagonalCoefficients=Yes), ops.basis_diagcoef_layer over
rgcn_basis_diagcoef_forward / _backward, against a float64 gather restatement of the reference layer
(gcn_basis_times_diag.py), the reference-code goldens of tests/golden/make_times_diag_golden.py, and a driver run.
Tolerance 1e-4 relative (max |error| / max |reference|): fp32 kernels with non-deterministic reduction order."""
import numpy as np
import pytest
import torch

import diagcoef_walks as dw
import fresh_process
from relationprediction_b200 import _lib, ops
from relationprediction_b200 import train as driver
from relationprediction_b200.common import model_builder
from test_gpu_reference_golden import layers_of
from test_gpu_train import TOY_EXP, write_toy
from test_plugin_host import merged_settings
from test_times_diag_cpu import CASES, case_shape, load_case
import times_diag_oracle as td

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KEEP = 0.8
NAMES = ("H", "W_forward", "W_backward", "C_forward", "C_backward", "W_self", "b")


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def make_messages(V_dst, V_src, R, M, seed, dominant=None):
    """Random messages (dst < V_dst, src < V_src, weight id < 2R, positive norms); `dominant`: share of the messages
    that carry weight id 0."""
    rng = np.random.RandomState(seed)
    dst = rng.randint(0, V_dst, M)
    src = rng.randint(0, V_src, M)
    relw = rng.randint(0, 2 * R, M)
    if dominant is not None:
        relw[rng.rand(M) < dominant] = 0
    norm = rng.uniform(0.1, 1.0, M)
    return (dst.astype(np.int32), src.astype(np.int32), relw.astype(np.int32), norm.astype(np.float32))


def make_inputs(V_dst, V_src, R, B, d, seed, mask):
    g = torch.Generator().manual_seed(seed)
    std = 3 / np.sqrt(2 * d)
    w = {"H": torch.randn(V_src, d, generator=g), "W_forward": torch.randn(d, B, d, generator=g) * std,
         "W_backward": torch.randn(d, B, d, generator=g) * std, "C_forward": torch.randn(R, B, d, generator=g),
         "C_backward": torch.randn(R, B, d, generator=g), "W_self": torch.randn(d, d, generator=g) * std,
         "b": 0.1 * torch.randn(d, generator=g)}
    m = (torch.rand(V_dst, d, generator=g) < KEEP).to(torch.uint8) if mask else None
    return w, m


def reference(msgs, V_dst, R, w, mask, relu, dOut=None):
    """gcn_basis_times_diag.py restated over explicit messages, float64 on the GPU (autograd): message m reads
    P_dir[src] = H[src] V_dir with sigmoid(C_dir[r]) per channel and adds norm * sum_b into dst."""
    dst, src, relw, norm = (torch.as_tensor(a, device=DEV) for a in msgs)
    t = {k: v.to(DEV).double().requires_grad_(True) for k, v in w.items()}
    H = t["H"]
    d, B = H.shape[1], t["W_forward"].shape[1]
    back = (relw >= R)[:, None, None]
    r = (relw % R).long()
    sig = torch.sigmoid(torch.where(back, t["C_backward"][r], t["C_forward"][r]))
    Hs = H[src.long()]
    P = torch.where(back, (Hs @ t["W_backward"].reshape(d, B * d)).reshape(-1, B, d),
                    (Hs @ t["W_forward"].reshape(d, B * d)).reshape(-1, B, d))
    msg = (sig * P).sum(1) * norm.double()[:, None]
    S = H[:V_dst] @ t["W_self"]
    if mask is not None:
        S = S * mask.to(DEV).double() / KEEP
    pre = S.index_add(0, dst.long(), msg) + t["b"]
    out = torch.relu(pre) if relu else pre
    if dOut is None:
        return pre.detach(), None
    out.backward(dOut.to(DEV).double())
    return out.detach().cpu(), {k: v.grad.cpu() for k, v in t.items()}


def run_layer(graph, R, w, mask, relu, dOut):
    t = {k: v.to(DEV).float().contiguous().requires_grad_(True) for k, v in w.items()}
    out = ops.basis_diagcoef_layer(*(t[k] for k in NAMES), graph, None if mask is None else mask.to(DEV),
                                   KEEP if mask is not None else 1.0, relu)
    out.backward(dOut.to(DEV).float())
    torch.cuda.synchronize()
    return out.detach().double().cpu(), {k: v.grad.double().cpu() for k, v in t.items()}


def check_case(msgs, V_dst, V_src, R, B, d, seed, relu, mask, tol=1e-4):
    w, m = make_inputs(V_dst, V_src, R, B, d, seed, mask)
    dOut = torch.randn(V_dst, d, generator=torch.Generator().manual_seed(seed + 1), dtype=torch.float64)
    if relu:   # zeros where the pre-activation lies within rounding of the ReLU kink
        pre, _ = reference(msgs, V_dst, R, w, m, relu)
        pre = pre.cpu()
        dOut = torch.where(pre.abs() < 1e-5 * pre.abs().max(), torch.zeros_like(dOut), dOut)
    graph = ops.Graph.from_messages(*msgs, V_dst, V_src, 2 * R, device=0)
    got_out, got = run_layer(graph, R, w, m, relu, dOut)
    ref_out, ref = reference(msgs, V_dst, R, w, m, relu, dOut)
    assert rel(got_out, ref_out) < tol
    for k in NAMES:
        assert rel(got[k], ref[k]) < tol, (k, rel(got[k], ref[k]))
    return got, ref


@pytest.mark.parametrize("d", [24, 200, 500, 512])
@pytest.mark.parametrize("B", [1, 2, 5, 8])
@pytest.mark.parametrize("relu_mask", [True, False], ids=["relu-mask", "linear"])
def test_layer_matches_float64(d, B, relu_mask):
    V, R = 300, 7
    msgs = make_messages(V, V, R, 3000, seed=d * 10 + B)
    check_case(msgs, V, V, R, B, d, seed=d + B, relu=relu_mask, mask=relu_mask)


@pytest.mark.parametrize("row", dw.ROWS, ids=[r.name for r in dw.ROWS])
def test_walk_row_matches_float64(row):
    V, R = 200, 5
    msgs = make_messages(V, V, R, 1500, seed=row.B * 1000 + row.d)
    check_case(msgs, V, V, R, row.B, row.d, seed=row.d, relu=True, mask=True)


def test_split_rows(monkeypatch):
    """RGCN_ITEM_MAX=8: most rows of every view are cut into several items (pre-zeroed dP rows, reduced partials)"""
    monkeypatch.setenv("RGCN_ITEM_MAX", "8")
    V, R = 120, 4
    for B, d in ((2, 24), (5, 500), (9, 200)):
        msgs = make_messages(V, V, R, 4000, seed=B + d)
        check_case(msgs, V, V, R, B, d, seed=d, relu=True, mask=True)


def test_one_relation_carries_most_messages():
    """90 % of the messages on weight id 0: the dC walk accumulates one table row from thousands of items"""
    V, R = 2000, 6
    msgs = make_messages(V, V, R, 60000, seed=5, dominant=0.9)
    got, ref = check_case(msgs, V, V, R, 5, 200, seed=6, relu=True, mask=False)
    assert float(ref["C_forward"][0].abs().max()) > 0


def test_halo_rows():
    """V_src > V_dst: rows [V_dst, V_src) of H only send; their dH comes from the messages alone, and a halo row that
    sends nothing gets exactly zero"""
    V_dst, V_src, R = 150, 260, 4
    msgs = make_messages(V_dst, V_src, R, 2500, seed=8)
    keep = msgs[1] != V_src - 1
    msgs = tuple(a[keep] for a in msgs)
    got, _ = check_case(msgs, V_dst, V_src, R, 3, 200, seed=9, relu=True, mask=True)
    assert float(got["H"][V_src - 1].abs().max()) == 0.0


def test_graph_without_weight_id_major_views_is_rejected():
    V, R, B, d = 60, 3, 2, 16
    msgs = make_messages(V, V, R, 300, seed=10)
    w, _ = make_inputs(V, V, R, B, d, 11, False)
    t = [w[k].to(DEV).contiguous() for k in NAMES]
    _lib.set_option("graph_views", 1)
    try:
        g1 = ops.Graph.from_device_messages(*(torch.as_tensor(a, device=DEV) for a in msgs), V, V, 2 * R)
    finally:
        _lib.set_option("graph_views", 3)
    with pytest.raises(_lib.RgcnError, match="weight-id-major"):
        ops.basis_diagcoef_layer(*t, g1)
    g3 = ops.Graph.from_device_messages(*(torch.as_tensor(a, device=DEV) for a in msgs), V, V, 2 * R)
    ops.basis_diagcoef_layer(*t, g3)
    with pytest.raises(_lib.RgcnError, match="d % 4"):
        ops.basis_diagcoef_layer(torch.zeros(V, 18, device=DEV), torch.zeros(18, B, 18, device=DEV),
                                 torch.zeros(18, B, 18, device=DEV), torch.zeros(R, B, 18, device=DEV),
                                 torch.zeros(R, B, 18, device=DEV), torch.zeros(18, 18, device=DEV),
                                 torch.zeros(18, device=DEV), g3)


# ---- the dispatch ----------------------------------------------------------------------------------------------------
_CHILD = """
import json
import numpy as np
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile, record_function
import diagcoef_walks as dw
import test_gpu_times_diag as t
rows = [dw.BY_NAME[n] for n in sys.argv[1:]]
V, R = 100, 3
msgs = t.make_messages(V, V, R, 600, seed=1)
g = t.ops.Graph.from_messages(*msgs, V, V, 2 * R, device=0)
inputs = {r.name: t.make_inputs(V, V, R, r.B, r.d, 2, True) for r in rows}
dOut = {r.name: torch.randn(V, r.d, dtype=torch.float64) for r in rows}
for r in rows:
    t.run_layer(g, R, inputs[r.name][0], inputs[r.name][1], True, dOut[r.name])
with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    for r in rows:
        with record_function("diag-row:" + r.name):
            t.run_layer(g, R, inputs[r.name][0], inputs[r.name][1], True, dOut[r.name])
events = list(prof.events())
ranges = [(e.time_range.start, e.time_range.end, e.name[len("diag-row:"):]) for e in events
          if e.name.startswith("diag-row:") and e.device_type == DeviceType.CPU]
launched = {r.name: [] for r in rows}
for e in events:
    c = dw.canonical(e.name)
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
    return {k: set(v) for k, v in fresh_process.run_json(_CHILD, *[r.name for r in dw.ROWS]).items()}


@pytest.mark.parametrize("row", dw.ROWS, ids=[r.name for r in dw.ROWS])
def test_walk_row_launches_exactly_its_kernels(traced_rows, row):
    launched = traced_rows[row.name]
    assert launched == row.kernels | set(dw.HELPERS), (sorted(launched), sorted(row.kernels))


# ---- the reference's own outputs ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_product_matches_reference_times_diag_outputs(toy, name):
    c = load_case(name)
    settings_file, overrides, norm_mode, n_layers, outproj, highway = case_shape(name)
    enc, dec = merged_settings(toy, settings_file, int(c["V"]), int(c["R"]), len(c["test_graph"]))
    for s in (enc, dec):
        for k, v in overrides.items():
            s.put(k, v)
        s.put("NormalizationMode", norm_mode)
    model = model_builder.build_decoder(model_builder.build_encoder(enc, c["test_graph"]), dec)
    model.set_device(DEV)
    model.initialize_train()
    names = td.weight_names(n_layers, outproj, highway)
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


def test_toy_training_with_diagonal_coefficients(toy, tmp_path, capsys):
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(TOY_EXP.format(layers=2, concat="No").replace("DiagonalCoefficients=No",
                                                                  "DiagonalCoefficients=Yes"))
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--save-path", str(tmp_path / "ckpt" / "Toy")])
    text = capsys.readouterr().out
    assert "Initial loss" in text and "Validation filtered MRR" in text
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and losses[-1] < losses[0]
    first = layers_of(model)[0]
    assert type(first).__name__ == "BasisGcnTimesDiag" and tuple(first.C_forward.shape) == (toy["R"], 2, 16)
    assert float(first.b.detach().abs().max()) > 0      # the bias trains
    summ = scorer.compute_scores(np.array(toy["train"])[:20]).get_summary()
    assert 0.0 < summ.results["Filtered"]["MRR"] <= 1.0
