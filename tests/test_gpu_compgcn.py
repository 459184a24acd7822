"""GPU: the CompGCN layer (Encoder Name=compgcn), ops.compgcn_layer over rgcn_compgcn_forward / _backward, against the
float64 restatement of tests/compgcn_oracle.py: every output and gradient across widths, compositions, ReLU and mask,
graph shapes (rows without messages, split rows, a dominant relation, halo rows, per-relation norms), the view
rejection, the kernels each walk row launches, a 2-layer encoder training step under DistMult and ComplEx, a driver run
on FB-Toutanova data with a checkpoint round trip, and the predict command with relation metrics.  Tolerance 1e-4
relative (max |error| / max |reference|): fp32 kernels with non-deterministic reduction order."""
import os

import numpy as np
import pytest
import torch

import compgcn_oracle as cg
import compgcn_walks as cw
import complex_oracle
import fresh_process
import relation_norm_oracle
from oracle import rgcn_oracle as oracle
from relationprediction_b200 import _lib, ops
from relationprediction_b200 import predict as predict_cmd
from relationprediction_b200 import train as driver
from relationprediction_b200.common import model_builder
from relationprediction_b200.encoders.message_gcns.compgcn import CompGcn
from test_compgcn_cpu import compgcn_settings
from test_gpu_train import TOY_EXP
from test_highway_cpu import chain_of

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KEEP = 0.8
NAMES = ("H", "Z", "z_loop", "W_cat", "W_rel", "b")
DATASETS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "datasets")


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


def make_inputs(V_dst, V_src, R, d_in, d_out, seed, mask):
    g = torch.Generator().manual_seed(seed)
    w = {"H": torch.randn(V_src, d_in, generator=g), "Z": torch.randn(2 * R, d_in, generator=g),
         "z_loop": torch.randn(d_in, generator=g), "W_cat": torch.randn(3 * d_in, d_out, generator=g) / np.sqrt(d_in),
         "W_rel": torch.randn(d_in, d_out, generator=g) / np.sqrt(d_in), "b": 0.1 * torch.randn(d_out, generator=g)}
    m = (torch.rand(V_dst, 2 * d_in, generator=g) < KEEP).to(torch.uint8) if mask else None
    return w, m


def reference(msgs, V_dst, w, composition, mask, relu, dOut=None, dZn=None):
    t = {k: v.to(DEV).double().requires_grad_(True) for k, v in w.items()}
    dst, src, relw, norm = (torch.as_tensor(a, device=DEV).long() if i < 3 else torch.as_tensor(a, device=DEV)
                            for i, a in enumerate(msgs))
    R = w["Z"].shape[0] // 2
    d = w["H"].shape[1]
    msg = norm.double()[:, None] * cg.phi(t["H"][src], t["Z"][relw], composition)
    fwd = relw < R
    A = torch.cat([torch.zeros(V_dst, d, dtype=torch.float64, device=DEV).index_add(0, dst[fwd], msg[fwd]),
                   torch.zeros(V_dst, d, dtype=torch.float64, device=DEV).index_add(0, dst[~fwd], msg[~fwd])], 1)
    if mask is not None:
        A = A * mask.to(DEV).double() / KEEP
    Cat = torch.cat([A, cg.phi(t["H"][:V_dst], t["z_loop"], composition)], 1) / 3
    pre = Cat @ t["W_cat"] + t["b"]
    out = torch.relu(pre) if relu else pre
    Zn = t["Z"] @ t["W_rel"]
    if dOut is None:
        return pre.detach().cpu(), None, None
    torch.autograd.backward([out, Zn], [dOut.to(DEV).double(), dZn.to(DEV).double()])
    return out.detach().cpu(), Zn.detach().cpu(), {k: v.grad.cpu() for k, v in t.items()}


def run_layer(graph, w, composition, mask, relu, dOut, dZn):
    t = {k: v.to(DEV).float().contiguous().requires_grad_(True) for k, v in w.items()}
    out, Zn = ops.compgcn_layer(*(t[k] for k in NAMES), graph, composition, None if mask is None else mask.to(DEV),
                                KEEP if mask is not None else 1.0, relu)
    torch.autograd.backward([out, Zn], [dOut.to(DEV).float(), dZn.to(DEV).float()])
    torch.cuda.synchronize()
    return out.detach().double().cpu(), Zn.detach().double().cpu(), {k: v.grad.double().cpu() for k, v in t.items()}


def check_case(msgs, V_dst, V_src, R, d_in, d_out, composition, seed, relu, mask, graph=None, tol=1e-4):
    w, m = make_inputs(V_dst, V_src, R, d_in, d_out, seed, mask)
    gen = torch.Generator().manual_seed(seed + 1)
    dOut = torch.randn(V_dst, d_out, generator=gen, dtype=torch.float64)
    dZn = torch.randn(2 * R, d_out, generator=gen, dtype=torch.float64)
    if relu:   # zeros where the pre-activation lies within rounding of the ReLU kink
        pre, _, _ = reference(msgs, V_dst, w, composition, m, relu)
        dOut = torch.where(pre.abs() < 1e-5 * pre.abs().max(), torch.zeros_like(dOut), dOut)
    if graph is None:
        graph = ops.Graph.from_messages(*msgs, V_dst, V_src, 2 * R, device=0)
    got_out, got_Zn, got = run_layer(graph, w, composition, m, relu, dOut, dZn)
    ref_out, ref_Zn, ref = reference(msgs, V_dst, w, composition, m, relu, dOut, dZn)
    assert rel(got_out, ref_out) < tol
    assert rel(got_Zn, ref_Zn) < tol
    for k in NAMES:
        assert rel(got[k], ref[k]) < tol, (k, rel(got[k], ref[k]))
    return got_out, got, ref


D_OUT = {4: 8, 24: 24, 200: 12, 500: 500, 512: 256, 516: 200}


@pytest.mark.parametrize("d", sorted(D_OUT))
@pytest.mark.parametrize("composition", ["mult", "sub"])
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "linear"])
@pytest.mark.parametrize("mask", [True, False], ids=["mask", "nomask"])
def test_layer_matches_float64(d, composition, relu, mask):
    V, R = 300, 7
    msgs = make_messages(V, V, R, 3000, seed=d * 10 + relu * 2 + mask)
    check_case(msgs, V, V, R, d, D_OUT[d], composition, seed=d + relu, relu=relu, mask=mask)


@pytest.mark.parametrize("composition", ["mult", "sub"])
def test_rows_without_messages_get_zero_message_slabs(composition):
    """destination rows 0..9 receive no message: with W_cat's loop block and b zero their output is exactly zero"""
    V, R, d = 200, 4, 200
    msgs = make_messages(V, V, R, 2000, seed=3, empty_dst=range(10))
    w, _ = make_inputs(V, V, R, d, d, 4, False)
    w["W_cat"][2 * d:] = 0
    w["b"].zero_()
    g = ops.Graph.from_messages(*msgs, V, V, 2 * R, device=0)
    out, _, _ = run_layer(g, w, composition, None, False, torch.zeros(V, d, dtype=torch.float64),
                          torch.zeros(2 * R, d, dtype=torch.float64))
    assert float(out[:10].abs().max()) == 0.0 and float(out[10:].abs().max()) > 0
    check_case(msgs, V, V, R, d, 24, composition, seed=5, relu=True, mask=True)


@pytest.mark.parametrize("composition", ["mult", "sub"])
def test_split_rows_on_both_views(monkeypatch, composition):
    """RGCN_ITEM_MAX=8: most rows of both CSR views are cut into several items (vector reductions into zeroed Cat rows
    forward, into zeroed dH rows backward; the loop slab and loop gradient once per row)"""
    monkeypatch.setenv("RGCN_ITEM_MAX", "8")
    V, R = 120, 4
    for d in (24, 500, 516):
        msgs = make_messages(V, V, R, 4000, seed=d)
        check_case(msgs, V, V, R, d, 20, composition, seed=d, relu=True, mask=True)


@pytest.mark.parametrize("composition", ["mult", "sub"])
def test_one_relation_carries_most_messages(composition):
    """90 % of the messages on weight id 0: thousands of runs reduce into one dZ row"""
    V, R = 2000, 6
    msgs = make_messages(V, V, R, 60000, seed=5, dominant=0.9)
    _, _, ref = check_case(msgs, V, V, R, 200, 200, composition, seed=6, relu=True, mask=False)
    assert float(ref["Z"][0].abs().max()) > 0


@pytest.mark.parametrize("composition", ["mult", "sub"])
def test_halo_rows(composition):
    """V_src > V_dst: rows [V_dst, V_src) of H only send, with no loop term; a halo row that sends nothing gets
    exactly zero gradient"""
    V_dst, V_src, R = 150, 260, 4
    msgs = make_messages(V_dst, V_src, R, 2500, seed=8)
    keep = msgs[1] != V_src - 1
    msgs = tuple(a[keep] for a in msgs)
    _, got, _ = check_case(msgs, V_dst, V_src, R, 200, 100, composition, seed=9, relu=True, mask=True)
    assert float(got["H"][V_src - 1].abs().max()) == 0.0


@pytest.mark.parametrize("composition", ["mult", "sub"])
def test_relation_normalised_graph(composition):
    """NormalizationMode=relation: the layer reads the graph's per-message norms, whatever they are"""
    rng = np.random.default_rng(11)
    V, R, E = 300, 5, 2500
    tri = np.stack([rng.integers(0, V, E), rng.integers(0, R, E), rng.integers(0, V, E)], 1).astype(np.int32)
    g = ops.Graph(tri, V, R, norm_mode="relation", device=0)
    nf, nb = relation_norm_oracle.relation_norms(tri, np.float64)
    msgs = cg.triple_messages(tri, R, nf, nb)
    check_case(msgs, V, V, R, 200, 200, composition, seed=12, relu=True, mask=True, graph=g)


def test_views_and_widths_are_checked():
    V, R, d = 60, 3, 16
    msgs = make_messages(V, V, R, 300, seed=10)
    w, _ = make_inputs(V, V, R, d, d, 11, False)
    t = [w[k].to(DEV).contiguous() for k in NAMES]
    _lib.set_option("graph_views", 2)
    try:
        g2 = ops.Graph.from_device_messages(*(torch.as_tensor(a, device=DEV) for a in msgs), V, V, 2 * R)
    finally:
        _lib.set_option("graph_views", 3)
    with pytest.raises(_lib.RgcnError, match="CSR"):
        ops.compgcn_layer(*t, g2)
    g3 = ops.Graph.from_device_messages(*(torch.as_tensor(a, device=DEV) for a in msgs), V, V, 2 * R)
    ops.compgcn_layer(*t, g3)
    with pytest.raises(_lib.RgcnError, match="d % 4"):
        ops.compgcn_layer(torch.zeros(V, 18, device=DEV), torch.zeros(2 * R, 18, device=DEV), torch.zeros(18, device=DEV),
                          torch.zeros(54, 16, device=DEV), torch.zeros(18, 16, device=DEV), torch.zeros(16, device=DEV),
                          g3)
    with pytest.raises(_lib.RgcnError, match="d_out % 4"):
        ops.compgcn_layer(t[0], t[1], t[2], torch.zeros(3 * d, 10, device=DEV), torch.zeros(d, 10, device=DEV),
                          torch.zeros(10, device=DEV), g3)


# ---- the dispatch ----------------------------------------------------------------------------------------------------
_CHILD = """
import json
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile, record_function
import compgcn_walks as cw
import test_gpu_compgcn as t
rows = [cw.BY_NAME[n] for n in sys.argv[1:]]
V, R = 100, 3
msgs = t.make_messages(V, V, R, 600, seed=1)
g = t.ops.Graph.from_messages(*msgs, V, V, 2 * R, device=0)
inputs = {r.name: t.make_inputs(V, V, R, r.d, 16, 2, True) for r in rows}
grads = {r.name: (torch.randn(V, 16, dtype=torch.float64), torch.randn(2 * R, 16, dtype=torch.float64)) for r in rows}
def run(r):
    t.run_layer(g, inputs[r.name][0], r.composition, inputs[r.name][1], True, *grads[r.name])
for r in rows:
    run(r)
with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    for r in rows:
        with record_function("compgcn-row:" + r.name):
            run(r)
events = list(prof.events())
ranges = [(e.time_range.start, e.time_range.end, e.name[len("compgcn-row:"):]) for e in events
          if e.name.startswith("compgcn-row:") and e.device_type == DeviceType.CPU]
launched = {r.name: [] for r in rows}
for e in events:
    c = cw.canonical(e.name)
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
    return {k: set(v) for k, v in fresh_process.run_json(_CHILD, *[r.name for r in cw.ROWS]).items()}


@pytest.mark.parametrize("row", cw.ROWS, ids=[r.name for r in cw.ROWS])
def test_walk_row_launches_exactly_its_kernels(traced_rows, row):
    assert traced_rows[row.name] == row.kernels, (sorted(traced_rows[row.name]), sorted(row.kernels))


@pytest.mark.parametrize("row", cw.ROWS, ids=[r.name for r in cw.ROWS])
def test_walk_row_matches_float64(row):
    V, R = 200, 5
    msgs = make_messages(V, V, R, 1500, seed=row.d)
    check_case(msgs, V, V, R, row.d, 16, row.composition, seed=row.d, relu=True, mask=True)


# ---- the encoder -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("composition", ["mult", "sub"])
@pytest.mark.parametrize("decoder", ["bilinear-diag", "complex"])
def test_two_layer_training_step_matches_the_oracle(toy, decoder, composition):
    train = np.asarray(toy["train"], np.int32)
    V, R = int(toy["V"]), int(toy["R"])
    enc, dec = compgcn_settings(toy, decoder=decoder, d="24", code="16", Composition=composition)
    model = model_builder.build_decoder(model_builder.build_encoder(enc, train), dec)
    model.set_device(DEV)
    np.random.seed(3)
    model.initialize_train()
    layers = [c for c in chain_of(model) if isinstance(c, CompGcn)][::-1]
    rng = np.random.default_rng(4)
    masks = []
    for layer in layers:
        m = torch.as_tensor(rng.random((V, 2 * layer.shape[0])) < KEEP).to(torch.uint8)
        masks.append(m)
        layer.make_drop_mask = (lambda rows, mode, m=m.to(DEV): (m, KEEP) if mode == 'train' else (None, 1.0))
    X = np.stack([rng.integers(0, V, 40), rng.integers(0, R, 40), rng.integers(0, V, 40)], 1).astype(np.int32)
    Y = (rng.random(40) < 0.3).astype(np.float32)
    graph = train[:30]
    total = model.train_loss(graph, X, Y)
    total.backward()
    names = cg.weight_names(2)
    ws = model.get_weights()[:len(names)]
    leaves = {nm: w.detach().cpu().double().requires_grad_(True) for nm, w in zip(names, ws)}
    nf, nb = oracle.graph_norms(graph, V, "canonical", np.float64)
    codes, relt = cg.encode(leaves, 2, graph, V, R, "train", masks, KEEP, nf, nb, composition)
    if decoder == "bilinear-diag":
        L, reg, _ = oracle.distmult_loss(codes, relt, X, Y, torch.float64)
    else:
        L, reg, _ = complex_oracle.complex_loss(codes, relt, X, Y, torch.float64)
    ref = L + float(dec["RegularizationParameter"]) * reg
    ref.backward()
    assert abs(total.item() - ref.item()) <= 1e-4 * abs(ref.item())
    for nm, w in zip(names, ws):
        if nm == "b_in":
            assert w.grad is None
            continue
        assert rel(w.grad.cpu(), leaves[nm].grad) < 1e-4, nm


def _toutanova(tmp_path):
    """FB-Toutanova's entity and relation names (numbered densely: the sample keeps the full dataset's ids) and a
    training prefix, with validation and test split off it"""
    base = os.path.join(DATASETS, "FB-Toutanova")
    for f in ("entities.dict", "relations.dict"):
        with open(os.path.join(base, f)) as fh:
            names = [l.split("\t")[1] for l in fh.read().splitlines() if l]
        (tmp_path / f).write_text("".join("%d\t%s\n" % kv for kv in enumerate(names)))
    with open(os.path.join(base, "train.txt")) as fh:
        lines = fh.read().splitlines()
    (tmp_path / "train.txt").write_text("\n".join(lines[:500]) + "\n")
    (tmp_path / "valid.txt").write_text("\n".join(lines[500:550]) + "\n")
    (tmp_path / "test.txt").write_text("\n".join(lines[550:]) + "\n")
    exp = tmp_path / "fb.exp"
    exp.write_text(TOY_EXP.format(layers=2, concat="No").replace("Name=gcn_basis", "Name=compgcn\n\tComposition=mult"))
    return exp


def test_driver_on_toutanova_data_with_a_checkpoint_round_trip(tmp_path, capsys):
    exp = _toutanova(tmp_path)
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--save-path", str(tmp_path / "ckpt" / "FB")])
    text = capsys.readouterr().out
    assert "Initial loss" in text and "Validation filtered MRR" in text
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and all(np.isfinite(losses)) and losses[-1] < losses[0]
    layers = [c for c in chain_of(model) if isinstance(c, CompGcn)]
    assert len(layers) == 2 and layers[-1].Z.shape[0] == 2 * model.relation_count
    X = np.array([[0, 0, 1], [2, 1, 3], [4, 2, 5]], np.int32)
    before = np.asarray(model.score(X), np.float64)
    it = model.save_iter
    model.save(str(tmp_path / "rt"))
    with torch.no_grad():
        for w in model.get_weights():
            w.zero_()
    model.load(str(tmp_path / ("rt-%d.pt" % it)))
    assert np.array_equal(before, np.asarray(model.score(X), np.float64))


def test_predict_top_k_and_relation_metrics_with_a_compgcn_checkpoint(tmp_path, capsys):
    exp = _toutanova(tmp_path)
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "40",
                                 "--no-save", "--no-early-stopping", "--final-eval", "0", "--relation-metrics"])
    out = capsys.readouterr().out
    assert "Relation prediction:" in out
    R = int(model.relation_count)
    test = [l.split("\t") for l in (tmp_path / "test.txt").read_text().splitlines()][:6]
    model.save(str(tmp_path / "FB"))
    ckpt = sorted(tmp_path.glob("FB-*.pt"))[-1]
    lines = []
    for s_, r_, o_ in test:
        lines += ["%s\t?\t%s" % (s_, o_), "%s\t%s\t?" % (s_, r_)]
    (tmp_path / "queries.tsv").write_text("\n".join(lines) + "\n")
    answers = tmp_path / "answers.tsv"
    k = min(5, R)
    predict_cmd.main(["--settings", str(exp), "--dataset", str(tmp_path), "--checkpoint", str(ckpt),
                      "--queries", str(tmp_path / "queries.tsv"), "--k", str(k), "--out", str(answers)])
    rows = [l.split("\t") for l in answers.read_text().splitlines()]
    assert {int(r[0]) for r in rows} == set(range(len(lines)))
    for q in range(len(lines)):
        got = [r for r in rows if int(r[0]) == q]
        assert [int(r[1]) for r in got] == list(range(1, len(got) + 1)) and 0 < len(got) <= k
        scores = [float(r[3]) for r in got]
        assert scores == sorted(scores, reverse=True) and all(0.0 <= s <= 1.0 for s in scores)
