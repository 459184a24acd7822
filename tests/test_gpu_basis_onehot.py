"""GPU: the one-hot (featureless) first basis layer, ops.basis_onehot_layer over rgcn_basis_onehot_forward /
rgcn_basis_onehot_backward, against float64 restatements of the reference layer (gcn_basis.py:15-71 with
onehot_input=True), the reference-code goldens of tests/golden/make_onehot_golden.py, and a driver run.
Tolerance 1e-4 relative (max |error| / max |reference|): fp32 kernels with non-deterministic reduction order."""
import numpy as np
import pytest
import torch

from oracle import rgcn_oracle as oracle
from relationprediction_b200 import _lib, ops
from relationprediction_b200 import train as driver
from relationprediction_b200.common import model_builder
from conftest import synthetic_kg
from test_basis_onehot_cpu import CASES, load_case, split_weights
from test_gpu_reference_golden import layers_of
from test_gpu_train import TOY_EXP, write_toy
from test_plugin_host import merged_settings

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KEEP = 0.8


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def make_weights(V, R, B, d, seed):
    g = torch.Generator().manual_seed(seed)
    std = 3 / np.sqrt(V + d)
    return {"W_forward": torch.randn(V, B, d, generator=g) * std, "W_backward": torch.randn(V, B, d, generator=g) * std,
            "C_forward": torch.randn(R, B, generator=g), "C_backward": torch.randn(R, B, generator=g),
            "W_self": torch.randn(V, d, generator=g) * std}


def run_layer(tr, V, R, w, mask, relu, dOut):
    """The product layer on the GPU: returns out and the five weight gradients as float64 CPU tensors."""
    graph = ops.Graph(tr, V, R, device=0)
    leaves = {k: v.to(DEV).float().contiguous().requires_grad_(True) for k, v in w.items()}
    m = None if mask is None else mask.to(DEV)
    out = ops.basis_onehot_layer(leaves["W_forward"], leaves["W_backward"], leaves["C_forward"], leaves["C_backward"],
                                 leaves["W_self"], graph, m, KEEP if mask is not None else 1.0, relu)
    out.backward(dOut.to(DEV).float())
    torch.cuda.synchronize()
    return out.detach().double().cpu(), {k: v.grad.double().cpu() for k, v in leaves.items()}


def oracle_layer(tr, V, w, mask, relu, dOut):
    """oracle.basis_gcn_forward with H = I_V (the matmul with a one-hot row is the lookup), float64, autograd."""
    nf, nb = oracle.graph_norms(tr, V, "canonical", np.float32)
    weights = dict(w, b=None)
    out, grads = oracle.layer_fwd_bwd("basis", torch.eye(V, dtype=torch.float64), tr, weights, nf, nb, dOut,
                                      mask, KEEP if mask is not None else 1.0, relu, torch.float64)
    return out, grads


def gather_reference(tr, V, R, w, mask, relu, dOut):
    """The same layer restated with row gathers instead of I_V (for graphs too large for a [V, V] input), float64 on
    the GPU: forward messages read W_forward[s] with C_forward[r] into o, backward ones W_backward[o] with
    C_backward[r] into s (gcn_basis.py:39-46, :73-79)."""
    nf, nb = oracle.graph_norms(tr, V, "canonical", np.float32)
    t = {k: v.to(DEV).double().requires_grad_(True) for k, v in w.items()}
    s, r, o = (torch.as_tensor(tr[:, i].astype(np.int64), device=DEV) for i in range(3))
    mf = (t["C_forward"][r].unsqueeze(-1) * t["W_forward"][s]).sum(1)
    mb = (t["C_backward"][r].unsqueeze(-1) * t["W_backward"][o]).sum(1)
    sl = t["W_self"] if mask is None else t["W_self"] * mask.to(DEV).double() / KEEP
    out = sl.index_add(0, o, mf * torch.as_tensor(nf, device=DEV).double()[:, None])
    out = out.index_add(0, s, mb * torch.as_tensor(nb, device=DEV).double()[:, None])
    if relu:
        out = torch.relu(out)
    out.backward(dOut.to(DEV).double())
    return out.detach().cpu(), {k: v.grad.cpu() for k, v in t.items()}


def off_kink(pre, dOut):
    """dOut with zeros where the pre-activation lies within rounding of the ReLU kink: there fp32 and float64 may
    legitimately disagree on relu', which would change G (and every gradient it feeds) by a full dOut entry."""
    return torch.where(pre.abs() < 1e-5 * pre.abs().max(), torch.zeros_like(dOut), dOut)


def check(got, ref, tol=1e-4):
    out, grads = got
    rout, rgrads = ref
    assert rel(out.numpy(), rout.numpy()) < tol, "out"
    for k in ("W_forward", "W_backward", "C_forward", "C_backward", "W_self"):
        assert rel(grads[k].numpy(), rgrads[k].numpy()) < tol, k


@pytest.mark.parametrize("d", [24, 200, 500, 512])
@pytest.mark.parametrize("B", [1, 2, 5, 8])
@pytest.mark.parametrize("relu,masked", [(True, True), (False, False)])
def test_layer_matches_float64_oracle(d, B, relu, masked):
    V, R = 300, 7
    tr = synthetic_kg(V, R, 3000, seed=d * 10 + B, skewed=True)
    w = make_weights(V, R, B, d, seed=d + B)
    g = torch.Generator().manual_seed(1)
    mask = (torch.rand(V, d, generator=g) < KEEP).to(torch.uint8) if masked else None
    dOut = torch.randn(V, d, generator=g, dtype=torch.float64)
    if relu:
        dOut = off_kink(oracle_layer(tr, V, w, mask, False, dOut)[0], dOut)
    check(run_layer(tr, V, R, w, mask, relu, dOut), oracle_layer(tr, V, w, mask, relu, dOut))


def test_split_rows(monkeypatch):
    """Rows of more than item_max messages are cut into several work items (RGCN_ITEM_MAX=8 forces it for most
    rows): the forward pushes per item, the backward combines the partial dW rows in pre-zeroed rows."""
    monkeypatch.setenv("RGCN_ITEM_MAX", "8")
    V, R, B, d = 200, 5, 5, 200
    tr = synthetic_kg(V, R, 4000, seed=3, skewed=True)
    w = make_weights(V, R, B, d, seed=4)
    g = torch.Generator().manual_seed(2)
    mask = (torch.rand(V, d, generator=g) < KEEP).to(torch.uint8)
    dOut = off_kink(oracle_layer(tr, V, w, mask, False, torch.zeros(V, d, dtype=torch.float64))[0],
                    torch.randn(V, d, generator=g, dtype=torch.float64))
    graph = ops.Graph(tr, V, R, device=0)
    assert graph.info()[12] == 8 and graph.info()[8] > 0      # item_max, split source rows
    check(run_layer(tr, V, R, w, mask, True, dOut), oracle_layer(tr, V, w, mask, True, dOut))


def test_rows_without_messages_are_exact():
    """A source with no message in a direction gets an exactly zero dW row in that direction (the gradient is
    dense); a node with no incoming message gets out = act(masked W_self) exactly."""
    V, R, B, d = 64, 3, 5, 200
    rng = np.random.RandomState(5)
    core = np.stack([rng.randint(0, 40, 600), rng.randint(0, R, 600), rng.randint(0, 40, 600)], 1)
    senders = np.stack([np.arange(40, 48), rng.randint(0, R, 8), rng.randint(0, 40, 8)], 1)  # subjects only
    tr = np.concatenate([core, senders]).astype(np.int32)                                     # 48..63 isolated
    w = make_weights(V, R, B, d, seed=6)
    g = torch.Generator().manual_seed(3)
    mask = (torch.rand(V, d, generator=g) < KEEP).to(torch.uint8)
    dOut = off_kink(oracle_layer(tr, V, w, mask, False, torch.zeros(V, d, dtype=torch.float64))[0],
                    torch.randn(V, d, generator=g, dtype=torch.float64))
    # poison the gradient buffers' previous contents: every row must be written
    torch.empty(4 * V * B * d, device=DEV).fill_(float("nan"))
    out, grads = run_layer(tr, V, R, w, mask, True, dOut)
    check((out, grads), oracle_layer(tr, V, w, mask, True, dOut))
    assert (grads["W_backward"][40:] == 0).all() and (grads["W_forward"][48:] == 0).all()
    assert (grads["W_forward"][40:48].abs().amax(dim=(1, 2)) > 0).all()
    Ws = w["W_self"].float()
    expect = torch.relu(torch.where(mask.bool(), Ws * torch.tensor(1.0 / KEEP, dtype=torch.float32), 0.0))
    assert torch.equal(out[48:].float(), expect[48:])


def test_sampled_train_step_graph_over_fb15k237_entities():
    """A 15 000-triple graph over V = 14 541 entities (the FB15k-237 train-step shape, d = 500, B = 5)."""
    V, R, B, d = 14541, 237, 5, 500
    tr = synthetic_kg(V, R, 15000, seed=11, skewed=True)
    w = make_weights(V, R, B, d, seed=12)
    g = torch.Generator().manual_seed(4)
    mask = (torch.rand(V, d, generator=g) < KEEP).to(torch.uint8)
    dOut = torch.randn(V, d, generator=g, dtype=torch.float64)
    dOut = off_kink(gather_reference(tr, V, R, w, mask, False, dOut)[0], dOut)
    check(run_layer(tr, V, R, w, mask, True, dOut), gather_reference(tr, V, R, w, mask, True, dOut))
    # the gather restatement is the oracle's layer (checked on a graph small enough for H = I_V)
    Vs = 150
    trs = synthetic_kg(Vs, 9, 1200, seed=13, skewed=True)
    ws = make_weights(Vs, 9, 3, 24, seed=14)
    dO = torch.randn(Vs, 24, dtype=torch.float64)
    check(gather_reference(trs, Vs, 9, ws, None, True, dO), oracle_layer(trs, Vs, ws, None, True, dO), tol=1e-12)


@pytest.mark.parametrize("name", sorted(CASES))
def test_product_matches_reference_onehot_outputs(toy, name):
    c = load_case(name)
    overrides, norm_mode = CASES[name]
    enc, dec = merged_settings(toy, "gcn_basis.exp", int(c["V"]), int(c["R"]), len(c["test_graph"]))
    for s in (enc, dec):
        for k, v in overrides.items():
            s.put(k, v)
        s.put("UseInputTransform", "No")
        s.put("NormalizationMode", norm_mode)
    model = model_builder.build_decoder(model_builder.build_encoder(enc, c["test_graph"]), dec)
    model.set_device(DEV)
    model.initialize_train()
    names, _, _ = split_weights(c)
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
        if bool(c["g%d_unused" % i]):
            assert w.grad is None or float(w.grad.abs().max()) == 0.0, nm
            continue
        assert rel(w.grad.cpu().numpy(), c["g%d" % i]) < 1e-4, nm
    model.preprocess(c["test_graph"])
    model.register_for_test(c["test_graph"])
    tX = c["test_X"]
    # scores compared on the logit scale where the sigmoid is not saturated, as in test_gpu_reference_golden.py
    for got, ref in ((model.score(tX), c["predict"]), (model.score_all_objects(tX), c["all_objects"]),
                     (model.score_all_subjects(tX), c["all_subjects"])):
        got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
        assert got.shape == ref.shape and np.abs(got - ref).max() < 2e-4
        live = (ref > 1e-3) & (ref < 1 - 1e-3) & (got > 0) & (got < 1)
        if live.any():
            lg, lr = np.log(got[live] / (1 - got[live])), np.log(ref[live] / (1 - ref[live]))
            assert np.abs(lg - lr).max() / max(1.0, np.abs(lr).max()) < 1e-4


def test_rejects_bad_shapes_and_graphs_without_csr_views():
    V, R, B, d = 50, 3, 2, 16
    tr = synthetic_kg(V, R, 200, seed=15)
    graph = ops.Graph(tr, V, R, device=0)
    w = {k: v.to(DEV).contiguous() for k, v in make_weights(V, R, B, d, seed=16).items()}
    args = [w["W_forward"], w["W_backward"], w["C_forward"], w["C_backward"], w["W_self"]]
    ops.basis_onehot_layer(*args, graph)
    for i, bad in [(0, torch.zeros(V - 1, B, d, device=DEV)), (1, torch.zeros(V, B + 1, d, device=DEV)),
                   (2, torch.zeros(R + 1, B, device=DEV)), (3, torch.zeros(R, B + 1, device=DEV)),
                   (4, torch.zeros(V, d + 4, device=DEV)), (4, w["W_self"].double())]:
        a = list(args)
        a[i] = bad
        with pytest.raises(_lib.RgcnError):
            ops.basis_onehot_layer(*a, graph)
    a = [torch.zeros(V, B, 18, device=DEV), torch.zeros(V, B, 18, device=DEV), args[2], args[3],
         torch.zeros(V, 18, device=DEV)]
    with pytest.raises(_lib.RgcnError, match="d % 4"):
        ops.basis_onehot_layer(*a, graph)
    with pytest.raises(_lib.RgcnError, match="drop_mask"):
        ops.basis_onehot_layer(*args, graph, drop_mask=torch.ones(V, d, device=DEV))
    _lib.set_option("graph_views", 2)
    try:
        g2 = ops.Graph.from_device_triples(torch.as_tensor(tr, device=DEV), V, R)
    finally:
        _lib.set_option("graph_views", 3)
    with pytest.raises(_lib.RgcnError, match="CSR"):
        ops.basis_onehot_layer(*args, g2)


def test_toy_training_with_featureless_encoder(toy, tmp_path, capsys):
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(TOY_EXP.format(layers=2, concat="No").replace("UseInputTransform=Yes", "UseInputTransform=No"))
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--save-path", str(tmp_path / "ckpt" / "Toy")])
    text = capsys.readouterr().out
    assert "Initial loss" in text and "Validation filtered MRR" in text
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and losses[-1] < losses[0]
    first = layers_of(model)[0]
    assert first.onehot_input and tuple(first.W_forward.shape) == (toy["V"], 2, 16)
    summ = scorer.compute_scores(np.array(toy["train"])[:20]).get_summary()
    assert 0.0 < summ.results["Filtered"]["MRR"] <= 1.0
