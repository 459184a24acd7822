"""GPU: the per-relation normaliser (RGCN_NORM_RELATION) on the device.

  * device preparation (graph_device.cu: the run lengths of the first destination-keyed sort, k_norm_relation) equals
    the host builder bit for bit, for every graph_views value, on Toy, a 15 k-triple graph, a skewed 1 M-edge graph
    where one relation carries most messages, and small work items / supertiles;
  * the build launches the canonical build's kernels with k_norm_relation in place of k_norm_canonical: no sort added;
  * block (s = 5, 8) and basis layers over relation-mode graphs match the float64 oracle forward and backward;
  * the product path (every layer type: block, basis, one-hot basis, DiagonalCoefficients, gcn_diag, highway, and the
    ComplEx decoder) matches the goldens of the reference's own 'local' code at 1e-4;
  * a Toy driver run with NormalizationMode=relation trains, evaluates and round-trips a checkpoint."""
import numpy as np
import pytest
import torch

import relation_norm_oracle as ron
import test_relation_norm_cpu as rn
from conftest import synthetic_kg
from oracle import rgcn_oracle as oracle
from relationprediction_b200 import _lib, ops
from relationprediction_b200 import train as driver
from test_gpu_reference_golden import layers_of, rel
from test_gpu_train import TOY_EXP, write_toy
from test_plugin_host import merged_settings

pytestmark = pytest.mark.gpu

CSR_EXPORTS = [_lib.X_DST_ROWPTR, _lib.X_DST_SRC, _lib.X_DST_RELW, _lib.X_DST_NORM, _lib.X_DST_MID,
               _lib.X_SRC_ROWPTR, _lib.X_SRC_DST, _lib.X_SRC_RELW, _lib.X_SRC_NORM, _lib.X_SRC_MID]
REL_EXPORTS = [_lib.X_REL_PTR, _lib.X_REL_DST, _lib.X_REL_SRC, _lib.X_REL_NORM, _lib.X_REL_MID,
               _lib.X_REL2_PTR, _lib.X_REL2_SRC, _lib.X_REL2_DST, _lib.X_REL2_NORM, _lib.X_REL2_MID]


@pytest.fixture
def graph_views():
    def set_views(v):
        _lib.set_option("graph_views", v)
    yield set_views
    _lib.set_option("graph_views", 3)


def one_relation_heavy(V, R, E, seed):
    """Skewed 1 M-edge style graph: ~90 % of the triples use relation 0, hub-heavy endpoints."""
    tr = synthetic_kg(V, R, E, seed=seed, skewed=True)
    rng = np.random.RandomState(seed)
    tr[rng.rand(E) < 0.9, 1] = 0
    return tr


def check_views(tr, V, R, views):
    gh = ops.Graph(tr, V, R, norm_mode="relation")
    gd = ops.Graph(tr, V, R, norm_mode="relation", device=0)
    dg = ops.Graph.from_device_triples(torch.from_numpy(tr).cuda(), V, R, norm_mode="relation")
    ih = gh.info()
    keys = [0, 1, 2, 3, 12, 13] + ([4, 5, 7, 8, 9] if views & 1 else []) + ([6, 14, 15] if views & 2 else [])
    exports = [_lib.X_MSG_NORM] + (CSR_EXPORTS if views & 1 else []) + (REL_EXPORTS if views & 2 else [])
    for g in (gd, dg):
        info = g.info()
        for k in keys:
            assert info[k] == ih[k], (k, info, ih)
        for which in exports:
            assert g.export(which).tobytes() == gh.export(which).tobytes(), (views, which)


CASES = {"toy": None, "15k": (14541, 237, 15000, False), "skewed_1M": (200000, 500, 1000000, True)}


@pytest.mark.parametrize("views", [1, 2, 3])
@pytest.mark.parametrize("case", sorted(CASES))
def test_device_prep_equals_host_prep(graph_views, toy, case, views):
    graph_views(views)
    if case == "toy":
        tr, V, R = np.array(toy["train"], np.int32), 16, 9
    elif CASES[case][3]:
        V, R, E, _ = CASES[case]
        tr = one_relation_heavy(V, R, E, seed=7)
    else:
        V, R, E, _ = CASES[case]
        tr = synthetic_kg(V, R, E, seed=6)
    check_views(tr, V, R, views)


@pytest.mark.parametrize("views", [1, 2, 3])
def test_device_prep_small_items_and_supertiles(graph_views, monkeypatch, views):
    monkeypatch.setenv("RGCN_ITEM_MAX", "8")
    monkeypatch.setenv("RGCN_SUPERTILE_ROWS", "100")
    graph_views(views)
    check_views(one_relation_heavy(1500, 11, 20000, seed=4), 1500, 11, views)
    dup = synthetic_kg(300, 3, 4000, seed=8, skewed=True)
    check_views(np.concatenate([dup, dup[:500]]), 300, 3, views)       # duplicate triples


@pytest.mark.parametrize("views", [1, 2, 3])
def test_relation_build_adds_only_the_norm_kernel(graph_views, views):
    """Same kernels as the canonical build, with k_norm_relation (launched inside the first view build) in place of
    k_norm_canonical: no sort or other pass was added."""
    graph_views(views)
    tr = synthetic_kg(5000, 40, 60000, seed=2, skewed=True)
    t = torch.from_numpy(tr).cuda()
    counts = {}
    for mode in ("canonical", "relation", "canonical", "relation"):      # second round: warmed up
        torch.cuda.synchronize()
        before = _lib.launch_count()
        ops.Graph.from_device_triples(t, 5000, 40, norm_mode=mode)
        counts[mode] = _lib.launch_count() - before
    new_norm_kernels, replaced_norm_kernels = 1, 1
    assert counts["relation"] - counts["canonical"] == new_norm_kernels - replaced_norm_kernels


def _cu(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x)).to(dtype).cuda().contiguous()


@pytest.mark.parametrize("variant,V,R,E,d,B", [("block", 3000, 37, 40000, 40, 8), ("block", 3000, 37, 40000, 64, 8),
                                               ("basis", 2000, 23, 30000, 32, 4)])
def test_layer_matches_float64_oracle(variant, V, R, E, d, B):
    """block s = 5 and s = 8, basis: forward and every gradient against the float64 oracle with relation norms."""
    rng = np.random.RandomState(3)
    tr = one_relation_heavy(V, R, E, seed=11)
    H = rng.normal(0, 1, (V, d)).astype(np.float32)
    dOut = rng.normal(0, 1, (V, d)).astype(np.float32)
    w = oracle.init_block_layer(rng, R, d, B) if variant == "block" else oracle.init_basis_layer(rng, R, d, B)
    nf, nb = ron.relation_norms(tr, np.float32)
    ref_out, ref_g = oracle.layer_fwd_bwd(variant, H, tr, w, nf, nb, dOut, None, 1.0, True, torch.float64)
    g = ops.Graph(tr, V, R, norm_mode="relation", device=0)
    Ht = _cu(H).requires_grad_(True)
    names = (("W_forward", "W_backward", "W_self") if variant == "block"
             else ("W_forward", "W_backward", "C_forward", "C_backward", "W_self"))
    ts = [_cu(w[k]).requires_grad_(True) for k in names]
    if variant == "block":
        out = ops.block_layer(Ht, ts[0], ts[1], ts[2], g, B, None, 1.0, True)
    else:
        out = ops.basis_layer(Ht, ts[0], ts[1], ts[2], ts[3], ts[4], g, None, 1.0, True)
    out.backward(_cu(dOut))
    torch.cuda.synchronize()
    assert rel(out.detach().cpu().numpy(), ref_out) < 1e-4
    assert rel(Ht.grad.cpu().numpy(), ref_g["H"]) < 1e-4
    for k, t in zip(names, ts):
        assert rel(t.grad.cpu().numpy(), ref_g[k]) < 1e-4, k


@pytest.mark.parametrize("name", sorted(rn.CASES))
def test_product_matches_reference_relation_outputs(toy, name):
    c = rn.load_case(name)
    V, R = int(c["V"]), int(c["R"])
    settings_file, overrides, decoder = rn.CASES[name]
    enc, dec = merged_settings(toy, settings_file, V, R, len(c["test_graph"]))
    for k, v in overrides.items():
        enc.put(k, v)
        if k != "Name":
            dec.put(k, v)
    for s in (enc, dec):
        s.put("NormalizationMode", "relation")
    if decoder:
        dec.put("Name", decoder)
    from relationprediction_b200.common import model_builder
    model = model_builder.build_decoder(model_builder.build_encoder(enc, c["test_graph"]), dec)
    model.set_device("cuda:0")
    model.initialize_train()
    ws = model.get_weights()
    assert len(ws) == int(c["n_weights"])
    with torch.no_grad():
        for i, w in enumerate(ws):
            w.copy_(torch.tensor(c["w%d" % i], dtype=torch.float32, device=w.device))
    masks = [torch.tensor(c["mask%d" % i], dtype=torch.uint8, device="cuda:0") for i in range(int(c["n_masks"]))]
    for layer, m in zip(layers_of(model), masks):
        layer.make_drop_mask = (lambda rows, mode, m=m, k=layer.dropout_keep_probability:
                                (m, k) if mode == 'train' else (None, 1.0))
    total = model.train_loss(c["graph_split"], c["X"], c["Y"])
    total.backward()
    ref_total = float(c["loss"]) + float(c["reg"])
    assert abs(total.item() - ref_total) <= 1e-4 * abs(ref_total)
    for i, w in enumerate(ws):
        if bool(c["g%d_unused" % i]):
            assert w.grad is None or float(w.grad.abs().max()) == 0.0, i
            continue
        assert rel(w.grad.cpu().numpy(), c["g%d" % i]) < 1e-4, i
    model.preprocess(c["test_graph"])
    model.register_for_test(c["test_graph"])
    # scores: every entry by absolute error; the pre-sigmoid energies (logits of both sides) wherever the sigmoid is
    # not saturated, relative to the largest energy magnitude of the case.  The per-relation norms weigh each message
    # up to 1 instead of 1/degree, so the Toy energies are sums of larger, cancelling fp32 terms: measured on an H100,
    # the worst live energy is off by 1.0e-4 (basis) and 1.8e-4 (ComplEx) of the energy scale, hence the 1e-3 bar
    errs, scale = [], 1.0
    for got, ref in ((model.score(c["test_X"]), c["predict"]), (model.score_all_objects(c["test_X"]), c["all_objects"]),
                     (model.score_all_subjects(c["test_X"]), c["all_subjects"])):
        got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
        assert got.shape == ref.shape and np.abs(got - ref).max() < 2e-4
        live = (ref > 1e-3) & (ref < 1 - 1e-3) & (got > 0) & (got < 1)
        if live.any():
            lg, lr = np.log(got[live] / (1 - got[live])), np.log(ref[live] / (1 - ref[live]))
            errs.append(np.abs(lg - lr).max())
            scale = max(scale, np.abs(lr).max())
    assert max(errs, default=0.0) / scale < 1e-3


def test_toy_driver_trains_evaluates_and_round_trips_a_checkpoint(toy, tmp_path, capsys):
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(TOY_EXP.format(layers=2, concat="Yes").replace("\tConcatenation=Yes\n",
                                                                  "\tConcatenation=Yes\n\tNormalizationMode=relation\n"))
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--save-path", str(tmp_path / "ckpt" / "Toy")])
    text = capsys.readouterr().out
    assert "Initial loss" in text and "Validation filtered MRR" in text
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and losses[-1] < losses[0]
    rep = model
    while rep is not None and type(rep).__name__ != "Representation":
        rep = rep.next_component
    assert rep is not None and rep.norm_mode == "relation"
    tri = np.array(toy["train"])[:20]
    summ = scorer.compute_scores(tri).get_summary()
    assert 0.0 < summ.results["Filtered"]["MRR"] <= 1.0
    before = np.asarray(model.score_all_objects(tri), np.float64)
    ckpt = "%s-%d.pt" % (tmp_path / "rt", model.save_iter)
    model.save(str(tmp_path / "rt"))
    saved = [w.detach().clone() for w in model.get_weights()]
    with torch.no_grad():
        for w in model.get_weights():
            w.zero_()
    model.load(ckpt)
    for a, b in zip(model.get_weights(), saved):
        assert torch.equal(a.detach(), b)
    # the weight-id-major block walks sum in a run-dependent order: equal up to fp32 rounding
    np.testing.assert_allclose(np.asarray(model.score_all_objects(tri), np.float64), before, rtol=1e-6, atol=1e-7)
