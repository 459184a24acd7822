"""CPU: the per-relation normaliser (NormalizationMode=relation, RGCN_NORM_RELATION: message k gets
1 / #{messages with the same destination and weight id}, the R-GCN paper's c_{i,r} and the reference's 'local' branch,
extras/graph_representations.py:94-107, :134-147).

  * the host builder (rgcn_graph_create, device = -1) gives the Toy known answers and equals a numpy restatement bit
    for bit, duplicate triples and isolated nodes included; every sorted view carries those norms;
  * the oracle chains and the host plugin chain reproduce the goldens of the reference's own 'local' code
    (tests/golden/make_relation_norm_golden.py) at 1e-10 for every layer type the mode reaches, with the
    relation norms of tests/relation_norm_oracle.py;
  * the node-shard planners use the global per-(dst, weight id) counts, and the torch planner equals the numpy one;
  * canonical and tf_unsorted_compat graphs are byte-identical to those of the library before the mode existed, and
    the settings map to the same constructor arguments as before."""
import hashlib
import os

import numpy as np
import pytest
import torch

import highway_oracle as hw
import relation_norm_oracle as ron
import test_basis_onehot_cpu as onehot_t
import test_complex_cpu as complex_t
import test_gcn_diag_cpu as gcn_diag_t
import test_highway_cpu as highway_t
import test_reference_golden as reference_t
import test_times_diag_cpu as times_diag_t
from conftest import synthetic_kg
from oracle import rgcn_oracle as oracle
from relationprediction_b200 import _lib, ops, parallel
from relationprediction_b200.common import model_builder
from relationprediction_b200.encoders.message_gcns.message_gcn import MessageGcn
from relationprediction_b200.extras import graph_representations
from test_plugin_chain_cpu import OracleGraph, oracle_basis_layer, oracle_block_layer, oracle_distmult
from test_plugin_host import merged_settings

@pytest.fixture(autouse=True)
def relation_oracle(monkeypatch):
    """The oracle chains look graph_norms up in oracle.rgcn_oracle: answer mode "relation" there (tests/relation_norm_oracle.py)."""
    ron.install(monkeypatch)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_relation_norm_golden.npz")
DT = torch.float64
ALL_EXPORTS = list(range(21))


def numpy_relation_norms(triples, R):
    """Independent restatement: count each (destination, weight id) pair over the 2E messages."""
    t = np.asarray(triples, np.int64).reshape(-1, 3)
    dst = np.concatenate([t[:, 2], t[:, 0]])
    relw = np.concatenate([t[:, 1], t[:, 1] + R])
    key = dst * (2 * R) + relw
    order = np.argsort(key, kind="stable")
    sk = key[order]
    starts = np.flatnonzero(np.r_[True, sk[1:] != sk[:-1]])
    lens = np.diff(np.r_[starts, len(sk)])
    count = np.empty(len(sk), np.int64)
    count[order] = np.repeat(lens, lens)
    return np.float32(1.0) / count.astype(np.float32), len(starts)


def graph_cases():
    toy = np.array(_toy()["train"], np.int32)
    dup = np.concatenate([toy, toy[:10], toy[3:4], toy[3:4]])             # duplicate triples count as often as they occur
    iso = np.array([[0, 0, 1], [1, 1, 0], [0, 0, 2], [2, 1, 0], [2, 0, 1]], np.int32)   # node 3 and 4 isolated
    return {"toy": (toy, 16, 9), "skewed": (synthetic_kg(3000, 37, 40000, seed=3, skewed=True), 3000, 37),
            "duplicates": (dup, 16, 9), "isolated": (iso, 5, 2)}


def _toy():
    import json
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "toy_golden.json")) as fh:
        return json.load(fh)


def test_toy_known_answers():
    tr = np.array(_toy()["train"], np.int32)
    g = ops.Graph(tr, 16, 9, norm_mode="relation")
    n, E = g.export(_lib.X_MSG_NORM), len(tr)
    np.testing.assert_array_equal(n[:8], np.float32([1 / 4, 1, 1, 1 / 4, 1, 1 / 2, 1, 1 / 2]))
    np.testing.assert_array_equal(n[E:E + 8], np.float32([1, 1, 1, 1, 1, 1, 1, 1 / 2]))
    assert g.info()[9] == 60          # 28 forward + 32 backward (dst, weight id) groups
    nf_can, _ = oracle.graph_norms(tr, 16, "canonical")
    np.testing.assert_array_equal(nf_can[:8], np.float32([1 / 7, 1 / 3, 1 / 3, 1 / 7, 1, 1 / 3, 1 / 4, 1 / 7]))


@pytest.mark.parametrize("case", ["toy", "skewed", "duplicates", "isolated"])
def test_host_builder_equals_numpy_restatement(case):
    tr, V, R = graph_cases()[case]
    g = ops.Graph(tr, V, R, norm_mode="relation")
    want, groups = numpy_relation_norms(tr, R)
    msg = g.export(_lib.X_MSG_NORM)
    assert msg.tobytes() == want.tobytes()
    assert g.info()[9] == groups
    nf, nb = ron.relation_norms(tr)
    assert np.concatenate([nf, nb]).tobytes() == want.tobytes()
    # every sorted view carries the message's norm
    for norm_sel, mid_sel in ((_lib.X_DST_NORM, _lib.X_DST_MID), (_lib.X_SRC_NORM, _lib.X_SRC_MID),
                              (_lib.X_REL_NORM, _lib.X_REL_MID), (_lib.X_REL2_NORM, _lib.X_REL2_MID)):
        assert g.export(norm_sel).tobytes() == msg[g.export(mid_sel)].tobytes()
    # the sorted views themselves are those of the canonical build: only the norm differs
    gc = ops.Graph(tr, V, R)
    for which in ALL_EXPORTS:
        if which not in (_lib.X_DST_NORM, _lib.X_SRC_NORM, _lib.X_REL_NORM, _lib.X_REL2_NORM, _lib.X_MSG_NORM):
            assert g.export(which).tobytes() == gc.export(which).tobytes(), which


def test_unknown_norm_mode_is_rejected():
    import ctypes
    tr = np.zeros((1, 3), np.int32)
    h = ctypes.c_void_p(0)
    rc = _lib.load().rgcn_graph_create(ctypes.c_void_p(tr.ctypes.data), 1, 2, 1, _lib.RGCN_NORM_RELATION + 1, None,
                                       None, -1, None, ctypes.byref(h))
    assert rc < 0 and "norm_mode" in _lib.load().rgcn_last_error().decode()


# ---------------------------------------------------------------------------------------------------------------
# goldens of the reference's own 'local' code
# ---------------------------------------------------------------------------------------------------------------
def _o(d, B=None, **extra):
    o = {"InternalEncoderDimension": str(d), "CodeDimension": str(d)}
    if B is not None:
        o["NumberOfBasisFunctions"] = str(B)
    o.update(extra)
    return o


# golden case -> (settings file, overrides of the generator, decoder name or None)
CASES = {
    "relation_block_toy_s5": ("gcn_block.exp", _o(40, 8), None),
    "relation_block_syn_s8": ("gcn_block.exp", _o(32, 4), None),
    "relation_basis_toy": ("gcn_basis.exp", _o(24, 5), None),
    "relation_onehot_toy": ("gcn_basis.exp", _o(24, 5, UseInputTransform="No"), None),
    "relation_times_diag_toy": ("gcn_basis.exp", _o(16, 3, DiagonalCoefficients="Yes"), None),
    "relation_gcn_diag_toy": ("gcn_basis.exp", dict(Name="gcn_diag", **_o(16)), None),
    "relation_highway_block_toy": ("gcn_block.exp", _o(20, 4, SkipConnections="Highway"), None),
    "relation_block_complex_toy": ("gcn_block.exp", _o(40, 8), "complex"),
}


def load_case(name):
    z = np.load(GOLDEN)
    if name.endswith("_canonical"):        # the sparse_softmax grouping suffix of test_reference_golden
        name = name[:-len("_canonical")]
    p = name + "/"
    c = {k[len(p):]: z[k] for k in z.files if k.startswith(p)}
    assert c, name
    return c


def test_golden_differs_from_the_canonical_norm(monkeypatch):
    """The fixture pins the 'local' branch: the canonical norm does not reproduce it."""
    monkeypatch.setattr(reference_t, "load_case", load_case)
    c = load_case("relation_block_toy_s5")
    split = c["graph_split"]
    nf_r, _ = ron.relation_norms(split)
    nf_c, _ = oracle.graph_norms(split, int(c["V"]), "canonical")
    assert not np.array_equal(nf_r, nf_c)
    with pytest.raises(AssertionError):
        reference_t.test_oracle_matches_reference_code_outputs("relation_block_toy_s5", "block", "canonical",
                                                               "canonical")


def _oracle_chain(monkeypatch, name):
    """Each layer type's existing float64 oracle chain (1e-10 on loss, regularisation, every gradient, scores, and
    1e-12 on raw / filtered MRR and Hits), fed this fixture and norm mode "relation"."""
    settings_file, overrides, decoder = CASES[name]
    if name == "relation_onehot_toy":
        mod = onehot_t
        monkeypatch.setitem(mod.CASES, name, ({k: v for k, v in overrides.items() if k != "UseInputTransform"},
                                              "relation"))
        run = lambda: mod.test_oracle_matches_reference_onehot_outputs(name)            # noqa: E731
    elif name == "relation_times_diag_toy":
        mod = times_diag_t
        monkeypatch.setitem(mod.CASES, name, (settings_file, overrides, "relation"))
        run = lambda: mod.test_oracle_matches_reference_times_diag_outputs(name)        # noqa: E731
    elif name == "relation_gcn_diag_toy":
        mod = gcn_diag_t
        monkeypatch.setitem(mod.CASES, name, (overrides, "bilinear-diag", "relation"))
        run = lambda: mod.test_oracle_matches_reference_gcn_diag_outputs(name)          # noqa: E731
    elif name == "relation_highway_block_toy":
        mod = highway_t
        monkeypatch.setitem(mod.CASES, name, (settings_file, overrides, "block", "relation"))
        run = lambda: mod.test_oracle_matches_reference_highway_outputs(name)           # noqa: E731
    elif decoder == "complex":
        mod = complex_t
        monkeypatch.setitem(mod.CASES, name, ("block", settings_file, overrides, "relation"))
        run = lambda: mod.test_oracle_matches_reference_complex_outputs(name)           # noqa: E731
    else:
        mod = reference_t
        variant = "block" if settings_file == "gcn_block.exp" else "basis"
        run = lambda: mod.test_oracle_matches_reference_code_outputs(name, variant, "canonical", "relation")  # noqa
    monkeypatch.setattr(mod, "load_case", load_case)
    run()


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_relation_outputs(monkeypatch, name):
    _oracle_chain(monkeypatch, name)


@pytest.fixture
def oracle_backed_ops(monkeypatch):
    monkeypatch.setattr(ops, "Graph", OracleGraph)
    monkeypatch.setattr(ops, "block_layer", oracle_block_layer)
    monkeypatch.setattr(ops, "basis_layer", oracle_basis_layer)
    monkeypatch.setattr(ops, "basis_onehot_layer", onehot_t.oracle_onehot_layer)
    monkeypatch.setattr(ops, "basis_diagcoef_layer", times_diag_t.oracle_times_diag_layer)
    monkeypatch.setattr(ops, "diag_layer", gcn_diag_t.oracle_diag_layer)
    monkeypatch.setattr(ops, "highway", hw.highway)
    monkeypatch.setattr(ops, "distmult", oracle_distmult)
    monkeypatch.setattr(ops, "complex_score", complex_t.oracle_complex)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)


def build_model(toy, name, c):
    settings_file, overrides, decoder = CASES[name]
    enc, dec = merged_settings(toy, settings_file, int(c["V"]), int(c["R"]), len(c["test_graph"]))
    for k, v in overrides.items():
        enc.put(k, v)
        if k != "Name":
            dec.put(k, v)
    for s in (enc, dec):
        s.put("NormalizationMode", "relation")
    if decoder:
        dec.put("Name", decoder)
    return model_builder.build_decoder(model_builder.build_encoder(enc, c["test_graph"]), dec)


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_chain_reproduces_reference_relation_outputs(toy, oracle_backed_ops, name):
    """The product's factory, Representation (NormalizationMode=relation -> ops.Graph(norm_mode="relation")), layers,
    decoders and Scorer, with the library calls replaced by the oracle, at 1e-10."""
    c = load_case(name)
    model = build_model(toy, name, c)
    model.set_device("cpu")
    model.initialize_train()
    ws = model.get_weights()
    assert len(ws) == int(c["n_weights"])
    for i, w in enumerate(ws):
        assert tuple(w.shape) == c["w%d" % i].shape, i
        w.data = torch.tensor(c["w%d" % i], dtype=DT)
    layers, comp = [], model
    while comp is not None:
        if isinstance(comp, MessageGcn):
            layers.append(comp)
        comp = comp.next_component
    for layer, i in zip(layers[::-1], range(int(c["n_masks"]))):   # masks in the order drawn: layer 0 first
        m = torch.tensor(c["mask%d" % i])
        layer.make_drop_mask = (lambda rows, mode, m=m, k=layer.dropout_keep_probability:
                                (m, k) if mode == 'train' else (None, 1.0))
    graph = model
    while graph is not None and not isinstance(graph, graph_representations.Representation):
        graph = graph.next_component
    assert graph is not None and graph.norm_mode == "relation"
    total = model.train_loss(c["graph_split"], c["X"], c["Y"])
    total.backward()
    ref_total = float(c["loss"]) + float(c["reg"])
    assert abs(total.item() - ref_total) <= 1e-10 * abs(ref_total)
    for i, w in enumerate(ws):
        if bool(c["g%d_unused" % i]):
            assert w.grad is None or float(w.grad.abs().max()) == 0.0, i
        else:
            assert rel(w.grad.numpy(), c["g%d" % i]) < 1e-10, i
    model.preprocess(c["test_graph"])
    model.register_for_test(c["test_graph"])
    for got, ref in ((model.score(c["test_X"]), c["predict"]),
                     (model.score_all_objects(c["test_X"]), c["all_objects"]),
                     (model.score_all_subjects(c["test_X"]), c["all_subjects"])):
        assert got.shape == ref.shape and np.abs(np.asarray(got, np.float64) - ref).max() < 1e-8
    got = highway_t.ranking(model, c["test_graph"], c["ranked"])
    assert np.abs(got - c["ranking"]).max() < 1e-12


# ---------------------------------------------------------------------------------------------------------------
# node-shard planners
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_shard_plans_use_global_relation_counts(world):
    V, R, E = 900, 6, 7000
    tr = synthetic_kg(V, R, E, seed=9, skewed=True)
    single = ops.Graph(tr, V, R, norm_mode="relation").export(_lib.X_MSG_NORM)
    dst, _, _, norm = parallel.global_messages(tr, V, R, "relation")
    assert norm.tobytes() == single.tobytes()
    seen = np.zeros(2 * E, bool)
    t = torch.from_numpy(tr)
    for rank in range(world):
        h = parallel.ShardPlan(tr, V, R, rank, world, norm_mode="relation")
        assert h.msg_norm.tobytes() == single[h.msg_global_id].tobytes()
        seen[h.msg_global_id] = True
        dv = parallel.ShardPlanDevice(t, V, R, rank, world, norm_mode="relation", keep_global_ids=True)
        assert (dv.lo, dv.hi, dv.n_local, dv.n_halo) == (h.lo, h.hi, h.n_local, h.n_halo)
        for name in ("msg_dst", "msg_src", "msg_relw", "msg_norm", "msg_global_id", "halo_nodes", "send_rows"):
            np.testing.assert_array_equal(getattr(dv, name).numpy(), getattr(h, name), err_msg=name)
        assert dv.msg_norm.dtype == torch.float32
    assert seen.all()


# ---------------------------------------------------------------------------------------------------------------
# the existing modes are unchanged
# ---------------------------------------------------------------------------------------------------------------
# sha256 over info() and every export of the graphs built by the library before NormalizationMode=relation existed
BEFORE = {
    ("toy", "canonical"): "bd5a9fa0db043a75231dda74e6d390c9a81e33dd73ff88c11ed58f2b9432b372",
    ("toy", "tf_unsorted_compat"): "7a409e95923c60476efd5e98da5fede72a1b5b6703bab4b734c7f639c9da9cea",
    ("skewed", "canonical"): "36e048c6af267c04c1941b585117d885860ba56b9b89e415eac69f2b8c052bba",
    ("skewed", "tf_unsorted_compat"): "dcb532ad5e6f27ddd5e295528f0cfaecab930d0320cdd2da8c4643948e8d70d8",
}


def graph_digest(tr, V, R, mode):
    if mode == "tf_unsorted_compat":
        nf = graph_representations._tf_compat(tr[:, 2], V)
        nb = graph_representations._tf_compat(tr[:, 0], V)
        g = ops.Graph(tr, V, R, norm_mode="explicit", norm_f=nf, norm_b=nb)
    else:
        g = ops.Graph(tr, V, R, norm_mode=mode)
    h = hashlib.sha256(np.array(g.info(), np.int64).tobytes())
    for which in ALL_EXPORTS:
        h.update(g.export(which).tobytes())
    return h.hexdigest()


@pytest.mark.parametrize("case,mode", sorted(BEFORE))
def test_existing_modes_build_byte_identical_graphs(case, mode):
    tr, V, R = graph_cases()[case]
    assert graph_digest(tr, V, R, mode) == BEFORE[(case, mode)]


@pytest.mark.parametrize("setting,expected", [(None, {"norm_mode": "canonical"}),
                                              ("canonical", {"norm_mode": "canonical"}),
                                              ("tf_unsorted_compat", {"norm_mode": "explicit"}),
                                              ("relation", {"norm_mode": "relation"}),
                                              ("something_else", {"norm_mode": "canonical"})])
def test_settings_select_the_constructor_arguments(monkeypatch, setting, expected):
    calls = []

    class Recorder(object):
        def __init__(self, triples, n_entities, n_relations, norm_mode="canonical", norm_f=None, norm_b=None,
                     device=None):
            calls.append(dict(norm_mode=norm_mode, norm_f=norm_f, norm_b=norm_b))

    monkeypatch.setattr(ops, "Graph", Recorder)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    tr = np.array(_toy()["train"], np.int32)
    settings = {"EntityCount": "16", "RelationCount": "9"}
    if setting is not None:
        settings["NormalizationMode"] = setting
    rep = graph_representations.Representation(tr, settings)
    rep.set_device("cpu")
    rep.local_initialize_train()
    rep.X.set(tr)
    rep.get_graph()
    assert len(calls) == 1 and calls[0]["norm_mode"] == expected["norm_mode"]
    if setting == "tf_unsorted_compat":
        np.testing.assert_array_equal(calls[0]["norm_f"], graph_representations._tf_compat(tr[:, 2], 16))
        np.testing.assert_array_equal(calls[0]["norm_b"], graph_representations._tf_compat(tr[:, 0], 16))
    else:
        assert calls[0]["norm_f"] is None and calls[0]["norm_b"] is None
