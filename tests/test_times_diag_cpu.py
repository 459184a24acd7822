"""CPU: the basis layer with per-channel sigmoid coefficients (DiagonalCoefficients=Yes) against golden vectors
produced by running the reference's own classes (tests/golden/make_times_diag_golden.py over tests/golden/tf1_shim.py).

  * the oracle chain (tests/times_diag_oracle.py, float64) reproduces loss, regularisation, every weight gradient, the
    test-mode scores and the reference Scorer's raw / filtered MRR and Hits at 1e-10;
  * the host plugin chain (factory, BasisGcnTimesDiag, HighwayLayer, RelationEmbedding, BilinearDiag, Scorer)
    reproduces the same outputs with the library calls replaced by the oracle inside this test;
  * the factory applies the reference's layer precedence, orders and initialises the weights like it, and still
    rejects AddDiagonal and the featureless combination;
  * checkpoints round-trip the layer's weights;
  * the new C-ABI entry points validate their arguments before touching a device."""
import ctypes
import os

import numpy as np
import pytest
import torch

import highway_oracle as hw
import times_diag_oracle as td
from oracle import rgcn_oracle as oracle
from relationprediction_b200 import _lib, ops
from relationprediction_b200.common import model_builder
from relationprediction_b200.encoders.affine_transform import AffineTransform
from relationprediction_b200.encoders.message_gcns.gcn_basis_times_diag import BasisGcnTimesDiag
from relationprediction_b200.encoders.message_gcns.message_gcn import MessageGcn
from relationprediction_b200.encoders.relation_embedding import RelationEmbedding
from relationprediction_b200.extras.highway_layer import HighwayLayer
from test_highway_cpu import OracleScores, chain_of, ranking, rel
from test_plugin_chain_cpu import OracleGraph, oracle_distmult
from test_plugin_host import merged_settings
from test_reference_golden import KEEP, LAMBDA

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_times_diag_golden.npz")
DT = torch.float64


def _o(d, B, code=None, **extra):
    o = {"InternalEncoderDimension": str(d), "CodeDimension": str(code or d), "NumberOfBasisFunctions": str(B),
         "DiagonalCoefficients": "Yes"}
    o.update(extra)
    return o


# golden case -> (settings file, overrides of the generator, library norm mode)
CASES = {
    "times_diag_basis_toy_tf_kernel": ("gcn_basis.exp", _o(16, 3), "tf_unsorted_compat"),
    "times_diag_basis_toy_canonical": ("gcn_basis.exp", _o(16, 3), "canonical"),
    "times_diag_basis_toy_1layer_canonical": ("gcn_basis.exp", _o(12, 2, NumberOfLayers="1"), "canonical"),
    "times_diag_basis_toy_3layer_canonical": ("gcn_basis.exp", _o(12, 2, NumberOfLayers="3"), "canonical"),
    "times_diag_basis_toy_outproj_canonical": ("gcn_basis.exp", _o(16, 2, code=12, UseOutputTransform="Yes"),
                                               "canonical"),
    "times_diag_basis_syn_canonical": ("gcn_basis.exp", _o(16, 4), "canonical"),
    "times_diag_highway_toy_canonical": ("gcn_basis.exp", _o(16, 2, SkipConnections="Highway"), "canonical"),
    "times_diag_block_toy_canonical": ("gcn_block.exp", _o(12, 3), "canonical"),
}


def load_case(name):
    z = np.load(GOLDEN)
    p = name + "/"
    return {k[len(p):]: z[k] for k in z.files if k.startswith(p)}


def case_shape(name):
    settings_file, overrides, norm_mode = CASES[name]
    n_layers = int(overrides.get("NumberOfLayers", "2"))
    outproj = overrides.get("UseOutputTransform") == "Yes"
    highway = overrides.get("SkipConnections") == "Highway"
    return settings_file, overrides, norm_mode, n_layers, outproj, highway


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_times_diag_outputs(name):
    c = load_case(name)
    _, _, norm_mode, n_layers, outproj, highway = case_shape(name)
    names = td.weight_names(n_layers, outproj, highway)
    assert len(names) == int(c["n_weights"])
    leaves = {nm: torch.tensor(c["w%d" % i], dtype=DT, requires_grad=True) for i, nm in enumerate(names)}
    V = int(c["V"])
    masks = [torch.tensor(c["mask%d" % i]) for i in range(int(c["n_masks"]))]
    assert len(masks) == n_layers
    codes = td.encode(leaves, n_layers, outproj, highway, c["graph_split"], V, "train", masks, KEEP, norm_mode)
    loss, reg, _ = oracle.distmult_loss(codes, leaves["W_relation"], c["X"], c["Y"], DT)
    (loss + LAMBDA * reg).backward()
    assert abs(loss.item() - float(c["loss"])) <= 1e-10 * abs(float(c["loss"]))
    assert abs(LAMBDA * reg.item() - float(c["reg"])) <= 1e-10 * abs(float(c["reg"]))
    for i, nm in enumerate(names):
        assert not bool(c["g%d_unused" % i]), nm        # the layer's bias is added: every weight has a gradient
        assert rel(leaves[nm].grad.numpy(), c["g%d" % i]) < 1e-10, nm
    with torch.no_grad():
        tc = td.encode(leaves, n_layers, outproj, highway, c["test_graph"], V, "test", masks, KEEP, norm_mode)
    Wr, tX = leaves["W_relation"].detach(), c["test_X"]
    e, _ = oracle.distmult_energies(tc, Wr, tX, DT)
    assert rel(torch.sigmoid(e).numpy(), c["predict"]) < 1e-10
    assert rel(oracle.distmult_predict_all_objects(tc, Wr, tX, DT).numpy(), c["all_objects"]) < 1e-10
    assert rel(oracle.distmult_predict_all_subjects(tc, Wr, tX, DT).numpy(), c["all_subjects"]) < 1e-10
    assert np.abs(ranking(OracleScores(tc, Wr), c["test_graph"], c["ranked"]) - c["ranking"]).max() < 1e-12


def test_layer_bias_gets_the_row_sum_of_the_output_gradient():
    """b is added (unlike BasisGcn / ConcatGcn): its gradient is nonzero and, for the last (linear) layer, equals the
    column sums of the layer's output gradient."""
    c = load_case("times_diag_basis_toy_1layer_canonical")
    names = td.weight_names(1, False)
    i = names.index("L0.b")
    assert float(np.abs(c["g%d" % i]).max()) > 1e-4
    leaves = {nm: torch.tensor(c["w%d" % k], dtype=DT, requires_grad=True) for k, nm in enumerate(names)}
    codes = td.encode(leaves, 1, False, False, c["graph_split"], int(c["V"]), "train", [torch.tensor(c["mask0"])],
                      KEEP, "canonical")
    codes.retain_grad()
    loss, reg, _ = oracle.distmult_loss(codes, leaves["W_relation"], c["X"], c["Y"], DT)
    (loss + LAMBDA * reg).backward()
    assert rel(codes.grad.sum(0).numpy(), c["g%d" % i]) < 1e-10


def oracle_times_diag_layer(H, Vf, Vb, Cf, Cb, Ws, b, graph, drop_mask=None, keep=1.0, relu=True):
    return td.times_diag_forward(H, graph.triples, Vf, Vb, Cf, Cb, Ws, b, graph.nf, graph.nb, drop_mask, keep, relu,
                                 DT)


@pytest.fixture
def oracle_backed_ops(monkeypatch):
    monkeypatch.setattr(ops, "Graph", OracleGraph)
    monkeypatch.setattr(ops, "basis_diagcoef_layer", oracle_times_diag_layer)
    monkeypatch.setattr(ops, "distmult", oracle_distmult)
    monkeypatch.setattr(ops, "highway", hw.highway)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)


def build_model(toy, name, V, R, E):
    settings_file, overrides, norm_mode, _, _, _ = case_shape(name)
    enc, dec = merged_settings(toy, settings_file, V, R, E)
    for s in (enc, dec):
        for k, v in overrides.items():
            s.put(k, v)
        s.put("NormalizationMode", norm_mode)
    return model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_chain_reproduces_reference_times_diag_outputs(toy, oracle_backed_ops, name):
    c = load_case(name)
    _, _, norm_mode, n_layers, outproj, highway = case_shape(name)
    model = build_model(toy, name, int(c["V"]), int(c["R"]), len(c["test_graph"]))
    model.set_device("cpu")
    model.initialize_train()
    names = td.weight_names(n_layers, outproj, highway)
    ws = model.get_weights()
    assert len(ws) == len(names)
    for i, w in enumerate(ws):
        assert tuple(w.shape) == c["w%d" % i].shape, names[i]
        w.data = torch.tensor(c["w%d" % i], dtype=DT)
    layers, comp = [], model
    while comp is not None:
        if isinstance(comp, MessageGcn):
            layers.append(comp)
        comp = comp.next_component
    assert len(layers) == n_layers and all(isinstance(l, BasisGcnTimesDiag) for l in layers)
    for layer, i in zip(layers[::-1], range(int(c["n_masks"]))):   # masks in the order drawn: layer 0 first
        m = torch.tensor(c["mask%d" % i])
        layer.make_drop_mask = (lambda rows, mode, m=m, k=layer.dropout_keep_probability:
                                (m, k) if mode == 'train' else (None, 1.0))
    total = model.train_loss(c["graph_split"], c["X"], c["Y"])
    total.backward()
    ref_total = float(c["loss"]) + float(c["reg"])
    tol = 1e-10 if norm_mode == "canonical" else 1e-6   # tf_unsorted_compat norms travel as float32
    assert abs(total.item() - ref_total) <= tol * abs(ref_total)
    for i, (nm, w) in enumerate(zip(names, ws)):
        assert rel(w.grad.numpy(), c["g%d" % i]) < tol, nm
    model.preprocess(c["test_graph"])
    model.register_for_test(c["test_graph"])
    for got, ref in ((model.score(c["test_X"]), c["predict"]),
                     (model.score_all_objects(c["test_X"]), c["all_objects"]),
                     (model.score_all_subjects(c["test_X"]), c["all_subjects"])):
        assert got.shape == ref.shape and np.abs(np.asarray(got, np.float64) - ref).max() < 100 * tol
    got = ranking(model, c["test_graph"], c["ranked"])
    assert np.abs(got - c["ranking"]).max() < (1e-12 if tol == 1e-10 else 5e-3)


def diag_settings(toy, settings_file="gcn_basis.exp", **flags):
    enc, dec = merged_settings(toy, settings_file, toy["V"], toy["R"], len(toy["train"]))
    enc.put("DiagonalCoefficients", "Yes")
    for k, v in flags.items():
        enc.put(k, v)
    return enc, dec


@pytest.mark.parametrize("settings_file,flags", [("gcn_basis.exp", {}), ("gcn_block.exp", {}),
                                                 ("gcn_basis.exp", {"Concatenation": "Yes"}),
                                                 ("gcn_basis.exp", {"StoreEdgeData": "Yes"}),
                                                 ("gcn_block.exp", {"StoreEdgeData": "Yes"})])
def test_factory_precedence_builds_the_times_diag_layer(toy, settings_file, flags):
    enc, dec = diag_settings(toy, settings_file, **flags)
    model = model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)
    chain = chain_of(model)
    assert [type(c) for c in chain[1:5]] == [RelationEmbedding, BasisGcnTimesDiag, BasisGcnTimesDiag, AffineTransform]
    assert not chain[2].use_nonlinearity and chain[3].use_nonlinearity
    assert chain[2].n_coefficients == int(enc["NumberOfBasisFunctions"])


def test_factory_add_diagonal_and_featureless_still_raise(toy):
    enc, _ = diag_settings(toy, AddDiagonal="Yes")
    with pytest.raises(NotImplementedError, match="AddDiagonal"):
        model_builder.build_encoder(enc, toy["train"])
    enc, _ = diag_settings(toy, "gcn_block.exp", AddDiagonal="Yes")
    with pytest.raises(NotImplementedError, match="AddDiagonal"):
        model_builder.build_encoder(enc, toy["train"])
    for extra in ({}, {"StoreEdgeData": "Yes"}):
        enc, _ = diag_settings(toy, UseInputTransform="No", **extra)
        with pytest.raises(NotImplementedError, match="push kernel"):
            model_builder.build_encoder(enc, toy["train"])
    with pytest.raises(NotImplementedError, match="push kernel"):
        BasisGcnTimesDiag([8, 8], {"DropoutKeepProbability": "1", "NumberOfBasisFunctions": "2"}, onehot_input=True)


def test_factory_wraps_times_diag_layers_in_highways(toy):
    enc, dec = diag_settings(toy, SkipConnections="Highway")
    model = model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)
    chain = chain_of(model)
    assert [type(c) for c in chain[1:7]] == [RelationEmbedding, HighwayLayer, BasisGcnTimesDiag, HighwayLayer,
                                             BasisGcnTimesDiag, AffineTransform]
    assert chain[2].next_component is chain[3] and chain[2].next_component_2 is chain[4]
    assert chain[4].next_component is chain[5] and chain[4].next_component_2 is chain[6]


def test_weight_shapes_order_and_initialisation(toy):
    enc, dec = diag_settings(toy, InternalEncoderDimension="200", CodeDimension="200", NumberOfBasisFunctions="5")
    model = model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)
    np.random.seed(5)
    model.set_device("cpu")
    model.initialize_train()
    top, first = chain_of(model)[2], chain_of(model)[3]
    d, B, R = 200, 5, toy["R"]
    assert [tuple(w.shape) for w in first.local_get_weights()] == [(d, B, d), (d, B, d), (R, B, d), (R, B, d),
                                                                  (d, d), (d,)]
    ws = model.get_weights()
    expect = chain_of(model)[4].local_get_weights() + first.local_get_weights() + top.local_get_weights()
    assert all(a is b for a, b in zip(ws, expect)) and len(ws) == len(expect) + 1
    std = 3 / np.sqrt(2 * d)             # glorot_variance([d, d]) as a std-dev (:26)
    for w in (first.W_forward, first.W_backward, first.W_self):
        assert abs(float(w.detach().std()) / std - 1) < 0.02 and abs(float(w.detach().mean())) < 0.01
    for w in (first.C_forward, first.C_backward):     # N(0, 1) (:31-33)
        assert abs(float(w.detach().std()) - 1) < 0.02 and abs(float(w.detach().mean())) < 0.02
    assert float(first.b.detach().abs().max()) == 0.0 and first.b.requires_grad
    assert first.local_get_regularization() == 0.0


def test_checkpoint_round_trips_times_diag_weights(toy, oracle_backed_ops, tmp_path):
    enc, dec = diag_settings(toy, InternalEncoderDimension="16", CodeDimension="16", NumberOfBasisFunctions="2")
    model = model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)
    np.random.seed(1)
    model.set_device("cpu")
    model.initialize_train()
    layers = [c for c in chain_of(model) if isinstance(c, BasisGcnTimesDiag)]
    with torch.no_grad():
        for i, l in enumerate(layers):
            l.b.add_(0.5 * (i + 1))
    saved = [w.detach().clone() for w in model.get_weights()]
    model.save(str(tmp_path / "ckpt"))
    with torch.no_grad():
        for w in model.get_weights():
            w.zero_()
    model.load(str(tmp_path / "ckpt-0.pt"))
    for a, b in zip(model.get_weights(), saved):
        assert torch.equal(a.detach(), b)
    assert torch.equal(layers[0].b.detach(), torch.full((16,), 0.5))
    assert layers[0].C_forward.shape == (toy["R"], 2, 16)


def test_times_diag_entry_points_reject_bad_arguments_without_a_gpu(toy):
    lib = _lib.load()
    g = ops.Graph(np.array(toy["train"], np.int32), toy["V"], toy["R"])   # host-only graph
    d, B = 8, 2
    buf = ctypes.create_string_buffer(1 << 22)
    assert lib.rgcn_basis_diagcoef_workspace_bytes(None, d, B, 0) == -1
    assert lib.rgcn_basis_diagcoef_workspace_bytes(g.handle, 0, B, 0) == -1
    assert lib.rgcn_basis_diagcoef_workspace_bytes(g.handle, d, 0, 0) == -1
    need_f = lib.rgcn_basis_diagcoef_workspace_bytes(g.handle, d, B, 0)
    need_b = lib.rgcn_basis_diagcoef_workspace_bytes(g.handle, d, B, 1)
    assert 0 < need_f < need_b <= len(buf)
    assert need_f >= 2 * toy["R"] * B * d * 4 and need_b - need_f >= toy["V"] * 2 * B * d * 4

    def fwd(gh=g.handle, d=d, B=B, H=buf, b=buf, out=buf, saved=buf, keep=1.0, ws=need_f):
        return lib.rgcn_basis_diagcoef_forward(gh, d, B, H, buf, buf, buf, buf, buf, b, None, keep, 1, out, saved,
                                               buf, ws, None)

    def bwd(gh=g.handle, d=d, B=B, H=buf, out=buf, db=buf, dCf=buf, keep=1.0, relu=1, ws=need_b):
        return lib.rgcn_basis_diagcoef_backward(gh, d, B, H, buf, buf, buf, buf, buf, None, keep, relu, out, buf, buf,
                                                buf, buf, buf, dCf, buf, buf, db, buf, ws, None)
    for call in (fwd, bwd):
        assert call(gh=None) == -1
        assert call(d=6) == -1 and b"d % 4" in lib.rgcn_last_error()
        assert call(d=0) == -1 and call(B=0) == -1
        assert call(H=None) == -1 and b"null pointer" in lib.rgcn_last_error()
        assert call(keep=0.0) == -1
        assert call(ws=16) == -4 and b"workspace" in lib.rgcn_last_error()
        assert call() == -5 and b"host-only" in lib.rgcn_last_error()     # valid arguments, host-only graph
    assert fwd(b=None) == -1 and fwd(out=None) == -1 and fwd(saved=None) == -1
    assert bwd(db=None) == -1 and bwd(dCf=None) == -1 and bwd(out=None) == -1
    assert bwd(out=None, relu=0) == -5     # out is only read for the ReLU gradient


def test_times_diag_op_rejects_cpu_tensors():
    class FakeGraph(object):
        V_dst = V_src = 6
        n_relw = 4
        handle = None
    d, B, R = 8, 2, 2
    with pytest.raises(_lib.RgcnError, match="CUDA float32"):
        ops.basis_diagcoef_layer(torch.zeros(6, d), torch.zeros(d, B, d), torch.zeros(d, B, d), torch.zeros(R, B, d),
                                 torch.zeros(R, B, d), torch.zeros(d, d), torch.zeros(d), FakeGraph())
    with pytest.raises(_lib.RgcnError, match=r"\[R, B, d\]"):
        ops.basis_diagcoef_layer(torch.zeros(6, d), torch.zeros(d, B, d), torch.zeros(d, B, d), torch.zeros(R, B),
                                 torch.zeros(R, B), torch.zeros(d, d), torch.zeros(d), FakeGraph())
