"""CPU: the highway skip connection (SkipConnections=Highway) against golden vectors produced by running the
reference's own classes (tests/golden/make_highway_golden.py over tests/golden/tf1_shim.py).

  * the oracle chain (tests/highway_oracle.py, float64) reproduces loss, regularisation, every weight gradient, the
    test-mode scores and the reference Scorer's raw / filtered MRR and Hits at 1e-10;
  * the host plugin chain (factory, HighwayLayer, the layers, RelationEmbedding, BilinearDiag, Scorer) reproduces the
    same outputs with the library calls replaced by the oracle inside this test;
  * the factory wraps every feature-input layer, orders the weights like the reference and initialises W and b like
    it; it rejects Highway on a featureless encoder, where the reference's gate is dead (also checked on the fixture);
  * checkpoints round-trip the highway weights;
  * the new C-ABI entry points validate their arguments before touching a device."""
import ctypes
import os

import numpy as np
import pytest
import torch

import highway_oracle as hw
from oracle import rgcn_oracle as oracle
from relationprediction_b200 import _lib, ops
from relationprediction_b200.common import evaluation, model_builder
from relationprediction_b200.encoders.affine_transform import AffineTransform
from relationprediction_b200.encoders.message_gcns.gcn_basis import BasisGcn
from relationprediction_b200.encoders.message_gcns.gcn_basis_concat import ConcatGcn
from relationprediction_b200.encoders.message_gcns.message_gcn import MessageGcn
from relationprediction_b200.encoders.relation_embedding import RelationEmbedding
from relationprediction_b200.extras.highway_layer import HighwayLayer
from test_plugin_chain_cpu import OracleGraph, oracle_basis_layer, oracle_block_layer, oracle_distmult
from test_plugin_host import merged_settings
from test_reference_golden import KEEP, LAMBDA

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_highway_golden.npz")
DT = torch.float64


def _o(d, B, code=None, **extra):
    o = {"InternalEncoderDimension": str(d), "CodeDimension": str(code or d), "NumberOfBasisFunctions": str(B),
         "SkipConnections": "Highway"}
    o.update(extra)
    return o


# golden case -> (settings file, overrides of the generator, oracle variant, library norm mode)
CASES = {
    "highway_block_toy_tf_kernel": ("gcn_block.exp", _o(20, 4), "block", "tf_unsorted_compat"),
    "highway_block_toy_canonical": ("gcn_block.exp", _o(20, 4), "block", "canonical"),
    "highway_basis_toy_canonical": ("gcn_basis.exp", _o(16, 3), "basis", "canonical"),
    "highway_block_toy_1layer_canonical": ("gcn_block.exp", _o(16, 4, NumberOfLayers="1"), "block", "canonical"),
    "highway_block_toy_3layer_canonical": ("gcn_block.exp", _o(16, 2, NumberOfLayers="3"), "block", "canonical"),
    "highway_block_toy_outproj_canonical": ("gcn_block.exp", _o(20, 4, code=12, UseOutputTransform="Yes"), "block",
                                            "canonical"),
    "highway_block_syn_canonical": ("gcn_block.exp", _o(16, 4), "block", "canonical"),
}
ONEHOT_CASE = "highway_onehot_toy_canonical"       # recorded only to document the reference's dead gate
ONEHOT_SETTINGS = ("gcn_basis.exp", _o(16, 2, UseInputTransform="No"), "onehot", "canonical")


def load_case(name):
    z = np.load(GOLDEN)
    p = name + "/"
    return {k[len(p):]: z[k] for k in z.files if k.startswith(p)}


def case_shape(name):
    settings_file, overrides, variant, norm_mode = ONEHOT_SETTINGS if name == ONEHOT_CASE else CASES[name]
    n_layers = int(overrides.get("NumberOfLayers", "2"))
    outproj = overrides.get("UseOutputTransform") == "Yes"
    return settings_file, overrides, variant, norm_mode, n_layers, outproj


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def ranking(model, known, ranked):
    sc = evaluation.Scorer({'Metric': 'MRR'})
    sc.register_data(known)
    sc.register_data(ranked)
    sc.register_model(model)
    res = sc.compute_scores(ranked).get_summary().results
    return np.array([[float(res[f][k]) for k in ('MRR', 'H@1', 'H@3', 'H@10')] for f in ('Raw', 'Filtered')])


class OracleScores(object):
    def __init__(self, codes, rel_table):
        self.codes, self.rel = codes, rel_table

    def score_all_subjects(self, triplets):
        return oracle.distmult_predict_all_subjects(self.codes, self.rel, triplets, DT).numpy()

    def score_all_objects(self, triplets):
        return oracle.distmult_predict_all_objects(self.codes, self.rel, triplets, DT).numpy()


@pytest.mark.parametrize("name", sorted(CASES) + [ONEHOT_CASE])
def test_oracle_matches_reference_highway_outputs(name):
    c = load_case(name)
    _, _, variant, norm_mode, n_layers, outproj = case_shape(name)
    names = hw.weight_names(variant, n_layers, outproj)
    assert len(names) == int(c["n_weights"])
    leaves = {nm: torch.tensor(c["w%d" % i], dtype=DT, requires_grad=True) for i, nm in enumerate(names)}
    V = int(c["V"])
    masks = [torch.tensor(c["mask%d" % i]) for i in range(int(c["n_masks"]))]
    assert len(masks) == n_layers
    codes = hw.encode(leaves, variant, n_layers, outproj, c["graph_split"], V, "train", masks, KEEP, norm_mode)
    loss, reg, _ = oracle.distmult_loss(codes, leaves["W_relation"], c["X"], c["Y"], DT)
    (loss + LAMBDA * reg).backward()
    assert abs(loss.item() - float(c["loss"])) <= 1e-10 * abs(float(c["loss"]))
    assert abs(LAMBDA * reg.item() - float(c["reg"])) <= 1e-10 * abs(float(c["reg"]))
    for i, nm in enumerate(names):
        if bool(c["g%d_unused" % i]):
            assert nm.endswith(".b") and nm.startswith("L") and leaves[nm].grad is None, nm   # never-added layer bias
            continue
        if variant == "onehot" and nm.startswith("HW"):
            assert float(leaves[nm].grad.abs().max()) == 0.0, nm
            continue
        assert rel(leaves[nm].grad.numpy(), c["g%d" % i]) < 1e-10, nm
    with torch.no_grad():
        tc = hw.encode(leaves, variant, n_layers, outproj, c["test_graph"], V, "test", masks, KEEP, norm_mode)
    Wr, tX = leaves["W_relation"].detach(), c["test_X"]
    e, _ = oracle.distmult_energies(tc, Wr, tX, DT)
    assert rel(torch.sigmoid(e).numpy(), c["predict"]) < 1e-10
    assert rel(oracle.distmult_predict_all_objects(tc, Wr, tX, DT).numpy(), c["all_objects"]) < 1e-10
    assert rel(oracle.distmult_predict_all_subjects(tc, Wr, tX, DT).numpy(), c["all_subjects"]) < 1e-10
    assert np.abs(ranking(OracleScores(tc, Wr), c["test_graph"], c["ranked"]) - c["ranking"]).max() < 1e-12


def test_reference_gate_is_dead_without_an_input_transform():
    """The reference's one-hot + Highway model: the highway weights get exactly zero gradient (they are used, so
    the gradient exists), while the layers' own weights train."""
    c = load_case(ONEHOT_CASE)
    names = hw.weight_names("onehot", 2, False)
    assert names[12:14] == ["HW1.W", "HW1.b"]
    for i in (12, 13):
        assert not bool(c["g%d_unused" % i]) and float(np.abs(c["g%d" % i]).max()) == 0.0
    assert float(np.abs(c["w12"]).max()) > 0.1 and np.all(c["w13"] == 1.0)
    for i in (0, 4, 6, 10, 14):
        assert float(np.abs(c["g%d" % i]).max()) > 1e-3, names[i]


def oracle_highway(c1, c2, W, b):
    return hw.highway(c1, c2, W, b)


@pytest.fixture
def oracle_backed_ops(monkeypatch):
    monkeypatch.setattr(ops, "Graph", OracleGraph)
    monkeypatch.setattr(ops, "block_layer", oracle_block_layer)
    monkeypatch.setattr(ops, "basis_layer", oracle_basis_layer)
    monkeypatch.setattr(ops, "distmult", oracle_distmult)
    monkeypatch.setattr(ops, "highway", oracle_highway)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)


def build_model(toy, name, V, R, E):
    settings_file, overrides, _, norm_mode, _, _ = case_shape(name)
    enc, dec = merged_settings(toy, settings_file, V, R, E)
    for s in (enc, dec):
        for k, v in overrides.items():
            s.put(k, v)
        s.put("NormalizationMode", norm_mode)
    return model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_chain_reproduces_reference_highway_outputs(toy, oracle_backed_ops, name):
    c = load_case(name)
    _, _, variant, norm_mode, n_layers, outproj = case_shape(name)
    model = build_model(toy, name, int(c["V"]), int(c["R"]), len(c["test_graph"]))
    model.set_device("cpu")
    model.initialize_train()
    names = hw.weight_names(variant, n_layers, outproj)
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
    assert len(layers) == n_layers
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
        if bool(c["g%d_unused" % i]):
            assert w.grad is None or float(w.grad.abs().max()) == 0.0, nm
        else:
            assert rel(w.grad.numpy(), c["g%d" % i]) < tol, nm
    model.preprocess(c["test_graph"])
    model.register_for_test(c["test_graph"])
    for got, ref in ((model.score(c["test_X"]), c["predict"]),
                     (model.score_all_objects(c["test_X"]), c["all_objects"]),
                     (model.score_all_subjects(c["test_X"]), c["all_subjects"])):
        assert got.shape == ref.shape and np.abs(np.asarray(got, np.float64) - ref).max() < 100 * tol
    got = ranking(model, c["test_graph"], c["ranked"])
    assert np.abs(got - c["ranking"]).max() < (1e-12 if tol == 1e-10 else 5e-3)


def highway_settings(toy, settings_file="gcn_block.exp", **flags):
    enc, dec = merged_settings(toy, settings_file, toy["V"], toy["R"], len(toy["train"]))
    enc.put("SkipConnections", "Highway")
    for k, v in flags.items():
        enc.put(k, v)
    return enc, dec


def chain_of(model):
    out, c = [], model
    while c is not None:
        out.append(c)
        c = c.next_component
    return out


@pytest.mark.parametrize("settings_file,concat,layer_type", [("gcn_block.exp", "Yes", ConcatGcn),
                                                             ("gcn_basis.exp", "No", BasisGcn)])
def test_factory_wraps_every_layer_and_orders_weights(toy, settings_file, concat, layer_type):
    enc, dec = highway_settings(toy, settings_file, Concatenation=concat)
    model = model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)
    chain = chain_of(model)
    assert [type(c) for c in chain[1:7]] == [RelationEmbedding, HighwayLayer, layer_type, HighwayLayer, layer_type,
                                             AffineTransform]
    emb, hw1, l1, hw0, l0, inp = chain[1:7]
    # the carry input of each highway is the wrapped layer's own input
    assert hw1.next_component is l1 and hw1.next_component_2 is hw0 and l1.next_component is hw0
    assert hw0.next_component is l0 and hw0.next_component_2 is inp and l0.next_component is inp
    assert not l1.use_nonlinearity and l0.use_nonlinearity
    np.random.seed(0)
    model.set_device("cpu")
    model.initialize_train()
    ws = model.get_weights()
    expect = (inp.local_get_weights() + l0.local_get_weights() + hw0.local_get_weights() + l1.local_get_weights()
              + hw1.local_get_weights() + emb.local_get_weights())
    assert len(ws) == len(expect) and all(a is b for a, b in zip(ws, expect))
    d = int(enc["InternalEncoderDimension"])
    assert [tuple(w.shape) for w in hw0.local_get_weights()] == [(d, d), (d,)]


def test_factory_residual_stays_a_no_op_and_one_layer_is_wrapped(toy):
    enc, dec = highway_settings(toy, SkipConnections="Residual")
    model = model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)
    assert not any(isinstance(c, HighwayLayer) for c in chain_of(model))
    enc, dec = highway_settings(toy, NumberOfLayers="1")
    chain = chain_of(model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec))
    assert [type(c) for c in chain[2:5]] == [HighwayLayer, ConcatGcn, AffineTransform]
    assert not chain[3].use_nonlinearity


def test_highway_initialisation_matches_the_reference():
    """W ~ N(0, glorot_variance([d, d]) = 3 / sqrt(2d)) as the std-dev, b = ones (make_tf_bias(init=1)); drawn from the
    global numpy stream before the wrapped layer's weights (local first, then delegate)."""
    d = 500
    np.random.seed(3)
    h = HighwayLayer([d, d])
    h.set_device("cpu")
    h.initialize_train()
    assert abs(float(h.W.detach().std()) / (3 / np.sqrt(2 * d)) - 1) < 0.01
    assert abs(float(h.W.detach().mean())) < 0.01
    assert h.b.dtype == torch.float32 and torch.equal(h.b.detach(), torch.ones(d))
    np.random.seed(3)
    assert np.array_equal(h.W.detach().numpy(), np.random.normal(0, 3 / np.sqrt(2 * d), (d, d)).astype(np.float32))


def test_factory_rejects_highway_without_an_input_transform(toy):
    enc, _ = highway_settings(toy, "gcn_basis.exp", UseInputTransform="No")
    with pytest.raises(NotImplementedError, match="UseInputTransform=No") as e:
        model_builder.build_encoder(enc, toy["train"])
    assert "dead" in str(e.value) and "cache" in str(e.value)
    enc, _ = highway_settings(toy, SkipConnections="Gated")
    with pytest.raises(NotImplementedError):
        model_builder.build_encoder(enc, toy["train"])


def test_checkpoint_round_trips_highway_weights(toy, oracle_backed_ops, tmp_path):
    enc, dec = highway_settings(toy, "gcn_basis.exp", InternalEncoderDimension="16", CodeDimension="16",
                                NumberOfBasisFunctions="2")
    model = model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)
    np.random.seed(1)
    model.set_device("cpu")
    model.initialize_train()
    hws = [c for c in chain_of(model) if isinstance(c, HighwayLayer)]
    assert len(hws) == 2
    with torch.no_grad():
        for i, h in enumerate(hws):
            h.b.add_(0.25 * (i + 1))
    saved = [w.detach().clone() for w in model.get_weights()]
    model.save(str(tmp_path / "ckpt"))
    with torch.no_grad():
        for w in model.get_weights():
            w.zero_()
    model.load(str(tmp_path / "ckpt-0.pt"))
    for a, b in zip(model.get_weights(), saved):
        assert torch.equal(a.detach(), b)
    assert torch.equal(hws[0].b.detach(), torch.full((16,), 1.25))    # hws: top layer first
    assert torch.equal(hws[1].b.detach(), torch.full((16,), 1.5))


def test_highway_entry_points_reject_bad_arguments_without_a_gpu():
    lib = _lib.load()
    buf = ctypes.create_string_buffer(1 << 16)
    assert lib.rgcn_highway_workspace_bytes(-1, 8, 0) == -1
    assert lib.rgcn_highway_workspace_bytes(10, 0, 0) == -1
    need_f = lib.rgcn_highway_workspace_bytes(10, 8, 0)
    need_b = lib.rgcn_highway_workspace_bytes(10, 8, 1)
    assert 2 * 8 * 8 * 4 <= need_f < need_b <= len(buf) and need_b - need_f >= 10 * 8 * 4

    def fwd(V=10, d=8, c1=buf, W=buf, b=buf, out=buf, gate=buf, ws=need_f):
        return lib.rgcn_highway_forward(c1, buf, W, b, V, d, out, gate, buf, ws, None)

    def bwd(V=10, d=8, c1=buf, W=buf, gate=buf, dW=buf, db=buf, ws=need_b):
        return lib.rgcn_highway_backward(c1, buf, W, gate, buf, V, d, buf, buf, dW, db, buf, ws, None)
    for call in (fwd, bwd):
        assert call(V=-1) == -1
        assert call(d=6) == -1 and b"d % 4" in lib.rgcn_last_error()
        assert call(d=0) == -1
        assert call(c1=None) == -1 and b"non-null" in lib.rgcn_last_error()
        assert call(W=None) == -1
        assert call(ws=16) == -4 and b"workspace" in lib.rgcn_last_error()
        assert call(V=0, ws=lib.rgcn_highway_workspace_bytes(0, 8, call is bwd)) == 0   # V = 0: nothing to do
    assert fwd(b=None) == -1 and fwd(out=None) == -1 and fwd(gate=None) == -1
    assert bwd(gate=None) == -1 and bwd(dW=None) == -1 and bwd(db=None) == -1


def test_highway_op_rejects_cpu_tensors():
    V, d = 6, 8
    with pytest.raises(_lib.RgcnError, match="CUDA float32"):
        ops.highway(torch.zeros(V, d), torch.zeros(V, d), torch.zeros(d, d), torch.ones(d))
