"""CPU: the variational encoders (Encoder Name=variational_embedding / variational_gcn_basis) against golden vectors
produced by running the reference's own classes (tests/golden/make_variational_golden.py over tests/golden/tf1_shim.py).

  * the float64 oracle (tests/variational_oracle.py): its closed-form gradients equal autograd of its forward;
  * the host plugin chain (factory, SplitModel / VariationalEncoding, the trunk layers, RelationEmbedding, BilinearDiag
    / Complex, Scorer) reproduces loss, regularisation, every weight gradient (matched by name: the reference's order
    is a set's order), the test-mode scores and the ranking at 1e-10, with the library calls replaced by oracles and
    the recorded eps draws replayed;
  * the factory's wiring, its fixed weight order, its rejections and the initialisation of the shared trunk;
  * checkpoints round-trip the head's weights;
  * the C-ABI entry points validate their arguments before touching a device."""
import ctypes
import os

import numpy as np
import pytest
import torch

import highway_oracle as hw
import variational_oracle as vo
from relationprediction_b200 import _lib, ops
from relationprediction_b200.common import model_builder
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag
from relationprediction_b200.decoders.complex import Complex
from relationprediction_b200.encoders.affine_transform import AffineTransform
from relationprediction_b200.encoders.message_gcns.gcn_basis import BasisGcn
from relationprediction_b200.encoders.message_gcns.message_gcn import MessageGcn
from relationprediction_b200.encoders.relation_embedding import RelationEmbedding
from relationprediction_b200.extras.variational_encoding import VariationalEncoding
from test_basis_onehot_cpu import oracle_onehot_layer
from test_complex_cpu import oracle_complex
from test_highway_cpu import ranking, rel
from test_plugin_chain_cpu import OracleGraph, oracle_basis_layer, oracle_block_layer, oracle_distmult
from test_plugin_host import merged_settings
from test_times_diag_cpu import oracle_times_diag_layer

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_variational_golden.npz")
DT = torch.float64
VE, VG = "variational_embedding", "variational_gcn_basis"


def _g(d, **extra):
    o = {"Name": VG, "InternalEncoderDimension": str(d), "CodeDimension": str(d), "NumberOfBasisFunctions": "3"}
    o.update(extra)
    return o


# golden case -> (settings file, encoder overrides of the generator, decoder name, library norm mode)
CASES = {
    "var_emb_toy_tf_kernel": ("distmult.exp", {"Name": VE, "CodeDimension": "16"}, None, "tf_unsorted_compat"),
    "var_emb_toy_canonical": ("distmult.exp", {"Name": VE, "CodeDimension": "16"}, None, "canonical"),
    "var_gcn_toy_tf_kernel": ("gcn_basis.exp", _g(16), None, "tf_unsorted_compat"),
    "var_gcn_toy_canonical": ("gcn_basis.exp", _g(16), None, "canonical"),
    "var_gcn_toy_1layer_canonical": ("gcn_basis.exp", _g(12, NumberOfLayers="1"), None, "canonical"),
    "var_gcn_toy_3layer_canonical": ("gcn_basis.exp", _g(12, NumberOfLayers="3"), None, "canonical"),
    "var_gcn_toy_onehot_canonical": ("gcn_basis.exp", _g(16, UseInputTransform="No"), None, "canonical"),
    "var_gcn_toy_outproj_canonical": ("gcn_basis.exp", _g(16, UseOutputTransform="Yes"), None, "canonical"),
    "var_gcn_syn_canonical": ("gcn_basis.exp", _g(20), None, "canonical"),
    "var_gcn_toy_diagcoef_canonical": ("gcn_basis.exp", _g(16, DiagonalCoefficients="Yes"), None, "canonical"),
    "var_gcn_toy_highway_canonical": ("gcn_basis.exp", _g(16, SkipConnections="Highway"), None, "canonical"),
    "var_gcn_block_toy_canonical": ("gcn_block.exp", _g(16, NumberOfBasisFunctions="4"), None, "canonical"),
    "var_gcn_complex_toy_canonical": ("gcn_basis.exp", _g(16), "complex", "canonical"),
}


def load_case(name):
    z = np.load(GOLDEN)
    p = name + "/"
    return {k[len(p):]: z[k] for k in z.files if k.startswith(p)}


def settings(toy, settings_file, overrides, decoder=None, V=None, R=None, E=None):
    enc, dec = merged_settings(toy, settings_file, V or toy["V"], R or toy["R"], E or len(toy["train"]))
    for k, v in overrides.items():
        enc.put(k, v)
        if k in ("CodeDimension", "NormalizationMode"):
            dec.put(k, v)
    if decoder:
        dec.put("Name", decoder)
    return enc, dec


def build(enc, triples, dec):
    return model_builder.build_decoder(model_builder.build_encoder(enc, triples), dec)


def chain_of(model):
    out = []
    while model is not None:
        out.append(model)
        model = model.next_component
    return out


def oracle_variational(H, W_mu, b_mu, W_sigma, b_sigma, eps):
    return vo.variational(H, W_mu, b_mu, W_sigma, b_sigma, eps)


@pytest.fixture
def oracle_backed_ops(monkeypatch):
    monkeypatch.setattr(ops, "Graph", OracleGraph)
    monkeypatch.setattr(ops, "basis_layer", oracle_basis_layer)
    monkeypatch.setattr(ops, "basis_onehot_layer", oracle_onehot_layer)
    monkeypatch.setattr(ops, "block_layer", oracle_block_layer)
    monkeypatch.setattr(ops, "basis_diagcoef_layer", oracle_times_diag_layer)
    monkeypatch.setattr(ops, "highway", hw.highway)
    monkeypatch.setattr(ops, "distmult", oracle_distmult)
    monkeypatch.setattr(ops, "complex_score", oracle_complex)
    monkeypatch.setattr(ops, "variational", oracle_variational)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)


@pytest.mark.parametrize("with_h", [False, True], ids=["embedding", "gcn"])
def test_oracle_gradients_are_the_closed_forms(with_h):
    gen = torch.Generator().manual_seed(3)
    V, d, w = 7, 5, 6
    r = lambda *s: torch.randn(*s, generator=gen, dtype=DT)
    H = r(V, d).requires_grad_(True) if with_h else None
    Wm, Ws = (r(d, w) if with_h else r(V, w)).requires_grad_(True), (0.3 * r(d if with_h else V, w)).requires_grad_(True)
    bm, bs = r(w).requires_grad_(True), r(w).requires_grad_(True)
    eps, dz = r(V, w), r(V, w)
    z, kl = vo.variational(H, Wm, bm, Ws, bs, eps)
    (torch.sum(z * dz) + 0.37 * kl).backward()
    got = vo.gradients(H, Wm, bm, Ws, bs, eps, dz, 0.37)
    for g, leaf in zip(got, (H, Wm, bm, Ws, bs)):
        if g is None:
            assert leaf is None or leaf.grad is None
        else:
            assert rel(g.detach().numpy(), leaf.grad.numpy()) < 1e-12


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_chain_reproduces_reference_variational_outputs(toy, oracle_backed_ops, name):
    c = load_case(name)
    settings_file, overrides, decoder, norm_mode = CASES[name]
    enc, dec = settings(toy, settings_file, dict(overrides, NormalizationMode=norm_mode), decoder, int(c["V"]),
                        int(c["R"]), len(c["test_graph"]))
    model = build(enc, toy["train"], dec)
    assert isinstance(model, Complex if decoder == "complex" else BilinearDiag)
    model.set_device("cpu")
    model.initialize_train()
    ws = model.get_weights()
    names = vo.weight_names(model)
    golden_names = [str(s) for s in c["w_names"]]
    assert sorted(names) == sorted(golden_names) and len(set(names)) == len(names)
    index = {nm: i for i, nm in enumerate(golden_names)}
    for nm, w in zip(names, ws):
        i = index[nm]
        assert tuple(w.shape) == c["w%d" % i].shape, nm
        w.data = torch.tensor(c["w%d" % i], dtype=DT)
    layers = [comp for comp in chain_of(model) if isinstance(comp, MessageGcn)]
    assert len(layers) == int(c["n_masks"])
    for layer, i in zip(layers[::-1], range(int(c["n_masks"]))):   # masks in the order drawn: layer 0 first
        m = torch.tensor(c["mask%d" % i])
        layer.make_drop_mask = (lambda rows, mode, m=m, k=layer.dropout_keep_probability:
                                (m, k) if mode == 'train' else (None, 1.0))
    head = [comp for comp in chain_of(model) if isinstance(comp, VariationalEncoding)]
    assert len(head) == 1
    draws = []
    head[0].draw_epsilon = lambda mode: (draws.append(mode),
                                         torch.tensor(c["eps0" if len(draws) == 1 else "eps1"], dtype=DT))[1]
    feed = (c["graph_split"], c["X"], c["Y"]) if model.needs_graph() else (c["X"], c["Y"])
    total = model.train_loss(*feed)
    total.backward()
    assert draws == ["train"]
    ref_total = float(c["loss"]) + float(c["reg"])
    tol = 1e-10 if norm_mode == "canonical" else 1e-6   # tf_unsorted_compat norms travel as float32
    assert abs(total.item() - ref_total) <= tol * abs(ref_total)
    for nm, w in zip(names, ws):
        i = index[nm]
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
    assert set(draws[1:]) == {"test"}                       # a fresh draw for every test-mode evaluation


def test_embedding_biases_are_listed_but_unused():
    c = load_case("var_emb_toy_canonical")
    names = [str(s) for s in c["w_names"]]
    for i, nm in enumerate(names):
        assert bool(c["g%d_unused" % i]) == nm.endswith("AffineTransform#1"), nm


def test_factory_wiring_and_fixed_weight_order(toy):
    enc, dec = settings(toy, "distmult.exp", {"Name": VE, "CodeDimension": "8"})
    model = build(enc, toy["train"], dec)
    head = chain_of(model)[2]
    assert [type(c) for c in chain_of(model)] == [BilinearDiag, RelationEmbedding, VariationalEncoding,
                                                   AffineTransform]
    assert not model.needs_graph()
    mu, sigma = head.mu_network, head.sigma_network
    for b in (mu, sigma):
        assert b.onehot_input and not b.use_bias and not b.use_nonlinearity and b.shape == [toy["V"], 8]
    model.set_device("cpu")
    model.initialize_train()
    assert [id(w) for w in model.get_weights()] == [id(w) for w in (mu.W, mu.b, sigma.W, sigma.b,
                                                                     chain_of(model)[1].W_relation)]
    assert [p.name for p in model.get_train_input_variables()] == ['X', 'Y']

    enc, dec = settings(toy, "gcn_basis.exp", _g(8, UseOutputTransform="Yes"))
    model = build(enc, toy["train"], dec)
    ch = chain_of(model)
    assert [type(c) for c in ch[:4]] == [BilinearDiag, RelationEmbedding, AffineTransform, VariationalEncoding]
    head, out = ch[3], ch[2]
    mu, sigma = head.mu_network, head.sigma_network
    assert mu.next_component is sigma.next_component and isinstance(mu.next_component, BasisGcn)
    for b in (mu, sigma):
        assert not b.onehot_input and b.use_bias and not b.use_nonlinearity and b.shape == [8, 8]
    assert head.shape == [toy["V"], 8] and model.needs_graph()
    model.set_device("cpu")
    model.initialize_train()
    trunk = []
    comp = mu.next_component
    while comp is not None:
        trunk.append(comp)
        comp = comp.next_component
    expect = [w for c in reversed(trunk) for w in c.local_get_weights()]
    expect += [mu.W, mu.b, sigma.W, sigma.b, out.W, out.b, ch[1].W_relation]
    assert [id(w) for w in model.get_weights()] == [id(w) for w in expect]
    assert [p.name for p in model.get_train_input_variables()] == ['graph_edges', 'X', 'Y']
    assert str(model.get_device()) == "cpu" and all(str(c.get_device()) == "cpu" for c in trunk + [sigma])


def test_shared_trunk_is_initialised_once(toy, monkeypatch):
    calls = []
    base = AffineTransform.local_initialize_train
    monkeypatch.setattr(AffineTransform, "local_initialize_train",
                        lambda self: (calls.append(id(self)), base(self))[1])
    enc, dec = settings(toy, "gcn_basis.exp", _g(500))
    model = build(enc, toy["train"], dec)
    np.random.seed(2)
    model.set_device("cpu")
    model.initialize_train()
    assert len(calls) == len(set(calls)) == 3          # input transform, mu head, sigma head
    head = chain_of(model)[2]
    for W in (head.mu_network.W, head.sigma_network.W):
        assert abs(float(W.detach().std()) / (3 / np.sqrt(1000)) - 1) < 0.01   # glorot_variance([d, d]) as a std-dev
    assert not torch.equal(head.mu_network.W, head.sigma_network.W)
    assert float(head.mu_network.b.detach().abs().max()) == 0.0


@pytest.mark.parametrize("flags, match", [
    ({"CodeDimension": "12"}, "CodeDimension == InternalEncoderDimension"),
    ({"UseInputTransform": "No", "RandomInput": "Yes"}, "graph object"),
    ({"UseInputTransform": "No", "PartiallyRandomInput": "Yes"}, "graph object"),
    ({"AddDiagonal": "Yes"}, "AddDiagonal"),
    ({"StoreEdgeData": "Yes"}, "StoreEdgeData"),
    ({"UseInputTransform": "No", "DiagonalCoefficients": "Yes"}, "DiagonalCoefficients"),
    ({"UseInputTransform": "No", "SkipConnections": "Highway"}, "Highway"),
], ids=["code-dim", "random-input", "partially-random", "add-diagonal", "store-edge-data", "onehot-diagcoef",
        "onehot-highway"])
def test_factory_rejections(toy, flags, match):
    enc, dec = settings(toy, "gcn_basis.exp", dict(_g(16), **flags))
    with pytest.raises((ValueError, NotImplementedError), match=match):
        model_builder.build_encoder(enc, toy["train"])


def test_random_input_with_an_input_transform_is_ignored(toy):
    enc, dec = settings(toy, "gcn_basis.exp", _g(16, RandomInput="Yes"))   # the branch never reads it (:206-214)
    assert isinstance(chain_of(build(enc, toy["train"], dec))[2], VariationalEncoding)


def test_other_branch_shapes_raise():
    s = {"EntityCount": "6", "RelationCount": "2", "EdgeCount": "4"}
    one = AffineTransform([6, 4], s, onehot_input=True, use_bias=False)
    trunk = AffineTransform([6, 4], s, onehot_input=True)
    feat = AffineTransform([4, 4], s, next_component=trunk)
    other = AffineTransform([4, 4], s, next_component=AffineTransform([6, 4], s, onehot_input=True))
    with pytest.raises(NotImplementedError):
        VariationalEncoding([6, 4], s, mu_network=one, sigma_network=feat)
    with pytest.raises(NotImplementedError):
        VariationalEncoding([6, 4], s, mu_network=feat, sigma_network=other)
    with pytest.raises(NotImplementedError):
        VariationalEncoding([6, 4], s, mu_network=AffineTransform([6, 4], s, onehot_input=True, use_nonlinearity=True,
                                                                  use_bias=False), sigma_network=one)
    VariationalEncoding([6, 4], s, mu_network=feat, sigma_network=AffineTransform([4, 4], s, next_component=trunk))


def test_checkpoint_round_trips_the_head(toy, tmp_path):
    enc, dec = settings(toy, "gcn_basis.exp", _g(16))
    model = build(enc, toy["train"], dec)
    np.random.seed(1)
    model.set_device("cpu")
    model.initialize_train()
    head = chain_of(model)[2]
    with torch.no_grad():
        head.sigma_network.b.add_(0.25)
    saved = [w.detach().clone() for w in model.get_weights()]
    model.save(str(tmp_path / "ckpt"))
    with torch.no_grad():
        for w in model.get_weights():
            w.zero_()
    model.load(str(tmp_path / "ckpt-0.pt"))
    for a, b in zip(model.get_weights(), saved):
        assert torch.equal(a.detach(), b)
    assert torch.equal(head.sigma_network.b.detach(), torch.full((16,), 0.25))


def test_variational_entry_points_reject_bad_arguments_without_a_gpu():
    lib = _lib.load()
    buf = ctypes.create_string_buffer(1 << 20)
    V, d, w = 10, 8, 8
    assert lib.rgcn_variational_workspace_bytes(V, d, 6, 0) == -1 and b"w % 4" in lib.rgcn_last_error()
    assert lib.rgcn_variational_workspace_bytes(V, 6, w, 0) == -1
    assert lib.rgcn_variational_workspace_bytes(-1, d, w, 0) == -1
    assert lib.rgcn_variational_workspace_bytes(V, d, 0, 0) == -1
    need = {(dd, b): lib.rgcn_variational_workspace_bytes(V, dd, w, b) for dd in (0, d) for b in (0, 1)}
    assert all(0 < n <= len(buf) for n in need.values())
    assert need[(d, 1)] >= V * 2 * w * 4 + 2 * d * 2 * w * 4 and need[(d, 0)] >= 2 * d * 2 * w * 4

    def fwd(H=buf, d=d, w=w, Wm=buf, b=buf, z=buf, P=buf, kl=buf, ws=None):
        return lib.rgcn_variational_forward(H, V, d, w, Wm, b, buf, b, buf, z, P, kl, buf,
                                            need[(d if d in (0, 8) else 8, 0)] if ws is None else ws, None)

    def bwd(H=buf, d=d, w=w, P=buf, g=buf, dH=buf, db=buf, dWm=buf, ws=None):
        return lib.rgcn_variational_backward(H, V, d, w, buf, buf, P, buf, buf, g, dH, dWm, db, buf, db, buf,
                                             need[(d if d in (0, 8) else 8, 1)] if ws is None else ws, None)
    for call in (fwd, bwd):
        assert call(w=6) == -1 and b"w % 4" in lib.rgcn_last_error()
        assert call(d=6) == -1
        assert call(H=None) == -1 and b"NULL" in lib.rgcn_last_error()    # H NULL with d != 0
        assert call(d=0) == -1                                              # d == 0 with H given
        assert call(ws=16) == -4 and b"workspace" in lib.rgcn_last_error()
        assert call(H=None, d=0, ws=16) == -4                               # the embedding variant's own size
    assert fwd(P=None) == -1 and fwd(kl=None) == -1 and fwd(z=None) == -1 and fwd(b=None) == -1
    assert fwd(H=None, d=0, P=None, b=None, ws=16) == -4                   # P and the biases are gcn-only
    assert bwd(g=None) == -1 and bwd(dH=None) == -1 and bwd(db=None) == -1 and bwd(P=None) == -1
    assert bwd(H=None, d=0, P=None, dH=None, db=None, ws=16) == -4
    assert bwd(H=None, d=0, dWm=None) == -1


def test_variational_op_rejects_cpu_tensors():
    with pytest.raises(_lib.RgcnError, match="CUDA float32"):
        ops.variational(None, torch.zeros(6, 4), None, torch.zeros(6, 4), None, torch.zeros(6, 4))
