"""CPU: the diagonal R-GCN encoder (Encoder Name=gcn_diag) against golden vectors produced by running the reference's
own classes (tests/golden/make_gcn_diag_golden.py over tests/golden/tf1_shim.py).

  * the oracle chain (tests/gcn_diag_oracle.py, float64) reproduces loss, regularisation, every weight gradient, the
    test-mode scores and the reference Scorer's raw / filtered MRR and Hits at 1e-10;
  * the host plugin chain (factory, AffineTransform, DiagGcn, RelationEmbedding, BilinearDiag / Complex, Scorer)
    reproduces the same outputs with the library calls replaced by the oracle inside this test;
  * the factory builds the reference's chain, orders and initialises the weights like it, and ignores the flags the
    reference branch never reads;
  * checkpoints round-trip the layer's weights;
  * the new C-ABI entry points validate their arguments before touching a device."""
import ctypes
import os

import numpy as np
import pytest
import torch

import complex_oracle
import gcn_diag_oracle as gd
from oracle import rgcn_oracle as oracle
from relationprediction_b200 import _lib, ops
from relationprediction_b200.common import model_builder
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag
from relationprediction_b200.decoders.complex import Complex
from relationprediction_b200.encoders.affine_transform import AffineTransform
from relationprediction_b200.encoders.message_gcns.gcn_diag import DiagGcn
from relationprediction_b200.encoders.message_gcns.message_gcn import MessageGcn
from relationprediction_b200.encoders.relation_embedding import RelationEmbedding
from test_complex_cpu import oracle_complex
from test_highway_cpu import chain_of, ranking, rel
from test_plugin_chain_cpu import OracleGraph, oracle_distmult
from test_plugin_host import merged_settings
from test_reference_golden import KEEP, LAMBDA

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_gcn_diag_golden.npz")
DT = torch.float64
IGNORED = {"UseInputTransform": "No", "SkipConnections": "Highway", "Concatenation": "Yes",
           "DiagonalCoefficients": "Yes"}


def _o(d, code=None, **extra):
    o = {"Name": "gcn_diag", "InternalEncoderDimension": str(d), "CodeDimension": str(code or d)}
    o.update(extra)
    return o


# golden case -> (encoder overrides of the generator on gcn_basis.exp, decoder name, library norm mode)
CASES = {
    "gcn_diag_toy_tf_kernel": (_o(16), "bilinear-diag", "tf_unsorted_compat"),
    "gcn_diag_toy_canonical": (_o(16), "bilinear-diag", "canonical"),
    "gcn_diag_toy_1layer_canonical": (_o(12, NumberOfLayers="1"), "bilinear-diag", "canonical"),
    "gcn_diag_toy_3layer_canonical": (_o(12, NumberOfLayers="3"), "bilinear-diag", "canonical"),
    "gcn_diag_toy_outproj_canonical": (_o(16, code=12, UseOutputTransform="Yes"), "bilinear-diag", "canonical"),
    "gcn_diag_syn_canonical": (_o(20), "bilinear-diag", "canonical"),
    "gcn_diag_complex_toy_canonical": (_o(16), "complex", "canonical"),
    "gcn_diag_ignored_flags_toy_canonical": (_o(16, **IGNORED), "bilinear-diag", "canonical"),
}


def load_case(name):
    z = np.load(GOLDEN)
    p = name + "/"
    return {k[len(p):]: z[k] for k in z.files if k.startswith(p)}


def case_shape(name):
    overrides, decoder, norm_mode = CASES[name]
    return overrides, decoder, norm_mode, int(overrides.get("NumberOfLayers", "2")), \
        overrides.get("UseOutputTransform") == "Yes"


def decoder_fns(decoder):
    """(loss, energies, all objects, all subjects) of the oracle decoder"""
    if decoder == "complex":
        return (complex_oracle.complex_loss, complex_oracle.complex_energies,
                complex_oracle.complex_predict_all_objects, complex_oracle.complex_predict_all_subjects)
    return (oracle.distmult_loss, oracle.distmult_energies, oracle.distmult_predict_all_objects,
            oracle.distmult_predict_all_subjects)


class OracleScores(object):
    def __init__(self, codes, rel_table, decoder):
        self.codes, self.rel = codes, rel_table
        _, _, self.objects, self.subjects = decoder_fns(decoder)

    def score_all_subjects(self, triplets):
        return self.subjects(self.codes, self.rel, triplets, DT).numpy()

    def score_all_objects(self, triplets):
        return self.objects(self.codes, self.rel, triplets, DT).numpy()


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_gcn_diag_outputs(name):
    c = load_case(name)
    _, decoder, norm_mode, n_layers, outproj = case_shape(name)
    loss_fn, energies_fn, objects_fn, subjects_fn = decoder_fns(decoder)
    names = gd.weight_names(n_layers, outproj)
    assert len(names) == int(c["n_weights"])
    leaves = {nm: torch.tensor(c["w%d" % i], dtype=DT, requires_grad=True) for i, nm in enumerate(names)}
    V = int(c["V"])
    masks = [torch.tensor(c["mask%d" % i]) for i in range(int(c["n_masks"]))]
    assert len(masks) == n_layers
    codes = gd.encode(leaves, n_layers, outproj, c["graph_split"], V, "train", masks, KEEP, norm_mode)
    loss, reg, _ = loss_fn(codes, leaves["W_relation"], c["X"], c["Y"], DT)
    (loss + LAMBDA * reg).backward()
    assert abs(loss.item() - float(c["loss"])) <= 1e-10 * abs(float(c["loss"]))
    assert abs(LAMBDA * reg.item() - float(c["reg"])) <= 1e-10 * abs(float(c["reg"]))
    for i, nm in enumerate(names):
        assert not bool(c["g%d_unused" % i]), nm        # the layer's bias is added: every weight has a gradient
        assert rel(leaves[nm].grad.numpy(), c["g%d" % i]) < 1e-10, nm
    with torch.no_grad():
        tc = gd.encode(leaves, n_layers, outproj, c["test_graph"], V, "test", masks, KEEP, norm_mode)
    Wr, tX = leaves["W_relation"].detach(), c["test_X"]
    e, _ = energies_fn(tc, Wr, tX, DT)
    assert rel(torch.sigmoid(e).numpy(), c["predict"]) < 1e-10
    assert rel(objects_fn(tc, Wr, tX, DT).numpy(), c["all_objects"]) < 1e-10
    assert rel(subjects_fn(tc, Wr, tX, DT).numpy(), c["all_subjects"]) < 1e-10
    assert np.abs(ranking(OracleScores(tc, Wr, decoder), c["test_graph"], c["ranked"]) - c["ranking"]).max() < 1e-12


def test_ignored_flags_leave_the_reference_chain_unchanged():
    """The reference branch reads none of the flags: the fixture's weights have the plain chain's shapes and order,
    and the oracle of the plain chain reproduces it (checked above); the first layer still gets the input transform."""
    c = load_case("gcn_diag_ignored_flags_toy_canonical")
    plain = load_case("gcn_diag_toy_canonical")
    assert int(c["n_weights"]) == int(plain["n_weights"]) == len(gd.weight_names(2, False))
    for i in range(int(c["n_weights"])):
        assert c["w%d" % i].shape == plain["w%d" % i].shape
    assert c["w0"].shape == (int(c["V"]), 16)     # the input AffineTransform exists despite UseInputTransform=No


def test_layer_bias_gets_the_row_sum_of_the_output_gradient():
    """b is added (gcn_diag.py:50): for the last (linear) layer its gradient is the column sum of the output gradient."""
    c = load_case("gcn_diag_toy_1layer_canonical")
    names = gd.weight_names(1, False)
    i = names.index("L0.b")
    assert float(np.abs(c["g%d" % i]).max()) > 1e-4
    leaves = {nm: torch.tensor(c["w%d" % k], dtype=DT, requires_grad=True) for k, nm in enumerate(names)}
    codes = gd.encode(leaves, 1, False, c["graph_split"], int(c["V"]), "train", [torch.tensor(c["mask0"])], KEEP,
                      "canonical")
    codes.retain_grad()
    loss, reg, _ = oracle.distmult_loss(codes, leaves["W_relation"], c["X"], c["Y"], DT)
    (loss + LAMBDA * reg).backward()
    assert rel(codes.grad.sum(0).numpy(), c["g%d" % i]) < 1e-10


def oracle_diag_layer(H, Df, Db, Ws, b, graph, drop_mask=None, keep=1.0, relu=True):
    return gd.diag_forward(H, graph.triples, Df, Db, Ws, b, graph.nf, graph.nb, drop_mask, keep, relu, DT)


@pytest.fixture
def oracle_backed_ops(monkeypatch):
    monkeypatch.setattr(ops, "Graph", OracleGraph)
    monkeypatch.setattr(ops, "diag_layer", oracle_diag_layer)
    monkeypatch.setattr(ops, "distmult", oracle_distmult)
    monkeypatch.setattr(ops, "complex_score", oracle_complex)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)


def diag_settings(toy, V=None, R=None, E=None, decoder=None, **enc_overrides):
    enc, dec = merged_settings(toy, "gcn_basis.exp", V or toy["V"], R or toy["R"], E or len(toy["train"]))
    enc.put("Name", "gcn_diag")
    for k, v in enc_overrides.items():
        enc.put(k, v)
        if k == "CodeDimension":
            dec.put(k, v)
    if decoder:
        dec.put("Name", decoder)
    return enc, dec


def build_model(toy, name, V, R, E):
    overrides, decoder, norm_mode, _, _ = case_shape(name)
    over = {k: v for k, v in overrides.items() if k != "Name"}
    enc, dec = diag_settings(toy, V, R, E, decoder=decoder, NormalizationMode=norm_mode, **over)
    dec.put("NormalizationMode", norm_mode)
    return model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_chain_reproduces_reference_gcn_diag_outputs(toy, oracle_backed_ops, name):
    c = load_case(name)
    _, decoder, norm_mode, n_layers, outproj = case_shape(name)
    model = build_model(toy, name, int(c["V"]), int(c["R"]), len(c["test_graph"]))
    assert isinstance(model, Complex if decoder == "complex" else BilinearDiag)
    model.set_device("cpu")
    model.initialize_train()
    names = gd.weight_names(n_layers, outproj)
    ws = model.get_weights()
    assert len(ws) == len(names)
    for i, w in enumerate(ws):
        assert tuple(w.shape) == c["w%d" % i].shape, names[i]
        w.data = torch.tensor(c["w%d" % i], dtype=DT)
    layers = [comp for comp in chain_of(model) if isinstance(comp, MessageGcn)]
    assert len(layers) == n_layers and all(isinstance(l, DiagGcn) for l in layers)
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


@pytest.mark.parametrize("flags", [{}, IGNORED, {"AddDiagonal": "Yes"}, {"StoreEdgeData": "Yes"},
                                   {"RandomInput": "Yes"}, {"SkipConnections": "Residual"}],
                         ids=["plain", "ignored", "AddDiagonal", "StoreEdgeData", "RandomInput", "Residual"])
def test_factory_builds_the_reference_chain_and_ignores_unread_flags(toy, flags):
    enc, dec = diag_settings(toy, **flags)
    model = model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)
    chain = chain_of(model)
    assert [type(c) for c in chain[1:5]] == [RelationEmbedding, DiagGcn, DiagGcn, AffineTransform]
    assert not chain[2].use_nonlinearity and chain[3].use_nonlinearity
    assert not chain[2].onehot_input and not chain[3].onehot_input
    inp = chain[4]
    assert inp.onehot_input and inp.use_bias and inp.use_nonlinearity     # model_builder.py:89-94
    assert chain[5].__class__.__name__ == "Representation"
    enc, dec = diag_settings(toy, UseOutputTransform="Yes", CodeDimension="12", InternalEncoderDimension="16")
    chain = chain_of(model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec))
    assert [type(c) for c in chain[1:4]] == [RelationEmbedding, AffineTransform, DiagGcn]
    assert chain[2].shape == [16, 12] and chain[2].use_bias and not chain[2].use_nonlinearity
    with pytest.raises(NotImplementedError, match="feature input"):
        DiagGcn([8, 8], {"DropoutKeepProbability": "1"}, onehot_input=True)


def test_weight_shapes_order_and_initialisation(toy):
    enc, dec = diag_settings(toy, InternalEncoderDimension="500", CodeDimension="500")
    model = model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)
    np.random.seed(5)
    model.set_device("cpu")
    model.initialize_train()
    top, first = chain_of(model)[2], chain_of(model)[3]
    d, R = 500, toy["R"]
    assert [tuple(w.shape) for w in first.local_get_weights()] == [(R, d), (R, d), (d, d), (d,)]
    assert first.local_get_weights()[0] is first.D_types_forward and first.local_get_weights()[2] is first.W_self
    ws = model.get_weights()
    expect = chain_of(model)[4].local_get_weights() + first.local_get_weights() + top.local_get_weights()
    assert all(a is b for a, b in zip(ws, expect)) and len(ws) == len(expect) + 1
    std = 3 / np.sqrt(2 * d)             # glorot_variance([d, d]) as a std-dev (:17-18)
    w = first.W_self.detach()
    assert abs(float(w.std()) / std - 1) < 0.01 and abs(float(w.mean())) < 0.01 * std
    both = torch.cat([first.D_types_forward.detach().flatten(), first.D_types_backward.detach().flatten(),
                      top.D_types_forward.detach().flatten(), top.D_types_backward.detach().flatten()])
    assert abs(float(both.std()) - 1) < 0.03 and abs(float(both.mean())) < 0.03     # N(0, 1) (:20-22)
    assert float(first.b.detach().abs().max()) == 0.0 and first.b.requires_grad
    assert first.local_get_regularization() == 0.0


def test_checkpoint_round_trips_gcn_diag_weights(toy, oracle_backed_ops, tmp_path):
    enc, dec = diag_settings(toy, InternalEncoderDimension="16", CodeDimension="16")
    model = model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)
    np.random.seed(1)
    model.set_device("cpu")
    model.initialize_train()
    layers = [c for c in chain_of(model) if isinstance(c, DiagGcn)]
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
    assert layers[0].D_types_forward.shape == (toy["R"], 16)


def test_gcn_diag_entry_points_reject_bad_arguments_without_a_gpu(toy):
    lib = _lib.load()
    g = ops.Graph(np.array(toy["train"], np.int32), toy["V"], toy["R"])   # host-only graph
    d = 8
    buf = ctypes.create_string_buffer(1 << 20)
    assert lib.rgcn_diag_workspace_bytes(None, d, 0) == -1
    assert lib.rgcn_diag_workspace_bytes(g.handle, 0, 0) == -1
    need_f = lib.rgcn_diag_workspace_bytes(g.handle, d, 0)
    need_b = lib.rgcn_diag_workspace_bytes(g.handle, d, 1)
    assert 0 < need_f < need_b <= len(buf)
    assert need_f >= 2 * d * d * 4 and need_b - need_f >= 2 * toy["V"] * d * 4 - 4096

    def fwd(gh=g.handle, d=d, H=buf, Df=buf, b=buf, out=buf, keep=1.0, ws=need_f):
        return lib.rgcn_diag_forward(gh, d, H, Df, buf, buf, b, None, keep, 1, out, buf, ws, None)

    def bwd(gh=g.handle, d=d, H=buf, out=buf, dDf=buf, db=buf, keep=1.0, relu=1, ws=need_b):
        return lib.rgcn_diag_backward(gh, d, H, buf, buf, buf, None, keep, relu, out, buf, buf, dDf, buf, buf, db,
                                      None, buf, ws, None)
    for call in (fwd, bwd):
        assert call(gh=None) == -1
        assert call(d=6) == -1 and b"d % 4" in lib.rgcn_last_error()
        assert call(d=0) == -1
        assert call(H=None) == -1 and b"null pointer" in lib.rgcn_last_error()
        assert call(keep=0.0) == -1 and call(keep=-1.0) == -1
        assert call(ws=16) == -4 and b"workspace" in lib.rgcn_last_error()
        assert call() == -5 and b"host-only" in lib.rgcn_last_error()     # valid arguments, host-only graph
    assert fwd(Df=None) == -1 and fwd(b=None) == -1 and fwd(out=None) == -1
    assert bwd(db=None) == -1 and bwd(dDf=None) == -1 and bwd(out=None) == -1
    assert bwd(out=None, relu=0) == -5     # out is only read for the ReLU gradient


def test_diag_op_rejects_cpu_tensors():
    class FakeGraph(object):
        V_dst = V_src = 6
        n_relw = 4
        handle = None
    d, R = 8, 2
    with pytest.raises(_lib.RgcnError, match="CUDA float32"):
        ops.diag_layer(torch.zeros(6, d), torch.zeros(R, d), torch.zeros(R, d), torch.zeros(d, d), torch.zeros(d),
                       FakeGraph())
