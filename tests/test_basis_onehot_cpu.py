"""CPU: the featureless gcn_basis encoder (UseInputTransform=No: layer 0 is BasisGcn with one-hot input) against
golden vectors produced by running the reference's own classes (tests/golden/make_onehot_golden.py over
tests/golden/tf1_shim.py).

  * the oracle chain (float64; the one-hot layer is oracle.basis_gcn_forward with H = I_V, the matmul with a one-hot
    row being the lookup) reproduces loss, regularisation, every weight gradient, the test-mode scores and the
    reference Scorer's raw / filtered MRR and Hits at 1e-10;
  * the host plugin chain (factory, Representation, BasisGcn, RelationEmbedding, BilinearDiag, Scorer) reproduces the
    same outputs with the library calls replaced by the oracle inside this test;
  * the factory builds the reference's chain, weight shapes and initialisation, and still rejects the variants
    outside the accelerated path;
  * the new C-ABI entry points validate their arguments before touching a device."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import rgcn_oracle as oracle
from relationprediction_b200 import _lib, ops
from relationprediction_b200.common import evaluation, model_builder
from relationprediction_b200.encoders.message_gcns.gcn_basis import BasisGcn
from relationprediction_b200.encoders.message_gcns.message_gcn import MessageGcn
from relationprediction_b200.encoders.relation_embedding import RelationEmbedding
from relationprediction_b200.extras.graph_representations import Representation
from test_plugin_chain_cpu import OracleGraph, oracle_basis_layer, oracle_distmult
from test_plugin_host import merged_settings
from test_reference_golden import KEEP, LAMBDA

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_onehot_golden.npz")
DT = torch.float64
LAYER_KEYS = ["W_forward", "W_backward", "C_forward", "C_backward", "W_self", "b"]

# golden case -> (encoder/shared overrides of gcn_basis.exp, library norm mode)
CASES = {
    "onehot_toy_tf_kernel": ({"InternalEncoderDimension": "24", "CodeDimension": "24", "NumberOfBasisFunctions": "5"},
                             "tf_unsorted_compat"),
    "onehot_toy_canonical": ({"InternalEncoderDimension": "24", "CodeDimension": "24", "NumberOfBasisFunctions": "5"},
                             "canonical"),
    "onehot_toy_1layer_canonical": ({"InternalEncoderDimension": "16", "CodeDimension": "16",
                                     "NumberOfBasisFunctions": "2", "NumberOfLayers": "1"}, "canonical"),
    "onehot_syn_canonical": ({"InternalEncoderDimension": "20", "CodeDimension": "20", "NumberOfBasisFunctions": "3"},
                             "canonical"),
    "onehot_toy_outproj_canonical": ({"InternalEncoderDimension": "20", "CodeDimension": "12",
                                      "NumberOfBasisFunctions": "4", "UseOutputTransform": "Yes"}, "canonical"),
}


def load_case(name):
    z = np.load(GOLDEN)
    p = name + "/"
    return {k[len(p):]: z[k] for k in z.files if k.startswith(p)}


def split_weights(c):
    """Reference get_weights() order (deepest first): per layer [W_forward, W_backward, C_forward, C_backward,
    W_self, b], (output AffineTransform [W, b],) RelationEmbedding [W_relation].  No input transform."""
    n = int(c["n_weights"])
    outproj = (n - 1) % 6 == 2
    n_layers = (n - 1 - (2 if outproj else 0)) // 6
    names = ["L%d.%s" % (l, k) for l in range(n_layers) for k in LAYER_KEYS]
    names += (["W_out", "b_out"] if outproj else []) + ["W_relation"]
    assert len(names) == n
    return names, n_layers, outproj


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def oracle_encode(leaves, n_layers, outproj, triples, V, mode, masks, norm_mode):
    """model_builder.py:166-167 + :273-309: Representation -> one-hot BasisGcn -> BasisGcn ... (last layer linear)."""
    nf, nb = oracle.graph_norms(triples, V, norm_mode, np.float64)
    H = torch.eye(V, dtype=DT)                      # one-hot input: H @ W is the lookup of W's rows
    for l in range(n_layers):
        lp = {k: leaves["L%d.%s" % (l, k)] for k in LAYER_KEYS[:-1]}
        train = mode == "train"
        H = oracle.basis_gcn_forward(H, triples, lp["W_forward"], lp["W_backward"], lp["C_forward"],
                                     lp["C_backward"], lp["W_self"], nf, nb, masks[l] if train else None,
                                     KEEP if train else 1.0, l < n_layers - 1, DT)
    if outproj:
        H = H @ leaves["W_out"] + leaves["b_out"]
    return H


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


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_onehot_outputs(name):
    c = load_case(name)
    norm_mode = CASES[name][1]
    names, n_layers, outproj = split_weights(c)
    leaves = {nm: torch.tensor(c["w%d" % i], dtype=DT, requires_grad=True) for i, nm in enumerate(names)}
    V = int(c["V"])
    masks = [torch.tensor(c["mask%d" % i]) for i in range(int(c["n_masks"]))]
    assert len(masks) == n_layers
    assert tuple(leaves["L0.W_forward"].shape)[0] == V and tuple(leaves["L0.W_self"].shape)[0] == V
    codes = oracle_encode(leaves, n_layers, outproj, c["graph_split"], V, "train", masks, norm_mode)
    loss, reg, _ = oracle.distmult_loss(codes, leaves["W_relation"], c["X"], c["Y"], DT)
    (loss + LAMBDA * reg).backward()
    assert abs(loss.item() - float(c["loss"])) <= 1e-10 * abs(float(c["loss"]))
    assert abs(LAMBDA * reg.item() - float(c["reg"])) <= 1e-10 * abs(float(c["reg"]))
    for i, nm in enumerate(names):
        if bool(c["g%d_unused" % i]):
            assert nm.endswith(".b") and leaves[nm].grad is None, nm   # the layer bias is never added
            continue
        assert rel(leaves[nm].grad.numpy(), c["g%d" % i]) < 1e-10, nm
    with torch.no_grad():
        tc = oracle_encode(leaves, n_layers, outproj, c["test_graph"], V, "test", masks, norm_mode)
    Wr, tX = leaves["W_relation"].detach(), c["test_X"]
    e, _ = oracle.distmult_energies(tc, Wr, tX, DT)
    assert rel(torch.sigmoid(e).numpy(), c["predict"]) < 1e-10
    assert rel(oracle.distmult_predict_all_objects(tc, Wr, tX, DT).numpy(), c["all_objects"]) < 1e-10
    assert rel(oracle.distmult_predict_all_subjects(tc, Wr, tX, DT).numpy(), c["all_subjects"]) < 1e-10
    assert np.abs(ranking(OracleScores(tc, Wr), c["test_graph"], c["ranked"]) - c["ranking"]).max() < 1e-12


def oracle_onehot_layer(Wf, Wb, Cf, Cb, Ws, graph, drop_mask=None, keep=1.0, use_nonlinearity=True):
    return oracle.basis_gcn_forward(torch.eye(graph.V_src, dtype=DT), graph.triples, Wf, Wb, Cf, Cb, Ws, graph.nf,
                                    graph.nb, drop_mask, keep, use_nonlinearity, DT)


@pytest.fixture
def oracle_backed_ops(monkeypatch):
    monkeypatch.setattr(ops, "Graph", OracleGraph)
    monkeypatch.setattr(ops, "basis_layer", oracle_basis_layer)
    monkeypatch.setattr(ops, "basis_onehot_layer", oracle_onehot_layer)
    monkeypatch.setattr(ops, "distmult", oracle_distmult)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)


def build_model(toy, c, overrides, norm_mode):
    enc, dec = merged_settings(toy, "gcn_basis.exp", int(c["V"]), int(c["R"]), len(c["test_graph"]))
    for s in (enc, dec):
        for k, v in overrides.items():
            s.put(k, v)
        s.put("UseInputTransform", "No")
        s.put("NormalizationMode", norm_mode)
    return model_builder.build_decoder(model_builder.build_encoder(enc, c["test_graph"]), dec)


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_chain_reproduces_reference_onehot_outputs(toy, oracle_backed_ops, name):
    c = load_case(name)
    overrides, norm_mode = CASES[name]
    model = build_model(toy, c, overrides, norm_mode)
    model.set_device("cpu")
    model.initialize_train()
    names, _, _ = split_weights(c)
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


def onehot_settings(toy, **flags):
    enc, dec = merged_settings(toy, "gcn_basis.exp", toy["V"], toy["R"], len(toy["train"]))
    enc.put("UseInputTransform", "No")
    for k, v in flags.items():
        enc.put(k, v)
    return enc, dec


def test_factory_builds_the_featureless_chain(toy):
    enc, dec = onehot_settings(toy)
    model = model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)
    emb = model.next_component
    top, first = emb.next_component, emb.next_component.next_component
    assert isinstance(emb, RelationEmbedding)
    assert type(top) is BasisGcn and not top.onehot_input and not top.use_nonlinearity
    assert type(first) is BasisGcn and first.onehot_input and first.use_nonlinearity
    assert isinstance(first.next_component, Representation)
    np.random.seed(0)
    model.set_device("cpu")
    model.initialize_train()
    V, R, d, B = toy["V"], toy["R"], 500, 5
    assert [tuple(w.shape) for w in first.local_get_weights()] == [(V, B, d), (V, B, d), (R, B), (R, B), (V, d), (d,)]
    assert [tuple(w.shape) for w in top.local_get_weights()] == [(d, B, d), (d, B, d), (R, B), (R, B), (d, d), (d,)]
    ws = model.get_weights()
    assert ws[:6] == first.local_get_weights() and len(ws) == 6 + 6 + 1
    std = 3 / np.sqrt(V + d)          # glorot_variance([V, d]) of gcn_basis.py:21 with vertex dimension V
    for w in (first.W_forward, first.W_backward, first.W_self):
        assert abs(float(w.detach().std()) / std - 1) < 0.05
    for w in (first.C_forward, first.C_backward):
        assert 0.6 < float(w.detach().std()) < 1.5
    assert float(first.b.detach().abs().max()) == 0.0


@pytest.mark.parametrize("flags", [{"RandomInput": "Yes"}, {"PartiallyRandomInput": "Yes"},
                                   {"Concatenation": "Yes"}, {"AddDiagonal": "Yes"}, {"DiagonalCoefficients": "Yes"},
                                   {"StoreEdgeData": "Yes"}, {"SkipConnections": "Highway"}])
def test_factory_still_rejects_variants_outside_the_accelerated_path(toy, flags):
    enc, _ = onehot_settings(toy, **flags)
    with pytest.raises(NotImplementedError) as e:
        model_builder.build_encoder(enc, toy["train"])
    if "Concatenation" in flags:
        assert "index vector" in str(e.value)


def test_onehot_entry_points_reject_bad_arguments_without_a_gpu(toy):
    lib = _lib.load()
    g = ops.Graph(np.array(toy["train"], np.int32), toy["V"], toy["R"])   # host-only graph
    h, buf = g.handle, ctypes.create_string_buffer(1 << 16)
    assert lib.rgcn_basis_onehot_workspace_bytes(None, 8, 2, 0) == -1
    assert lib.rgcn_basis_onehot_workspace_bytes(h, 0, 2, 0) == -1
    assert lib.rgcn_basis_onehot_workspace_bytes(h, 8, 0, 1) == -1
    need_f = lib.rgcn_basis_onehot_workspace_bytes(h, 8, 2, 0)
    need_b = lib.rgcn_basis_onehot_workspace_bytes(h, 8, 2, 1)
    assert 0 < need_f < need_b <= len(buf)

    def fwd(d=8, B=2, Wf=buf, keep=1.0, out=buf, ws=need_f, graph=h):
        return lib.rgcn_basis_onehot_forward(graph, d, B, Wf, buf, buf, buf, buf, None, keep, 1, out, buf, ws, None)

    def bwd(d=8, B=2, dWf=buf, relu=1, out=buf, ws=need_b, graph=h):
        return lib.rgcn_basis_onehot_backward(graph, d, B, buf, buf, buf, buf, None, 1.0, relu, out, buf, dWf, buf,
                                              buf, buf, buf, buf, ws, None)
    for call in (fwd, bwd):
        assert call(graph=None) == -1
        assert call(d=6) == -1 and b"d % 4" in lib.rgcn_last_error()
        assert call(B=0) == -1
        assert call(ws=16) == -4 and b"workspace" in lib.rgcn_last_error()
        assert call() == -5 and b"host-only" in lib.rgcn_last_error()   # valid arguments: no silent CPU path
    assert fwd(Wf=None) == -1 and b"null" in lib.rgcn_last_error()
    assert fwd(out=None) == -1
    assert fwd(keep=0.0) == -1
    assert bwd(dWf=None) == -1
    assert bwd(out=None) == -1                 # relu' needs the forward output
    assert bwd(out=None, relu=0) == -5


def test_onehot_layer_rejects_cpu_tensors(toy):
    g = ops.Graph(np.array(toy["train"], np.int32), toy["V"], toy["R"])
    V, R, B, d = toy["V"], toy["R"], 2, 8
    w = [torch.zeros(V, B, d), torch.zeros(V, B, d), torch.zeros(R, B), torch.zeros(R, B), torch.zeros(V, d)]
    with pytest.raises(_lib.RgcnError, match="CUDA float32"):
        ops.basis_onehot_layer(*w, g)
