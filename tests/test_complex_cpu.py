"""CPU: the ComplEx decoder (decoders/complex.py) against golden vectors produced by running the reference's own
Complex class (tests/golden/make_complex_golden.py over tests/golden/tf1_shim.py).

  * the oracle (float64) reproduces loss, regularisation, every weight gradient, the test-mode scores and the
    reference Scorer's raw / filtered MRR and Hits at 1e-10;
  * the host plugin chain (factory, Complex, RelationEmbedding, encoders, Scorer) reproduces the same outputs with
    the library calls replaced by the oracle inside this test;
  * the factory builds Complex with dimension = CodeDimension and the reference's get_weights() order."""
import os

import numpy as np
import pytest
import torch

from oracle import rgcn_oracle as oracle
from relationprediction_b200 import ops
from relationprediction_b200.common import evaluation, model_builder
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag
from relationprediction_b200.decoders.complex import Complex
from relationprediction_b200.encoders.message_gcns.message_gcn import MessageGcn
from relationprediction_b200.encoders.relation_embedding import RelationEmbedding
import complex_oracle
from test_plugin_chain_cpu import OracleGraph, oracle_basis_layer, oracle_block_layer
from test_plugin_host import merged_settings
from test_reference_golden import KEEP, LAMBDA, split_weights

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_complex_golden.npz")
DT = torch.float64

# golden case -> (variant of split_weights, settings file, encoder/shared overrides, sparse_softmax grouping)
CASES = {
    "complex_toy_canonical": ("embedding", "complex.exp", {"CodeDimension": "24"}, "canonical"),
    "complex_syn_canonical": ("embedding", "complex.exp", {"CodeDimension": "16"}, "canonical"),
    "block_complex_toy_tf_kernel": ("block", "gcn_block.exp", {"InternalEncoderDimension": "40",
                                                               "CodeDimension": "40", "NumberOfBasisFunctions": "8"},
                                    "tf_unsorted_compat"),
    "block_complex_toy_canonical": ("block", "gcn_block.exp", {"InternalEncoderDimension": "40",
                                                               "CodeDimension": "40", "NumberOfBasisFunctions": "8"},
                                    "canonical"),
}


def load_case(name):
    z = np.load(GOLDEN)
    p = name + "/"
    return {k[len(p):]: z[k] for k in z.files if k.startswith(p)}


def build_model(toy, name, c):
    """The product's factory over the case's settings: the shipped file, the generator's overrides, Name=complex."""
    variant, settings_file, overrides, norm_mode = CASES[name]
    enc, dec = merged_settings(toy, settings_file, int(c["V"]), int(c["R"]), len(c["test_graph"]))
    for s in (enc, dec):
        for k, v in overrides.items():
            s.put(k, v)
        s.put("NormalizationMode", norm_mode)
    dec.put("Name", "complex")
    return model_builder.build_decoder(model_builder.build_encoder(enc, c["test_graph"]), dec)


def replay_masks(model, masks):
    """Dropout masks in the order the reference drew them (input-side layer first)."""
    layers, comp = [], model
    while comp is not None:
        if isinstance(comp, MessageGcn):
            layers.append(comp)
        comp = comp.next_component
    for layer, m in zip(layers[::-1], masks):
        layer.make_drop_mask = (lambda rows, mode, m=m, k=layer.dropout_keep_probability:
                                (m, k) if mode == 'train' else (None, 1.0))


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def oracle_run(c, variant, norm_mode):
    names, n_layers = split_weights(c, variant)
    leaves = {nm: torch.tensor(c["w%d" % i], dtype=DT, requires_grad=True) for i, nm in enumerate(names)}
    p = {"W_in": leaves["W_in"], "b_in": leaves["b_in"],
         "layers": [{k.split(".")[1]: v for k, v in leaves.items() if k.startswith("L%d." % l) and not k.endswith(".b")}
                    for l in range(n_layers)]}
    V, R = int(c["V"]), int(c["R"])
    masks = [c["mask%d" % i] for i in range(int(c["n_masks"]))]

    def encode(graph, mode):
        if variant == "embedding":
            return oracle.affine_onehot(leaves["W_in"], leaves["b_in"], use_bias=False, use_nonlinearity=False)
        return oracle.encoder_forward(p, graph, V, R, variant, mode=mode,
                                      drop_masks=masks if mode == "train" else None, keep=KEEP, norm_mode=norm_mode,
                                      dtype=DT, norm_dtype=np.float64)
    codes = encode(c["graph_split"] if variant != "embedding" else None, "train")
    loss, reg, _ = complex_oracle.complex_loss(codes, leaves["W_relation"], c["X"], c["Y"], DT)
    (loss + LAMBDA * reg).backward()
    with torch.no_grad():
        tc = encode(c["test_graph"], "test").detach()
    return names, leaves, loss.item(), LAMBDA * reg.item(), tc


class OracleScores(object):
    """score_all_subjects / score_all_objects of a fixed code matrix, for the Scorer."""

    def __init__(self, codes, rel_table):
        self.codes, self.rel = codes, rel_table

    def score_all_subjects(self, triplets):
        return complex_oracle.complex_predict_all_subjects(self.codes, self.rel, triplets, DT).numpy()

    def score_all_objects(self, triplets):
        return complex_oracle.complex_predict_all_objects(self.codes, self.rel, triplets, DT).numpy()


def ranking(model, known, ranked):
    sc = evaluation.Scorer({'Metric': 'MRR'})
    sc.register_data(known)
    sc.register_data(ranked)
    sc.register_model(model)
    res = sc.compute_scores(ranked).get_summary().results
    return np.array([[float(res[f][k]) for k in ('MRR', 'H@1', 'H@3', 'H@10')] for f in ('Raw', 'Filtered')])


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_complex_outputs(name):
    c = load_case(name)
    variant, _, _, norm_mode = CASES[name]
    names, leaves, loss, reg, tc = oracle_run(c, variant, norm_mode)
    assert abs(loss - float(c["loss"])) <= 1e-10 * abs(float(c["loss"]))
    assert abs(reg - float(c["reg"])) <= 1e-10 * abs(float(c["reg"]))
    for i, nm in enumerate(names):
        if bool(c["g%d_unused" % i]):
            assert nm.endswith(".b") or (variant == "embedding" and nm == "b_in"), nm
            assert leaves[nm].grad is None
            continue
        assert rel(leaves[nm].grad.numpy(), c["g%d" % i]) < 1e-10, nm
    Wr, tX = leaves["W_relation"].detach(), c["test_X"]
    e, _ = complex_oracle.complex_energies(tc, Wr, tX, DT)
    assert rel(torch.sigmoid(e).numpy(), c["predict"]) < 1e-10
    assert rel(complex_oracle.complex_predict_all_objects(tc, Wr, tX, DT).numpy(), c["all_objects"]) < 1e-10
    assert rel(complex_oracle.complex_predict_all_subjects(tc, Wr, tX, DT).numpy(), c["all_subjects"]) < 1e-10
    assert np.abs(ranking(OracleScores(tc, Wr), c["test_graph"], c["ranked"]) - c["ranking"]).max() < 1e-12


def oracle_complex(codes, rel_table, X, Y=None):
    if Y is None:
        e, (e1s, rs, e2s) = complex_oracle.complex_energies(codes, rel_table, X, DT)
        return e, torch.zeros((), dtype=DT), (e1s ** 2).mean() + (rs ** 2).mean() + (e2s ** 2).mean()
    loss, reg, e = complex_oracle.complex_loss(codes, rel_table, X, Y, DT)
    return e, loss, reg


@pytest.fixture
def oracle_backed_ops(monkeypatch):
    monkeypatch.setattr(ops, "Graph", OracleGraph)
    monkeypatch.setattr(ops, "block_layer", oracle_block_layer)
    monkeypatch.setattr(ops, "basis_layer", oracle_basis_layer)
    monkeypatch.setattr(ops, "complex_score", oracle_complex)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_chain_reproduces_reference_complex_outputs(toy, oracle_backed_ops, name):
    c = load_case(name)
    variant = CASES[name][0]
    model = build_model(toy, name, c)
    model.set_device("cpu")
    model.initialize_train()
    names, _ = split_weights(c, variant)
    ws = model.get_weights()
    assert len(ws) == len(names)
    for i, w in enumerate(ws):
        assert tuple(w.shape) == c["w%d" % i].shape, names[i]
        w.data = torch.tensor(c["w%d" % i], dtype=DT)
    replay_masks(model, [torch.tensor(c["mask%d" % i]) for i in range(int(c["n_masks"]))])
    feed = (c["graph_split"], c["X"], c["Y"]) if model.needs_graph() else (c["X"], c["Y"])
    total = model.train_loss(*feed)
    total.backward()
    ref_total = float(c["loss"]) + float(c["reg"])
    tol = 1e-10 if CASES[name][3] == "canonical" else 1e-6   # tf_unsorted_compat norms travel as float32
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


@pytest.mark.parametrize("settings_file,d", [("complex.exp", 500), ("gcn_block.exp", 40)])
def test_factory_builds_complex_with_code_dimension(toy, settings_file, d):
    enc, dec = merged_settings(toy, settings_file, toy["V"], toy["R"], len(toy["train"]))
    for s in (enc, dec):
        s.put("CodeDimension", str(d))
        s.put("InternalEncoderDimension", str(d))
        s.put("NumberOfBasisFunctions", "8")
    dec.put("Name", "complex")
    encoder = model_builder.build_encoder(enc, np.array(toy["train"]))
    model = model_builder.build_decoder(encoder, dec)
    assert type(model) is Complex and model.dimension == d and model.next_component is encoder
    assert isinstance(encoder, RelationEmbedding)
    assert abs(model.regularization_parameter - 0.01) < 1e-15
    model.set_device("cpu")
    model.initialize_train()
    ws = model.get_weights()
    # reference get_weights() order: deepest component first, the relation table (RelationEmbedding) last
    assert ws[-1] is encoder.W_relation and tuple(ws[-1].shape) == (toy["V"], d)
    if settings_file == "complex.exp":
        assert [tuple(w.shape) for w in ws] == [(toy["V"], d), (d,), (toy["V"], d)]
    else:
        assert len(ws) == 2 + 2 * 4 + 1
    assert model.get_train_input_variables()[-2:] == [model.X, model.Y]
    assert model.get_test_input_variables()[-1] is model.X


def test_factory_keeps_other_names():
    from relationprediction_b200.common.settings_reader import read_string
    s = read_string("[Decoder]\n\tName=nonlinear-transform\n\tRegularizationParameter=0.01\n")["Decoder"]
    assert model_builder.build_decoder(None, s) is None


def test_caches_are_per_instance(toy):
    enc, dec = merged_settings(toy, "complex.exp", toy["V"], toy["R"], len(toy["train"]))
    a = model_builder.build_decoder(model_builder.build_encoder(enc, None), dec)
    b = model_builder.build_decoder(model_builder.build_encoder(enc, None), dec)
    a.encoder_cache['test'] = "x"
    assert b.encoder_cache['test'] is None
    assert Complex.known_bit_mask is BilinearDiag.known_bit_mask
