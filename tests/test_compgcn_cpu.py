"""CPU: the CompGCN encoder (Encoder Name=compgcn) -- the float64 oracle (gradcheck for both compositions), the
Composition key and every refusal, the factory's chain, widths and weight order, the host plugin chain under DistMult,
ComplEx, RotatE and ConvE and the training driver with the library calls replaced by the oracle (the substitution
lives in this file; the product has no CPU path), a checkpoint round trip, and the C-ABI argument checks, which all
return before any device work."""
import ctypes

import numpy as np
import pytest
import torch

import compgcn_oracle as cg
import complex_oracle
import rotate_oracle as ro
from oracle import rgcn_oracle as oracle
from relationprediction_b200 import _lib, ops
from relationprediction_b200 import train as driver
from relationprediction_b200.common import model_builder
from relationprediction_b200.encoders.affine_transform import AffineTransform
from relationprediction_b200.encoders.message_gcns.compgcn import CompGcn, parse_composition
from test_complex_cpu import oracle_complex
from test_conve_cpu import DenseLabels, oracle_conve  # noqa: F401  (fixture)
from test_gpu_train import TOY_EXP, write_toy
from test_highway_cpu import chain_of, rel
from test_plugin_chain_cpu import oracle_backed_ops  # noqa: F401  (fixture)
from test_plugin_host import merged_settings
from test_rotate_cpu import oracle_rotate  # noqa: F401  (fixture)
from test_train_loop_cpu import cpu_driver  # noqa: F401  (fixture)

DT = torch.float64


def random_messages(rng, V_dst, V_src, R, M):
    return (rng.integers(0, V_dst, M), rng.integers(0, V_src, M), rng.integers(0, 2 * R, M), rng.random(M) + 0.1)


# ---- the oracle ----
@pytest.mark.parametrize("composition", ["mult", "sub"])
def test_oracle_gradcheck(composition):
    rng = np.random.default_rng(3)
    V_dst, V_src, R, d_in, d_out = 5, 7, 2, 4, 3
    dst, src, relw, norm = random_messages(rng, V_dst, V_src, R, 14)
    g = torch.Generator().manual_seed(0)
    args = [torch.randn(s, dtype=DT, generator=g, requires_grad=True)
            for s in ((V_src, d_in), (2 * R, d_in), (d_in,), (3 * d_in, d_out), (d_in, d_out), (d_out,))]
    mask = torch.as_tensor(rng.random((V_dst, 2 * d_in)) < 0.7)
    for m, relu in ((None, False), (mask, True)):
        def f(*a):
            return cg.layer(*a, dst, src, relw, norm, V_dst, composition, m, 0.7, relu)
        assert torch.autograd.gradcheck(f, args)


def test_oracle_runs_compose_once():
    """The walk's identity: within a run of one weight id, sum n phi(h, z) = phi applied to the summed rows."""
    rng = np.random.default_rng(4)
    H, z = torch.randn(6, 8, dtype=DT), torch.randn(8, dtype=DT)
    n = torch.as_tensor(rng.random(6))
    np.testing.assert_allclose((n[:, None] * cg.phi(H, z, "mult")).sum(0), z * (n[:, None] * H).sum(0), rtol=1e-12)
    np.testing.assert_allclose((n[:, None] * cg.phi(H, z, "sub")).sum(0), (n[:, None] * H).sum(0) - n.sum() * z,
                               rtol=1e-12)


# ---- settings, factory, refusals ----
def compgcn_settings(toy, decoder=None, d="16", code=None, **enc_overrides):
    enc, dec = merged_settings(toy, "gcn_basis.exp", toy["V"], toy["R"], len(toy["train"]))
    enc.put("Name", "compgcn")
    enc.put("InternalEncoderDimension", d)
    for s in (enc, dec):
        s.put("CodeDimension", code or d)
    for k, v in enc_overrides.items():
        enc.put(k, v)
    if decoder:
        dec.put("Name", decoder)
    return enc, dec


def build(toy, **kw):
    enc, dec = compgcn_settings(toy, **kw)
    return model_builder.build_decoder(model_builder.build_encoder(enc, toy["train"]), dec)


def test_composition_parsing():
    assert parse_composition({}) == "mult"
    assert parse_composition({"Composition": "mult"}) == "mult"
    assert parse_composition({"Composition": "sub"}) == "sub"
    with pytest.raises(NotImplementedError, match="circular correlation"):
        parse_composition({"Composition": "corr"})
    for bad in ("Mult", "add", ""):
        with pytest.raises(ValueError, match="Composition"):
            parse_composition({"Composition": bad})
    with pytest.raises(ValueError, match="composition"):
        ops.compgcn_layer(None, None, None, None, None, None, None, composition="corr")


@pytest.mark.parametrize("flags,exc,match", [
    ({"Composition": "corr"}, NotImplementedError, "circular correlation"),
    ({"Composition": "div"}, ValueError, "Composition"),
    ({"UseOutputTransform": "Yes"}, ValueError, "UseOutputTransform"),
    ({"SkipConnections": "Highway"}, ValueError, "SkipConnections"),
    ({"SkipConnections": "Residual"}, ValueError, "SkipConnections"),
    ({"NumberOfLayers": "0"}, ValueError, "NumberOfLayers"),
], ids=["corr", "unknown", "outproj", "highway", "residual", "no-layers"])
def test_factory_refusals(toy, flags, exc, match):
    with pytest.raises(exc, match=match):
        build(toy, **flags)


@pytest.mark.parametrize("flags", [{}, {"AddDiagonal": "Yes", "DiagonalCoefficients": "Yes", "StoreEdgeData": "Yes",
                                        "Concatenation": "Yes", "NumberOfBasisFunctions": "3",
                                        "UseInputTransform": "No", "RandomInput": "Yes"}],
                         ids=["plain", "unread-flags"])
def test_factory_chain_widths_and_weight_order(toy, flags):
    model = build(toy, d="16", code="12", NumberOfLayers="3", **flags)
    chain = chain_of(model)
    assert [type(c) for c in chain[1:5]] == [CompGcn, CompGcn, CompGcn, AffineTransform]
    top, mid, bottom, emb = chain[1:5]
    assert chain[5].__class__.__name__ == "Representation"
    assert (top.shape, mid.shape, bottom.shape) == ([16, 12], [16, 16], [16, 16])
    assert top.top and not mid.top and not bottom.top
    assert bottom.owns_relations and not mid.owns_relations and not top.owns_relations
    assert not top.use_nonlinearity and mid.use_nonlinearity and bottom.use_nonlinearity
    assert emb.onehot_input and not emb.use_bias and not emb.use_nonlinearity
    assert emb.shape == [toy["V"], 16]
    np.random.seed(5)
    model.set_device("cpu")
    model.initialize_train()
    R = toy["R"]
    assert [tuple(w.shape) for w in bottom.local_get_weights()] == [(2 * R, 16), (16,), (48, 16), (16, 16), (16,)]
    assert [tuple(w.shape) for w in top.local_get_weights()] == [(16,), (48, 12), (16, 12), (12,)]
    assert bottom.local_get_weights()[0] is bottom.Z and top.local_get_weights()[1] is top.W_cat
    ws = model.get_weights()
    expect = emb.local_get_weights() + bottom.local_get_weights() + mid.local_get_weights() + top.local_get_weights()
    assert len(ws) == len(expect) == len(cg.weight_names(3)) and all(a is b for a, b in zip(ws, expect))
    assert float(top.b.detach().abs().max()) == 0.0 and top.b.requires_grad
    assert top.local_get_regularization() == 0.0


def test_initialisation(toy):
    model = build(toy, d="200")
    np.random.seed(2)
    model.set_device("cpu")
    model.initialize_train()
    top, bottom = chain_of(model)[1], chain_of(model)[2]
    R = toy["R"]
    for w, shape in ((bottom.Z, (2 * R, 200)), (top.W_cat, (600, 200)), (top.W_rel, (200, 200))):
        std = 3 / np.sqrt(shape[0] + shape[1])      # glorot_variance as a std-dev
        assert abs(float(w.detach().std()) / std - 1) < 0.1 and abs(float(w.detach().mean())) < 0.1 * std
    assert abs(float(top.z_loop.detach().std()) / (3 / np.sqrt(201)) - 1) < 0.2


# ---- the host plugin chain with the library calls replaced by the oracle ----
def oracle_compgcn_layer(H, Z, z_loop, W_cat, W_rel, b, graph, composition="mult", drop_mask=None, keep=1.0,
                         relu=True):
    dst, src, relw, norm = cg.triple_messages(graph.triples, Z.shape[0] // 2, graph.nf, graph.nb)
    return cg.layer(H, Z, z_loop, W_cat, W_rel, b, dst, src, relw, norm, graph.V_dst, composition, drop_mask, keep,
                    relu)


@pytest.fixture
def oracle_compgcn(monkeypatch, oracle_backed_ops):  # noqa: F811
    monkeypatch.setattr(ops, "compgcn_layer", oracle_compgcn_layer)
    monkeypatch.setattr(ops, "complex_score", oracle_complex)


def _fixed_masks(model, keep, rng):
    layers = [c for c in chain_of(model) if isinstance(c, CompGcn)][::-1]    # layer 0 first
    masks = []
    for layer in layers:
        m = torch.as_tensor(rng.random((layer_rows(model), 2 * layer.shape[0])) < keep).to(torch.uint8)
        masks.append(m)
        layer.make_drop_mask = (lambda rows, mode, m=m: (m, keep) if mode == 'train' else (None, 1.0))
    return masks


def layer_rows(model):
    return int(model.entity_count)


@pytest.mark.parametrize("composition", ["mult", "sub"])
@pytest.mark.parametrize("decoder", ["bilinear-diag", "complex", "rotate", "conve"])
def test_host_chain(toy, oracle_compgcn, oracle_rotate, oracle_conve, decoder, composition):  # noqa: F811
    train = np.asarray(toy["train"], np.int32)
    V, R = int(toy["V"]), int(toy["R"])
    enc, dec = compgcn_settings(toy, decoder=decoder, code="12", Composition=composition)
    keep = float(enc["DropoutKeepProbability"])
    if decoder == "conve":
        dec.put("TrainingObjective", "1-N")
        dec.put("EmbeddingHeight", "3")
        dec.put("ConvFilters", "2")
    model = model_builder.build_decoder(model_builder.build_encoder(enc, train), dec)
    model.set_device("cpu")
    model.initialize_train()
    if decoder == "conve":
        model.set_one_to_n_labels(DenseLabels(train, V))
    torch.manual_seed(0)
    ws = model.get_weights()
    for w in ws:
        w.data = torch.randn(w.shape, dtype=DT) * 0.3
    masks = _fixed_masks(model, keep, np.random.default_rng(1))
    rng = np.random.default_rng(7)
    X = np.stack([rng.integers(0, V, 30), rng.integers(0, R, 30), rng.integers(0, V, 30)], 1).astype(np.int32)
    Y = (rng.random(30) < 0.3).astype(np.float32)
    graph = train[:20]
    total = model.train_loss(graph, X, Y)
    total.backward()

    # the encoder's codes are the oracle chain's, and the decoder reads Z^L[0:R]
    names = cg.weight_names(2)
    enc_ws = ws[:len(names)]
    leaves = {nm: w.detach().clone().requires_grad_(True) for nm, w in zip(names, enc_ws)}
    nf, nb = oracle.graph_norms(graph, V, "canonical", np.float64)
    codes, relt = cg.encode(leaves, 2, graph, V, R, "train", masks, keep, nf, nb, composition)
    got_codes, got_rel, _ = model.next_component.get_all_codes(mode='train')
    assert tuple(got_rel.shape) == (R, 12) and got_rel.is_contiguous()
    assert rel(got_codes.detach(), codes.detach()) < 1e-12 and rel(got_rel.detach(), relt.detach()) < 1e-12
    param = float(dec["RegularizationParameter"])
    if decoder in ("bilinear-diag", "complex", "rotate"):
        if decoder == "bilinear-diag":
            L, reg, _ = oracle.distmult_loss(codes, relt, X, Y, DT)
        elif decoder == "complex":
            L, reg, _ = complex_oracle.complex_loss(codes, relt, X, Y, DT)
        else:
            L, reg, _ = ro.ns_loss(codes, relt, X, torch.as_tensor(Y), 12.0)
        ref = L + param * reg
        assert abs(total.item() - ref.item()) <= 1e-12 * abs(ref.item())
        ref.backward()
        for nm, w in zip(names, enc_ws):
            if nm == "b_in":   # the embedding has no bias
                assert w.grad is None and leaves[nm].grad is None
                continue
            assert rel(w.grad, leaves[nm].grad) < 1e-10, nm
    else:
        assert np.isfinite(total.item())
    for nm, w in zip(names, enc_ws):
        if nm != "b_in":
            assert w.grad is not None and float(w.grad.abs().max()) > 0, nm
    # test mode: no dropout, the same chain
    model.preprocess(train)
    model.register_for_test(train)
    test = np.asarray(toy["test"], np.int32)
    with torch.no_grad():
        p = np.asarray(model.score(test))
        tc, tr = cg.encode(leaves, 2, train, V, R, "test", None, 1.0,
                           *oracle.graph_norms(train, V, "canonical", np.float64), composition)
        got_codes, got_rel, _ = model.next_component.get_all_codes(mode='test')
    assert rel(got_codes, tc) < 1e-12 and rel(got_rel, tr) < 1e-12
    assert p.shape == (len(test),) and np.isfinite(p).all()


def test_driver_trains_on_toy(toy, tmp_path, capsys, cpu_driver, monkeypatch):  # noqa: F811
    monkeypatch.setattr(ops, "compgcn_layer", oracle_compgcn_layer)
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(TOY_EXP.format(layers=2, concat="No").replace("Name=gcn_basis", "Name=compgcn\n\tComposition=sub"))
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--device", "cpu"])
    text = capsys.readouterr().out
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and all(np.isfinite(losses)) and losses[-1] < losses[0]
    assert [c.composition for c in chain_of(model) if isinstance(c, CompGcn)] == ["sub", "sub"]
    summ = scorer.compute_scores(np.array(toy["train"])[:20]).get_summary()
    assert 0.0 < summ.results["Filtered"]["MRR"] <= 1.0


def test_checkpoint_round_trips_compgcn_weights(toy, oracle_compgcn, tmp_path):
    model = build(toy)
    np.random.seed(1)
    model.set_device("cpu")
    model.initialize_train()
    layers = [c for c in chain_of(model) if isinstance(c, CompGcn)]
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
    assert torch.equal(layers[0].b.detach(), torch.full((16,), 0.5)) and layers[-1].Z.shape == (2 * toy["R"], 16)


# ---- C-ABI: every bad argument is refused before any device work ----
def test_compgcn_entry_points_reject_bad_arguments_without_a_gpu(toy):
    lib = _lib.load()
    g = ops.Graph(np.array(toy["train"], np.int32), toy["V"], toy["R"])   # host-only graph
    d_in, d_out = 8, 12
    buf = ctypes.create_string_buffer(1 << 20)
    assert lib.rgcn_compgcn_workspace_bytes(None, d_in, d_out, 0) == -1
    assert lib.rgcn_compgcn_workspace_bytes(g.handle, 0, d_out, 0) == -1
    assert lib.rgcn_compgcn_workspace_bytes(g.handle, d_in, 0, 1) == -1
    need_f = lib.rgcn_compgcn_workspace_bytes(g.handle, d_in, d_out, 0)
    need_b = lib.rgcn_compgcn_workspace_bytes(g.handle, d_in, d_out, 1)
    assert 0 < need_f < need_b <= len(buf)
    assert need_f >= 2 * 3 * d_in * d_out * 4 and need_b - need_f >= toy["V"] * (d_out + 3 * d_in) * 4

    def fwd(gh=g.handle, d_in=d_in, d_out=d_out, op=0, H=buf, Z=buf, zl=buf, b=buf, Cat=buf, Zn=buf, keep=1.0,
            ws=need_f):
        return lib.rgcn_compgcn_forward(gh, d_in, d_out, op, H, Z, zl, buf, buf, b, None, keep, 1, Cat, buf, Zn, buf,
                                        ws, None)

    def bwd(gh=g.handle, d_in=d_in, d_out=d_out, op=1, H=buf, Z=buf, zl=buf, b=buf, Cat=buf, Zn=buf, keep=1.0,
            ws=need_b, out=buf, relu=1):
        return lib.rgcn_compgcn_backward(gh, d_in, d_out, op, H, Z, zl, buf, buf, None, keep, relu, Cat, out, buf, Zn,
                                         buf, buf, buf, buf, buf, b, buf, ws, None)
    for call in (fwd, bwd):
        assert call(gh=None) == -1
        assert call(d_in=6) == -1 and b"d % 4" in lib.rgcn_last_error()
        assert call(d_out=10) == -1 and b"d_out % 4" in lib.rgcn_last_error()
        assert call(d_in=0) == -1 and call(d_out=0) == -1
        assert call(op=2) == -1 and b"composition" in lib.rgcn_last_error()
        assert call(op=-1) == -1
        for k in ("H", "Z", "zl", "b", "Cat", "Zn"):
            assert call(**{k: None}) == -1 and b"null pointer" in lib.rgcn_last_error(), k
        assert call(keep=0.0) == -1 and call(keep=-1.0) == -1
        assert call(ws=16) == -4 and b"workspace" in lib.rgcn_last_error()
        assert call() == -5 and b"host-only" in lib.rgcn_last_error()     # valid arguments, host-only graph
    assert bwd(out=None) == -1
    assert bwd(out=None, relu=0) == -5     # out is only read for the ReLU gradient


def test_compgcn_op_rejects_cpu_tensors():
    class FakeGraph(object):
        V_dst = V_src = 6
        n_relw = 4
        handle = None
    d = 8
    with pytest.raises(_lib.RgcnError, match="CUDA float32"):
        ops.compgcn_layer(torch.zeros(6, d), torch.zeros(4, d), torch.zeros(d), torch.zeros(3 * d, d),
                          torch.zeros(d, d), torch.zeros(d), FakeGraph())
