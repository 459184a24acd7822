"""GPU: the variational head, ops.variational over rgcn_variational_forward / rgcn_variational_backward, against the
float64 restatement of tests/variational_oracle.py with eps injected, the reference-code goldens of
tests/golden/make_variational_golden.py, and driver runs of both encoder names.

Error bound: max|a - b| / max|b| < 1e-4 per output (the suite's global bound); the inputs keep log sigma in about
[-1.5, 1.5] so exp does not dominate the comparison."""
import numpy as np
import pytest
import torch

import fresh_process
import variational_kernels as vk
import variational_oracle as vo
from relationprediction_b200 import ops
from relationprediction_b200 import train as driver
from relationprediction_b200.encoders.message_gcns.message_gcn import MessageGcn
from relationprediction_b200.extras.variational_encoding import VariationalEncoding
from test_gpu_train import TOY_EXP, write_toy
from test_variational_cpu import CASES, build, chain_of, load_case, settings

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def inputs(V, d, w, seed):
    """float32-exact float64 inputs; d = 0 is the embedding variant"""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64).float().double()
    if d == 0:
        x = {"H": None, "W_mu": r(V, w), "b_mu": r(w), "W_sigma": (0.5 * r(V, w)).float().double(), "b_sigma": r(w)}
    else:
        x = {"H": r(V, d), "W_mu": (r(d, w) / np.sqrt(d)).float().double(), "b_mu": r(w),
             "W_sigma": (0.5 * r(d, w) / np.sqrt(d)).float().double(), "b_sigma": (0.2 * r(w)).float().double()}
    return x, r(V, w), r(V, w)


def run_product(x, eps, dz, g):
    t = {k: None if v is None else v.to(DEV).float().contiguous().requires_grad_(True) for k, v in x.items()}
    z, kl = ops.variational(t["H"], t["W_mu"], t["b_mu"], t["W_sigma"], t["b_sigma"], eps.to(DEV).float())
    (torch.sum(z * dz.to(DEV).float()) + g * kl).backward()
    torch.cuda.synchronize()
    grads = {k: None if v is None or v.grad is None else v.grad.double().cpu() for k, v in t.items()}
    return z.detach().double().cpu(), float(kl.detach()), grads


W_SET = (4, 24, 200, 500, 512, 516)
V_SET = (1, 63, 64, 65, 5000)


@pytest.mark.parametrize("g", [0.0, 1.0, 0.37])
@pytest.mark.parametrize("V", V_SET)
@pytest.mark.parametrize("w", W_SET)
@pytest.mark.parametrize("variant", ["embedding", "gcn"])
def test_matches_float64(variant, w, V, g):
    d = 0 if variant == "embedding" else w
    x, eps, dz = inputs(V, d, w, seed=V * 7 + w)
    z, kl, grads = run_product(x, eps, dz, g)
    rz, rkl = vo.variational(x["H"], x["W_mu"], x["b_mu"], x["W_sigma"], x["b_sigma"], eps)
    assert rel(z, rz) < TOL
    assert abs(kl - float(rkl)) <= TOL * abs(float(rkl))
    ref = vo.gradients(x["H"], x["W_mu"], x["b_mu"], x["W_sigma"], x["b_sigma"], eps, dz, g)
    for name, r in zip(("H", "W_mu", "b_mu", "W_sigma", "b_sigma"), ref):
        if r is None:
            assert grads[name] is None, name      # the embedding variant's biases are never read
        else:
            assert rel(grads[name], r) < TOL, (name, rel(grads[name], r))


def test_gcn_head_with_a_narrower_code_than_the_trunk():
    x, eps, dz = inputs(300, 64, 200, seed=5)
    z, kl, grads = run_product(x, eps, dz, 0.37)
    ref = vo.gradients(x["H"], x["W_mu"], x["b_mu"], x["W_sigma"], x["b_sigma"], eps, dz, 0.37)
    assert rel(z, vo.variational(x["H"], x["W_mu"], x["b_mu"], x["W_sigma"], x["b_sigma"], eps)[0]) < TOL
    for name, r in zip(("H", "W_mu", "b_mu", "W_sigma", "b_sigma"), ref):
        assert rel(grads[name], r) < TOL, name


@pytest.mark.parametrize("variant", ["embedding", "gcn"])
def test_kl_and_gradients_are_bitwise_repeatable(variant):
    """KL, z, the bias gradients and dH are formed in a fixed order: two runs agree bit for bit.  The gcn variant's
    dW comes from the split-K TN GEMM, whose partial tiles are added with atomics, so it agrees to rounding only."""
    x, eps, dz = inputs(5000, 0 if variant == "embedding" else 500, 500, seed=11)
    a, b = run_product(x, eps, dz, 0.37), run_product(x, eps, dz, 0.37)
    assert torch.equal(a[0], b[0]) and a[1] == b[1]
    for name in ("H", "W_mu", "b_mu", "W_sigma", "b_sigma"):
        ga, gb = a[2][name], b[2][name]
        if ga is None:
            continue
        if variant == "gcn" and name in ("W_mu", "W_sigma"):
            assert rel(ga, gb) < 1e-6, name
        else:
            assert torch.equal(ga, gb), name


_TRACE = """
import json
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile
import test_gpu_variational as tv
from relationprediction_b200 import ops


def kernels(fn):
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == DeviceType.CUDA and "emcpy" not in e.name
            and "emset" not in e.name]


res = {}
for variant, d in (("embedding", 0), ("gcn", 256)):
    x, eps, dz = tv.inputs(4096, d, 256, seed=3)
    t = {k: None if v is None else v.to(tv.DEV).float().contiguous().requires_grad_(True) for k, v in x.items()}
    e, y = eps.to(tv.DEV).float(), dz.to(tv.DEV).float()
    args = (t["H"], t["W_mu"], t["b_mu"], t["W_sigma"], t["b_sigma"], e)
    z, kl = ops.variational(*args)
    (torch.sum(z * y) + kl).backward()                          # warm-up (module load)
    torch.cuda.synchronize()
    out = []
    res[variant + "/fwd"] = kernels(lambda: out.append(ops.variational(*args)))
    loss = torch.sum(out[0][0] * y) + out[0][1]
    res[variant + "/bwd"] = kernels(lambda: torch.autograd.grad(loss, [v for v in t.values() if v is not None and
                                                                       (d or v.dim() == 2)], allow_unused=True))
print("RESULT " + json.dumps(res))
"""


def test_launched_kernels_fresh_process():
    """Each call launches exactly the kernels of its row of tests/variational_kernels.py, in that order.  Traced with
    torch.profiler in a fresh interpreter (tests/fresh_process.py)."""
    traced = fresh_process.run_json(_TRACE)
    for (variant, direction), row in vk.ROWS.items():
        got = traced[variant + "/" + direction]
        own = [k for k in got if "k_var_" in k or "k_split_b" in k or "k_gemm" in k]
        assert len(own) == len(row), (variant, direction, got)
        for want, name in zip(row, own):
            assert want.split("<")[0] in name and (("<" not in want) or want[want.index("<"):] in name.replace(
                "(int)", "")), (want, name)


@pytest.fixture(scope="module")
def gpu_model_for():
    def make(toy, name):
        c = load_case(name)
        settings_file, overrides, decoder, norm_mode = CASES[name]
        enc, dec = settings(toy, settings_file, dict(overrides, NormalizationMode=norm_mode), decoder, int(c["V"]),
                            int(c["R"]), len(c["test_graph"]))
        model = build(enc, toy["train"], dec)
        model.set_device(DEV)
        model.initialize_train()
        return c, model
    return make


# the goldens whose values stay inside float32 comfortably (the others reach exp(l) of 1e20 and beyond)
GOLDEN_CASES = ["var_emb_toy_canonical", "var_gcn_toy_1layer_canonical", "var_gcn_syn_canonical",
                "var_gcn_toy_onehot_canonical", "var_gcn_toy_diagcoef_canonical"]


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_product_matches_reference_variational_outputs(toy, gpu_model_for, name):
    c, model = gpu_model_for(toy, name)
    ws = model.get_weights()
    names = vo.weight_names(model)
    index = {str(nm): i for i, nm in enumerate(c["w_names"])}
    for nm, w in zip(names, ws):
        w.data = torch.tensor(c["w%d" % index[nm]], dtype=torch.float32, device=DEV)
    layers = [comp for comp in chain_of(model) if isinstance(comp, MessageGcn)]
    for layer, i in zip(layers[::-1], range(int(c["n_masks"]))):
        m = torch.tensor(c["mask%d" % i], device=DEV)
        layer.make_drop_mask = (lambda rows, mode, m=m, k=layer.dropout_keep_probability:
                                (m, k) if mode == 'train' else (None, 1.0))
    head = [comp for comp in chain_of(model) if isinstance(comp, VariationalEncoding)][0]
    draws = []
    head.draw_epsilon = lambda mode: (draws.append(mode), torch.tensor(
        c["eps0" if len(draws) == 1 else "eps1"], dtype=torch.float32, device=DEV))[1]
    feed = (c["graph_split"], c["X"], c["Y"]) if model.needs_graph() else (c["X"], c["Y"])
    total = model.train_loss(*feed)
    total.backward()
    ref_total = float(c["loss"]) + float(c["reg"])
    assert abs(total.item() - ref_total) <= TOL * abs(ref_total)
    for nm, w in zip(names, ws):
        i = index[nm]
        if bool(c["g%d_unused" % i]):
            assert w.grad is None or float(w.grad.abs().max()) == 0.0, nm
        else:
            assert rel(w.grad.double().cpu().numpy(), c["g%d" % i]) < TOL, nm
    model.preprocess(c["test_graph"])
    model.register_for_test(c["test_graph"])
    for got, ref in ((model.score(c["test_X"]), c["predict"]),
                     (model.score_all_objects(c["test_X"]), c["all_objects"]),
                     (model.score_all_subjects(c["test_X"]), c["all_subjects"])):
        assert got.shape == ref.shape and np.abs(np.asarray(got, np.float64) - ref).max() < 1e-3


def test_uninjected_eps_is_standard_normal_and_fresh(toy, gpu_model_for):
    """eps comes from torch.randn on the layer's device: z - mu over sigma has N(0, 1) moments, and it differs between
    two train evaluations and between train and test mode (the reference's codes are stochastic in both)."""
    c, model = gpu_model_for(toy, "var_emb_toy_canonical")
    head = chain_of(model)[2]
    with torch.no_grad():
        head.mu_network.W.copy_(torch.randn(head.mu_network.W.shape, device=DEV))
        head.sigma_network.W.fill_(0.0)
    codes = []
    for mode in ("train", "train", "test"):
        model.clear_cache()
        with torch.no_grad():
            z = head.get_all_codes(mode=mode)[0]
        codes.append((z - head.mu_network.W).detach())        # sigma = exp(0) = 1: this is eps itself
    e = torch.cat([x.flatten() for x in codes])
    assert abs(float(e.mean())) < 0.1 and abs(float(e.std()) - 1) < 0.1
    assert not torch.equal(codes[0], codes[1]) and not torch.equal(codes[1], codes[2])


@pytest.mark.parametrize("name", ["variational_embedding", "variational_gcn_basis"])
def test_toy_training_with_each_variational_encoder(toy, tmp_path, capsys, name):
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(TOY_EXP.format(layers=1, concat="No").replace("Name=gcn_basis", "Name=" + name))
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--save-path", str(tmp_path / "ckpt" / "Toy")])
    text = capsys.readouterr().out
    assert "Initial loss" in text and "Validation filtered MRR" in text
    assert any(isinstance(comp, VariationalEncoding) for comp in chain_of(model))
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and all(np.isfinite(losses))
    summ = scorer.compute_scores(np.array(toy["train"])[:20]).get_summary()
    assert 0.0 < summ.results["Filtered"]["MRR"] <= 1.0
