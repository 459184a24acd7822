"""GPU: 1-N training (ops.one_to_n_loss, ops.OneToNLabels) against the float64 oracle of tests/one_to_n_oracle.py,
at max|a - b| / max|b| < 1e-4 for the loss, dcodes and drel."""
import numpy as np
import pytest
import torch

import fresh_process
import one_to_n_kernels as ok
import one_to_n_oracle as oo
from relationprediction_b200 import ops
from relationprediction_b200 import train as driver
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag
from test_gpu_train import TOY_EXP, write_toy

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4
REG_WEIGHT = 0.3


def rel(a, b):
    a, b = a.detach(), b.detach()
    return float((a.double() - b.double()).abs().max() / max(float(b.double().abs().max()), 1e-30))


def case(decoder, V, d, n, R=5, density=0.05, seed=0, scale=0.5):
    g = torch.Generator().manual_seed(seed)
    codes = (torch.randn(V, d, generator=g) * scale).float()
    relt = (torch.randn(max(R, 1) + 2, d, generator=g) * scale).float()   # rows R.. are never queried
    rng = np.random.default_rng(seed)
    qs = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, 2, n)], 1).astype(np.int32)
    qs = qs[np.lexsort((qs[:, 0], qs[:, 1], qs[:, 2]))]
    y = (rng.random((n, V)) < density).astype(np.float64)
    return codes, relt, qs, y


def run(decoder, codes, relt, qs, y, eps, R=5):
    c = codes.to(DEV).requires_grad_(True)
    r = relt.to(DEV).requires_grad_(True)
    labels = torch.as_tensor(oo.bits(y), device=DEV)
    loss, reg = ops.one_to_n_loss(c, r, qs, labels, eps, decoder, R)
    (loss + REG_WEIGHT * reg).backward()
    return loss.detach(), reg.detach(), c.grad, r.grad


def oracle(decoder, codes, relt, qs, y, eps):
    c = codes.to(DEV).double().requires_grad_(True)
    r = relt.to(DEV).double().requires_grad_(True)
    loss, reg = oo.loss(c, r, qs, torch.as_tensor(y, device=DEV), eps, decoder)
    (loss + REG_WEIGHT * reg).backward()
    return loss.detach(), reg.detach(), c.grad, r.grad


def check(decoder, codes, relt, qs, y, eps, R=5):
    got = run(decoder, codes, relt, qs, y, eps, R)
    ref = oracle(decoder, codes, relt, qs, y, eps)
    for name, a, b in zip(("loss", "reg", "dcodes", "drel"), got, ref):
        assert torch.isfinite(a).all(), name
        assert rel(a, b) < TOL, (name, rel(a, b))
    return got


SHAPES = ([(V, d, n) for d in (4, 8, 24, 500, 512, 516) for V, n in ((129, 65),)] +
          [(V, 8, n) for V, n in ((1, 63), (127, 64), (128, 129), (129, 1), (14541, 129))] +
          [(128, 24, n) for n in (1, 63, 64, 65, 128, 129)] + [(1000, 500, 5000)])


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
@pytest.mark.parametrize("V,d,n", SHAPES)
@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_matches_float64(decoder, V, d, n, eps):
    check(decoder, *case(decoder, V, d, n), eps)


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
def test_empty_and_full_label_rows(decoder):
    codes, relt, qs, y = case(decoder, 300, 24, 40)
    y[::3] = 0.0
    y[1::3] = 1.0
    check(decoder, codes, relt, qs, y, 0.0)
    check(decoder, codes, relt, qs, y, 0.1)


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
def test_saturated_energies(decoder):
    codes, relt, qs, y = case(decoder, 200, 16, 30, scale=4.0)
    z = oo.query_rows(codes.double(), relt.double(), qs, decoder) @ codes.double().T
    assert float(z.abs().min()) < 40 < float(z.abs().max()) and float((z.abs() >= 40).double().mean()) > 0.1
    check(decoder, codes, relt, qs, y, 0.1)


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
def test_small_chunks_equal_one_pass(decoder, monkeypatch):
    codes, relt, qs, y = case(decoder, 700, 24, 300)
    whole = run(decoder, codes, relt, qs, y, 0.1)
    monkeypatch.setattr(ops, "ONE_TO_N_CHUNK_BYTES", (700 + 4 * 24) * 4 * 37)   # 37 queries per pass
    chunked = run(decoder, codes, relt, qs, y, 0.1)
    for a, b in zip(chunked, whole):
        assert rel(a, b) < 1e-5


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
def test_loss_is_bitwise_repeatable(decoder):
    codes, relt, qs, y = case(decoder, 2000, 64, 700)
    a, b = run(decoder, codes, relt, qs, y, 0.1), run(decoder, codes, relt, qs, y, 0.1)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_label_rows_match_numpy(toy):
    train = np.asarray(toy["train"], np.int32)
    V = int(train[:, [0, 2]].max()) + 1
    R = int(train[:, 1].max()) + 1
    labels = ops.OneToNLabels(train, V, R, DEV)
    qs = oo.queries(train)
    got = labels.rows(qs).cpu().numpy()
    assert oo.unbits(got, V).tolist() == oo.dense_labels(train, qs, V).tolist()
    # queries in any order, including ones no training triple completes (empty rows)
    extra = np.array([[a, r, side] for a in range(V) for r in range(R) for side in (1, 0)][::7], np.int32)
    assert oo.unbits(labels.rows(extra).cpu().numpy(), V).tolist() == oo.dense_labels(train, extra, V).tolist()


def test_block_chain_end_to_end():
    """codes from an R-GCN block layer: the fused loss backpropagates through the layer exactly as the float64 chain
    rule does -- the layer's own backward applied to the oracle's gradient of the codes"""
    g = torch.Generator().manual_seed(5)
    V, d, R, B = 300, 16, 4, 4
    tri = torch.stack([torch.randint(0, V, (2000,), generator=g), torch.randint(0, R, (2000,), generator=g),
                       torch.randint(0, V, (2000,), generator=g)], 1).int().numpy()
    graph = ops.Graph(tri, V, R, device=0)
    H = (torch.randn(V, d, generator=g) * 0.5).float()
    Wf, Wb = [(torch.randn(R, B, d // B, d // B, generator=g) * 0.3).float() for _ in range(2)]
    Ws = (torch.randn(d, d, generator=g) * 0.3).float()
    relt = (torch.randn(R, d, generator=g) * 0.5).float()
    qs = ops.one_to_n_queries(tri[:500])
    y = oo.dense_labels(tri, qs, V)
    for decoder in ("distmult", "complex"):
        params = [t.to(DEV).requires_grad_(True) for t in (H, Wf, Wb, Ws)]
        r = relt.to(DEV).requires_grad_(True)
        codes = ops.block_layer(*params, graph, B, None, 1.0, True)
        loss, reg = ops.one_to_n_loss(codes, r, qs, torch.as_tensor(oo.bits(y), device=DEV), 0.1, decoder)
        grads = torch.autograd.grad(loss + REG_WEIGHT * reg, params + [r])
        c64 = codes.detach().double().requires_grad_(True)
        r64 = relt.to(DEV).double().requires_grad_(True)
        L, Rg = oo.loss(c64, r64, qs, torch.as_tensor(y, device=DEV), 0.1, decoder)
        dc, dr = torch.autograd.grad(L + REG_WEIGHT * Rg, [c64, r64])
        codes2 = ops.block_layer(*params, graph, B, None, 1.0, True)
        ref = torch.autograd.grad(codes2, params, grad_outputs=dc.float())
        assert rel(loss, L) < TOL and rel(grads[-1], dr) < TOL, decoder
        for got, want in zip(grads[:-1], ref):
            assert rel(got, want) < TOL, decoder


_TRACE = """
import json
import numpy as np
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile
import one_to_n_oracle as oo
import test_gpu_one_to_n as tg
from relationprediction_b200 import ops


def kernels(fn):
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == DeviceType.CUDA and "emcpy" not in e.name
            and "emset" not in e.name]


res = {}
for name, decoder, d in (("distmult", "distmult", 64), ("complex4", "complex", 64), ("complex2", "complex", 60)):
    codes, relt, qs, y = tg.case(decoder, 500, d, 200)
    c, r = codes.to(tg.DEV).requires_grad_(True), relt.to(tg.DEV).requires_grad_(True)
    labels = torch.as_tensor(oo.bits(y), device=tg.DEV)
    sum(ops.one_to_n_loss(c, r, qs, labels, 0.1, decoder, 5)).backward()     # warm-up (module load)
    torch.cuda.synchronize()
    with torch.no_grad():
        res[name + "/loss"] = kernels(lambda: ops.one_to_n_loss(c, r, qs, labels, 0.1, decoder, 5))
    out = []
    res[name + "/fwd"] = kernels(lambda: out.append(ops.one_to_n_loss(c, r, qs, labels, 0.1, decoder, 5)))
    total = out[0][0] + out[0][1]
    res[name + "/bwd"] = kernels(lambda: torch.autograd.grad(total, [c, r]))
lab = ops.OneToNLabels(np.array([[0, 0, 1], [1, 0, 2]], np.int32), 4, 1, tg.DEV)
lab.rows(np.array([[1, 0, 0], [0, 0, 1]], np.int32))
res["labels/loss"] = kernels(lambda: lab.rows(np.array([[1, 0, 0], [0, 0, 1]], np.int32)))
print("RESULT " + json.dumps(res))
"""


def test_launched_kernels_fresh_process():
    """Each call launches exactly the kernels of its row of tests/one_to_n_kernels.py, in that order."""
    traced = fresh_process.run_json(_TRACE)
    for (variant, direction), row in ok.ROWS.items():
        got = traced[variant + "/" + direction]
        own = [k for k in got if any(p in k for p in ("k_onen_", "k_split_b", "k_gemm", "rank_prepare"))]
        assert len(own) == len(row), (variant, direction, got)
        for want, name in zip(row, own):
            assert want.split("<")[0] in name and (("<" not in want) or want[want.index("<"):] in name.replace(
                "(int)", "")), (want, name)


ONE_TO_N_EXP = TOY_EXP.replace("[General]\n", "[General]\n\tTrainingObjective=1-N\n\tLabelSmoothing=0.1\n")


@pytest.mark.parametrize("decoder", ["distmult", "complex"])
def test_upstream_gradients_scale_the_two_terms(decoder):
    """the backward scales the forward's loss gradient and adds the L2 term: any upstream weights, and a second
    backward through the same graph, give the float64 gradient of g0 loss + g1 reg"""
    codes, relt, qs, y = case(decoder, 300, 24, 90)
    c, r = codes.to(DEV).requires_grad_(True), relt.to(DEV).requires_grad_(True)
    loss, reg = ops.one_to_n_loss(c, r, qs, torch.as_tensor(oo.bits(y), device=DEV), 0.1, decoder, 5)
    c64, r64 = codes.to(DEV).double().requires_grad_(True), relt.to(DEV).double().requires_grad_(True)
    L, Rg = oo.loss(c64, r64, qs, torch.as_tensor(y, device=DEV), 0.1, decoder)
    for g0, g1 in ((2.5, 0.0), (0.0, 1.7), (-0.4, 3.0)):
        got = torch.autograd.grad(g0 * loss + g1 * reg, [c, r], retain_graph=True)
        want = torch.autograd.grad(g0 * L + g1 * Rg, [c64, r64], retain_graph=True)
        for a, b in zip(got, want):
            assert rel(a, b) < TOL, (g0, g1)
    with torch.no_grad():   # a forward without gradients computes the same loss
        l2, r2 = ops.one_to_n_loss(c, r, qs, torch.as_tensor(oo.bits(y), device=DEV), 0.1, decoder, 5)
    assert torch.equal(l2, loss.detach()) and torch.equal(r2, reg.detach())


@pytest.mark.parametrize("decoder", ["bilinear-diag", "complex"])
def test_toy_training_one_to_n(toy, tmp_path, capsys, decoder):
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(ONE_TO_N_EXP.format(layers=1, concat="No").replace("Name=bilinear-diag", "Name=" + decoder))
    np.random.seed(0)
    torch.manual_seed(0)
    ckpt = tmp_path / "ckpt" / "Toy"
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--save-path", str(ckpt)])
    text = capsys.readouterr().out
    assert "Training objective: 1-N, label smoothing 0.1" in text
    assert "Initial loss" in text and "Validation filtered MRR" in text and "MRR" in text
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and all(np.isfinite(losses)) and losses[-1] < losses[0]
    assert list((tmp_path / "ckpt").glob("Toy-*.pt"))
    saved = [w.detach().clone() for w in model.get_weights()]
    model.save(str(tmp_path / "rt"))
    for w in model.get_weights():
        w.data.zero_()
    model.load("%s-%d.pt" % (tmp_path / "rt", model.save_iter - 1))
    assert all(torch.equal(a, w.detach()) for a, w in zip(saved, model.get_weights()))


@pytest.mark.parametrize("sampling", [[], ["--numpy-sampling"]])
def test_toy_training_one_to_n_with_graph_batches(toy, tmp_path, capsys, sampling):
    """GraphBatchSize < |train|: the positives come from the edge sampler (the library's one-call sample at rate 0,
    or the host draw and split), and are fed as X without negatives"""
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(ONE_TO_N_EXP.format(layers=1, concat="No").replace(
        "[General]\n", "[General]\n\tGraphBatchSize=30\n"))
    np.random.seed(0)
    torch.manual_seed(0)
    fed = []
    real = BilinearDiag._one_to_n

    def spy(self):
        fed.append(np.asarray(self.X.value).copy())
        return real(self)
    BilinearDiag._one_to_n = spy
    try:
        model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "40",
                                     "--no-save"] + sampling)
    finally:
        BilinearDiag._one_to_n = real
    text = capsys.readouterr().out
    assert "Training objective: 1-N" in text
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 2 and all(np.isfinite(losses))
    train = {tuple(t) for t in np.asarray(toy["train"]).tolist()}
    assert len(fed) >= 40 and all(len(x) == 30 and {tuple(t) for t in x.tolist()} <= train for x in fed)
    assert len({x.tobytes() for x in fed}) > 1   # a fresh graph batch every step
