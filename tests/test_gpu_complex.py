"""GPU: the ComplEx kernels (complex.cu through rgcn_complex_*) and the decoder plugin.

  * forward energies / loss / reg and backward dcodes / drel against the float64 oracle, on both load paths
    (float4 when d % 8 == 0, float2 when d % 8 == 4), with empty, tail-sized and hot-entity batches;
  * the relation table's IndexedSlices sum of squares against the materialised per-triple slices;
  * fused ranks: exact on integer codes with ties, near-exact at FB15k-237 shape;
  * the product path against the reference-code goldens (tests/golden/reference_complex_golden.npz);
  * a driver run of a complex.exp model on Toy: the loss decreases, fused ranking agrees with the matrix path,
    a checkpoint is written;
  * invalid widths and sides are rejected by the host-side checks."""
import numpy as np
import pytest
import torch

from oracle import rgcn_oracle as oracle
from relationprediction_b200 import _lib, ops
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag
import complex_oracle
from test_complex_cpu import CASES, build_model, load_case, replay_masks
from test_gpu_rank import make_known
from test_reference_golden import split_weights

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def rel(a, b):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    a, b = a.astype(np.float64), b.astype(np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def triples(rng, V, Vrel, N, hot=False):
    X = np.stack([rng.randint(0, V, N), rng.randint(0, Vrel, N), rng.randint(0, V, N)], 1).astype(np.int32)
    if hot and N:
        X[: N // 3, 0] = 7                  # one hot entity
        X[N // 3: N // 2, 2] = X[N // 3: N // 2, 0]   # s == o
    return X


def oracle_grads(codes, rel_table, X, Y, g_energy=None, lam=0.01):
    c = torch.tensor(codes, dtype=torch.float64, requires_grad=True)
    r = torch.tensor(rel_table, dtype=torch.float64, requires_grad=True)
    if Y is None:
        e, (e1s, rs, e2s) = complex_oracle.complex_energies(c, r, X, torch.float64)
        loss = torch.zeros((), dtype=torch.float64)
        reg = (e1s ** 2).mean() + (rs ** 2).mean() + (e2s ** 2).mean()
    else:
        loss, reg, e = complex_oracle.complex_loss(c, r, X, Y, torch.float64)
    total = loss + lam * reg
    if g_energy is not None:
        total = total + (e * torch.tensor(g_energy, dtype=torch.float64)).sum()
    total.backward()
    return e.detach(), loss.detach(), reg.detach(), c.grad, r.grad


@pytest.mark.parametrize("d", [8, 24, 500, 512])
@pytest.mark.parametrize("N,Vrel,hot", [(1000, 37, False), (333, None, True)])
def test_forward_backward_match_float64_oracle(d, N, Vrel, hot):
    rng = np.random.RandomState(d + N)
    V = 300
    Vrel = V if Vrel is None else Vrel            # the reference sizes the relation table [EntityCount, d]
    codes = rng.normal(0, 0.5, (V, d)).astype(np.float32)
    rel_table = rng.normal(0, 0.5, (Vrel, d)).astype(np.float32)
    X = triples(rng, V, Vrel, N, hot)
    Y = (rng.uniform(size=N) < 0.1).astype(np.float32)
    ct = torch.tensor(codes, device=DEV, requires_grad=True)
    rt = torch.tensor(rel_table, device=DEV, requires_grad=True)
    e, loss, reg = ops.complex_score(ct, rt, torch.tensor(X, device=DEV), torch.tensor(Y, device=DEV))
    (loss + 0.01 * reg).backward()
    e64, l64, q64, dc64, dr64 = oracle_grads(codes, rel_table, X, Y)
    assert rel(e, e64) < 1e-4
    assert abs(loss.item() - l64.item()) <= 1e-4 * abs(l64.item())
    assert abs(reg.item() - q64.item()) <= 1e-4 * abs(q64.item())
    assert rel(ct.grad, dc64) < 1e-4
    assert rel(rt.grad, dr64) < 1e-4


@pytest.mark.parametrize("d", [24, 500])
def test_upstream_energy_gradient_without_labels(d):
    """Y = None: no loss term; the energies' own upstream gradient (g_energy) and the L2 term drive the backward."""
    rng = np.random.RandomState(d)
    V, N = 200, 517
    codes = rng.normal(0, 0.5, (V, d)).astype(np.float32)
    rel_table = rng.normal(0, 0.5, (V, d)).astype(np.float32)
    X = triples(rng, V, V, N, hot=True)
    ge = rng.normal(0, 1, N).astype(np.float32)
    ct = torch.tensor(codes, device=DEV, requires_grad=True)
    rt = torch.tensor(rel_table, device=DEV, requires_grad=True)
    e, loss, reg = ops.complex_score(ct, rt, torch.tensor(X, device=DEV))
    assert loss.item() == 0.0
    ((e * torch.tensor(ge, device=DEV)).sum() + 0.01 * reg).backward()
    e64, _, q64, dc64, dr64 = oracle_grads(codes, rel_table, X, None, g_energy=ge)
    assert rel(e, e64) < 1e-4 and abs(reg.item() - q64.item()) <= 1e-4 * q64.item()
    assert rel(ct.grad, dc64) < 1e-4
    assert rel(rt.grad, dr64) < 1e-4


def test_empty_batch():
    ct = torch.randn(10, 8, device=DEV, requires_grad=True)
    rt = torch.randn(10, 8, device=DEV, requires_grad=True)
    e, loss, reg = ops.complex_score(ct, rt, torch.zeros(0, 3, dtype=torch.int32, device=DEV),
                                     torch.zeros(0, device=DEV))
    (loss + reg).backward()
    assert e.numel() == 0 and loss.item() == 0.0 and reg.item() == 0.0
    assert float(ct.grad.abs().max()) == 0.0 and float(rt.grad.abs().max()) == 0.0


@pytest.mark.parametrize("d", [24, 500])
def test_relation_slice_sum_of_squares(d):
    """sum over triples of |d(loss + lam reg)/d(gathered relation row)|^2, i.e. the norm of the un-aggregated
    IndexedSlices gradient, against the per-triple slices materialised in float64."""
    rng = np.random.RandomState(3)
    V, N, lam = 150, 700, 0.01
    codes = rng.normal(0, 0.5, (V, d)).astype(np.float32)
    rel_table = rng.normal(0, 0.5, (V, d)).astype(np.float32)
    X = triples(rng, V, 20, N)
    Y = (rng.uniform(size=N) < 0.1).astype(np.float32)
    c64 = torch.tensor(codes, dtype=torch.float64)
    rs = torch.tensor(rel_table, dtype=torch.float64)[torch.tensor(X[:, 1]).long()].requires_grad_(True)
    e1s, e2s = c64[torch.tensor(X[:, 0]).long()], c64[torch.tensor(X[:, 2]).long()]
    h = d // 2
    e = (e1s[:, :h] * rs[:, :h] * e2s[:, :h]).sum(1) + (e1s[:, h:] * rs[:, :h] * e2s[:, h:]).sum(1) \
        + (e1s[:, :h] * rs[:, h:] * e2s[:, h:]).sum(1) - (e1s[:, h:] * rs[:, h:] * e2s[:, :h]).sum(1)
    loss = oracle.weighted_cross_entropy_with_logits(torch.tensor(Y, dtype=torch.float64), e, 1).mean()
    (loss + lam * ((e1s ** 2).mean() + (rs ** 2).mean() + (e2s ** 2).mean())).backward()
    ref = float((rs.grad ** 2).sum())
    ops.set_slice_norms(True)
    try:
        rt = torch.tensor(rel_table, device=DEV, requires_grad=True)
        _, l, r = ops.complex_score(torch.tensor(codes, device=DEV), rt, torch.tensor(X, device=DEV),
                                    torch.tensor(Y, device=DEV))
        (l + lam * r).backward()
        got = float(rt._slice_sumsq)
    finally:
        ops.set_slice_norms(False)
    assert abs(got - ref) <= 1e-4 * ref


def complex_reference_ranks(codes, rel_table, X, side, known_lists, sigmoid=True):
    """raw = #{score >= gold}, filtered = raw - #{known with score >= gold} + 1, float64 energies."""
    c, r = codes.astype(np.float64), rel_table.astype(np.float64)
    h = c.shape[1] // 2
    s, p, o = X[:, 0], X[:, 1], X[:, 2]
    rr, ri = r[p, :h], r[p, h:]
    if side == 0:
        er, ei = c[o, :h], c[o, h:]
        q = np.concatenate([rr * er + ri * ei, rr * ei - ri * er], 1)
    else:
        er, ei = c[s, :h], c[s, h:]
        q = np.concatenate([er * rr - ei * ri, ei * rr + er * ri], 1)
    gold = s if side == 0 else o
    e = q @ c.T
    if sigmoid:
        e = (1.0 / (1.0 + np.exp(-e.astype(np.float32)))).astype(np.float32)
    g = e[np.arange(len(X)), gold]
    raw = (e >= g[:, None]).sum(1)
    kn = np.array([int((e[i, np.asarray(k, dtype=np.int64)] >= g[i]).sum()) if len(k) else 0
                   for i, k in enumerate(known_lists)])
    return raw, raw - kn + 1


@pytest.mark.parametrize("V,d,n", [(1000, 64, 300), (4133, 500, 777), (129, 200, 5)])
def test_integer_codes_give_exact_ranks_with_ties(V, d, n):
    rng = np.random.RandomState(0)
    codes = rng.randint(-1, 2, (V, d)).astype(np.float32) * (rng.uniform(size=(V, d)) < 0.05)
    rel_table = rng.randint(-1, 2, (V, d)).astype(np.float32)
    X = np.stack([rng.randint(0, V, n), rng.randint(0, V, n), rng.randint(0, V, n)], 1).astype(np.int32)
    ranker = ops.ComplexRanker(torch.as_tensor(codes, device=DEV), torch.as_tensor(rel_table, device=DEV))
    for side in (0, 1):
        known = make_known(rng, X, V, side)
        mask = torch.as_tensor(BilinearDiag.known_bit_mask(known, V), device=DEV)
        raw, filt = ranker.rank(torch.as_tensor(X, device=DEV), side, mask)
        ref_raw, ref_filt = complex_reference_ranks(codes, rel_table, X, side, known, sigmoid=False)
        np.testing.assert_array_equal(raw.cpu().numpy(), ref_raw)
        np.testing.assert_array_equal(filt.cpu().numpy(), ref_filt)
        raw2, none = ranker.rank(torch.as_tensor(X, device=DEV), side, None)
        assert none is None
        np.testing.assert_array_equal(raw2.cpu().numpy(), ref_raw)


def test_float_codes_ranks_match_float64_up_to_near_ties():
    rng = np.random.RandomState(1)
    V, d, n = 14541, 500, 1000            # FB15k-237 sizes, complex.exp width, one reference chunk
    codes = rng.normal(0, 0.3, (V, d)).astype(np.float32)
    rel_table = rng.normal(0, 1, (V, d)).astype(np.float32)
    X = np.stack([rng.randint(0, V, n), rng.randint(0, 237, n), rng.randint(0, V, n)], 1).astype(np.int32)
    ranker = ops.ComplexRanker(torch.as_tensor(codes, device=DEV), torch.as_tensor(rel_table, device=DEV))
    for side in (0, 1):
        known = make_known(rng, X, V, side)
        mask = torch.as_tensor(BilinearDiag.known_bit_mask(known, V), device=DEV)
        raw, filt = ranker.rank(torch.as_tensor(X, device=DEV), side, mask)
        ref_raw, ref_filt = complex_reference_ranks(codes, rel_table, X, side, known)
        dr = np.abs(raw.cpu().numpy() - ref_raw)
        df = np.abs(filt.cpu().numpy() - ref_filt)
        assert (dr == 0).mean() > 0.97 and dr.max() <= max(3, 0.002 * V), (dr.mean(), dr.max())
        assert (df == 0).mean() > 0.97 and df.max() <= max(3, 0.002 * V)
        mrr = lambda r: float(np.mean(1.0 / r))
        assert abs(mrr(filt.cpu().numpy()) - mrr(ref_filt)) < 1e-4


@pytest.mark.parametrize("name", sorted(CASES))
def test_product_matches_reference_complex_outputs(toy, name):
    c = load_case(name)
    model = build_model(toy, name, c)
    model.set_device(DEV)
    model.initialize_train()
    names, _ = split_weights(c, CASES[name][0])
    ws = model.get_weights()
    assert len(ws) == len(names)
    with torch.no_grad():
        for i, w in enumerate(ws):
            g = torch.tensor(c["w%d" % i], dtype=torch.float32, device=w.device)
            assert tuple(w.shape) == tuple(g.shape), names[i]
            w.copy_(g)
    replay_masks(model, [torch.tensor(c["mask%d" % i], dtype=torch.uint8, device=DEV)
                         for i in range(int(c["n_masks"]))])
    total = model.train_loss(*((c["graph_split"], c["X"], c["Y"]) if model.needs_graph() else (c["X"], c["Y"])))
    total.backward()
    ref_total = float(c["loss"]) + float(c["reg"])
    assert abs(total.item() - ref_total) <= 1e-4 * abs(ref_total)
    for i, (nm, w) in enumerate(zip(names, ws)):
        if bool(c["g%d_unused" % i]):
            assert w.grad is None or float(w.grad.abs().max()) == 0.0, nm
            continue
        assert rel(w.grad, c["g%d" % i]) < 1e-4, nm
    model.preprocess(c["test_graph"])
    model.register_for_test(c["test_graph"])
    tX = c["test_X"]
    # pre-sigmoid comparison where the sigmoid is not saturated, tight absolute error everywhere
    for got, ref in ((model.score(tX), c["predict"]), (model.score_all_objects(tX), c["all_objects"]),
                     (model.score_all_subjects(tX), c["all_subjects"])):
        got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
        assert got.shape == ref.shape
        assert np.abs(got - ref).max() < 2e-4
        live = (ref > 1e-3) & (ref < 1 - 1e-3) & (got > 0) & (got < 1)
        if live.any():
            lg, lr = np.log(got[live] / (1 - got[live])), np.log(ref[live] / (1 - ref[live]))
            assert np.abs(lg - lr).max() / max(1.0, np.abs(lr).max()) < 1e-4


def test_complex_exp_trains_on_toy_and_fused_ranking_agrees(toy, tmp_path, capsys):
    from relationprediction_b200 import train as driver
    from test_gpu_train import write_toy
    write_toy(toy, tmp_path)
    exp = tmp_path / "complex.exp"
    exp.write_text(toy["settings_text"]["complex.exp"].replace("CodeDimension=500", "CodeDimension=32")
                   .replace("ReportTrainLossEvery=100", "ReportTrainLossEvery=20")
                   .replace("CheckEvery=2000", "CheckEvery=40").replace("BurninPhaseDuration=6000",
                                                                        "BurninPhaseDuration=40"))
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--save-path", str(tmp_path / "ckpt" / "Toy")])
    text = capsys.readouterr().out
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and losses[-1] < losses[0]
    assert list((tmp_path / "ckpt").glob("Toy-*.pt"))
    test = np.array(toy["train"])
    assert model.supports_fused_ranking()
    fused = scorer.compute_scores(test).get_summary().results
    model.supports_fused_ranking = lambda: False
    matrix = scorer.compute_scores(test).get_summary().results
    for kind in ("Raw", "Filtered"):
        for k in ("MRR", "H@1", "H@3", "H@10"):
            assert abs(fused[kind][k] - matrix[kind][k]) < 2e-2, (kind, k, fused[kind][k], matrix[kind][k])


def test_invalid_arguments_are_rejected():
    ct = torch.randn(10, 6, device=DEV)
    X = torch.zeros(4, 3, dtype=torch.int32, device=DEV)
    with pytest.raises(_lib.RgcnError, match="d % 4"):
        ops.complex_score(ct, torch.randn(10, 6, device=DEV), X)
    ranker = ops.ComplexRanker(torch.randn(10, 8, device=DEV), torch.randn(10, 8, device=DEV))
    with pytest.raises(_lib.RgcnError, match="side"):
        ranker.rank(X, 2, None)
    with pytest.raises(_lib.RgcnError, match="d % 4"):
        ops.ComplexRanker(ct, torch.randn(10, 6, device=DEV)).rank(X, 0, None)
