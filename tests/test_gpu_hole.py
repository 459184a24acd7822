"""GPU: the HolE decoder against the float64 oracle of tests/hole_oracle.py -- the library's basis and transforms, the
chain transform -> kernel -> inverse for the scorer, the self-adversarial and 1-N objectives (max|a - b| / max|b| <
1e-4 against the float64 correlation energy of the raw rows for the loss, the L2 term, the energies, dcodes, drel and
the relation table's IndexedSlices norm), entity and relation ranks and top-k (exact on dyadic tables in the basis
with zero DC and Nyquist columns, where sqrt(d/2) is a power of two and every query row and energy is exact in float32),
ranks of random tables, chunked calls, the kernels the paths launch, and Toy runs of the driver under each objective,
the predict command and the gcn_basis + HolE and CompGCN + HolE chains."""
import json
import re

import numpy as np
import pytest
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

import hole_oracle as ho
import one_to_n_oracle as oo
from relationprediction_b200 import ops
from relationprediction_b200 import predict as predict_cmd
from relationprediction_b200 import train as driver
from relationprediction_b200.decoders.bilinear_diag import BilinearDiag
from test_gpu_train import TOY_EXP, write_toy

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4
REG_WEIGHT = 0.3
mask_of = BilinearDiag.known_bit_mask


def rel(a, b):
    a, b = torch.as_tensor(a).detach(), torch.as_tensor(b).detach()
    return float((a.double() - b.double().to(a.device)).abs().max() / max(float(b.double().abs().max()), 1e-30))


@pytest.fixture(autouse=True)
def slice_norms():
    ops.set_slice_norms(True)
    yield
    ops.set_slice_norms(False)


def layout(rng, V, R, n, K):
    """n positives, then K blocks of their corruptions, as the negative sampler lays them out"""
    pos = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, V, n)], 1)
    neg = np.tile(pos, (K, 1))
    side = rng.integers(0, 2, n * K) * 2
    neg[np.arange(n * K), side] = rng.integers(0, V, n * K)
    return np.concatenate([pos, neg]).astype(np.int32)


def tables(d, V, R, seed=0, scale=0.5):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(V, d, generator=g) * scale).float(), (torch.randn(R, d, generator=g) * scale).float()


# ---- the basis and the transforms ----
@pytest.mark.parametrize("d", [4, 8, 200, 500, 512, 516])
def test_basis_and_round_trip(d):
    U = ops.hole_basis(d, DEV)
    assert float((U.double().cpu() - ho.basis(d)).abs().max()) < 1e-7
    g = torch.Generator().manual_seed(d)
    x = torch.randn(1000, d, generator=g)
    xt = ops.hole_transform(x.to(DEV))
    assert rel(xt, x.double() @ ho.basis(d)) < 1e-5
    back = ops.hole_transform(xt, inverse=True)
    assert rel(back, x) < 1e-5
    # the basis is built once per (device, d)
    assert ops.hole_basis(d, DEV) is U


def test_transform_backward_is_the_inverse():
    d = 36
    x = torch.randn(50, d, device=DEV, requires_grad=True)
    g = torch.randn(50, d, device=DEV)
    ops.hole_transform(x).backward(g)
    assert rel(x.grad, g.double().cpu() @ ho.basis(d).T) < 1e-5


# ---- the chain transform -> kernel -> inverse against the direct correlation ----
def float64_grads(codes, relt, X, loss_fn):
    c = codes.double().requires_grad_(True)
    r = relt.double().requires_grad_(True)
    rg = r[torch.as_tensor(X[:, 1].astype(np.int64))].detach().requires_grad_(True)
    L, reg, e = loss_fn(c, r, rg)
    (L + REG_WEIGHT * reg).backward()
    drel = torch.zeros_like(r).index_add_(0, torch.as_tensor(X[:, 1].astype(np.int64)), rg.grad)
    return L, reg, e, c.grad, drel, float((rg.grad ** 2).sum())


def check_step(codes, relt, X, gpu_fn, loss_fn):
    c = codes.to(DEV).requires_grad_(True)
    r = relt.to(DEV).requires_grad_(True)
    L, reg, e = gpu_fn(ops.hole_transform(c), ops.hole_transform(r), torch.as_tensor(X, device=DEV))
    (L + REG_WEIGHT * reg).backward()
    L64, reg64, e64, dc64, dr64, ss64 = float64_grads(codes, relt, X, loss_fn)
    errs = {"loss": rel(L, L64), "reg": rel(reg, reg64), "energies": rel(e, e64), "dcodes": rel(c.grad, dc64),
            "drel": rel(r.grad, dr64), "slice_norm": rel(r._slice_sumsq, torch.tensor(ss64))}
    del r._slice_sumsq
    assert all(v < TOL for v in errs.values()), errs


@pytest.mark.parametrize("d", [4, 8, 12, 200, 500, 512])
@pytest.mark.parametrize("N,rows", [(333, 50), (5001, 7)])
def test_scorer_and_backward_match_float64(d, N, rows):
    rng = np.random.default_rng(d + N)
    codes, relt = tables(d, rows, 5, seed=d, scale=1.0 / np.sqrt(d))
    X = layout(rng, rows, 5, N, 0)
    Y = rng.integers(0, 2, N).astype(np.float32)

    def gpu(c, r, Xd):
        e, L, reg = ops.hole_score(c, r, Xd, torch.as_tensor(Y, device=DEV))
        return L, reg, e
    check_step(codes, relt, X, gpu, lambda c, r, rg: ho.ns_loss(c, r, X, torch.as_tensor(Y), rg))


@pytest.mark.parametrize("d,n,K,alpha", [(8, 64, 1, 1.0), (500, 300, 10, 1.0), (512, 101, 33, 0.5), (4, 7, 256, 2.0)])
def test_self_adversarial_matches_float64(d, n, K, alpha):
    rng = np.random.default_rng(K)
    codes, relt = tables(d, 40, 6, seed=K, scale=1.0 / np.sqrt(d))
    X = layout(rng, 40, 6, n, K)

    def gpu(c, r, Xd):
        return ops.self_adversarial_loss(c, r, Xd, K, alpha, "hole")
    check_step(codes, relt, X, gpu, lambda c, r, rg: ho.self_adversarial_loss(c, r, X, K, alpha, rg))


def test_slice_norm_reaches_the_table_a_row_range_was_taken_from():
    """the decoder transforms rel[0:R] of the encoder's [V, d] relation table: the slice norm lands on the table"""
    codes, relt = tables(16, 30, 30, seed=4)
    X = layout(np.random.default_rng(4), 30, 5, 40, 0)
    c = codes.to(DEV).requires_grad_(True)
    r = relt.to(DEV).requires_grad_(True)
    e, L, reg = ops.hole_score(ops.hole_transform(c), ops.hole_transform(r[:5]), torch.as_tensor(X, device=DEV),
                               torch.ones(40, device=DEV))
    (L + REG_WEIGHT * reg).backward()
    ss64 = float64_grads(codes, relt, X, lambda c, r, rg: ho.ns_loss(c, r, X, torch.ones(40), rg))[-1]
    assert rel(r._slice_sumsq, torch.tensor(ss64)) < TOL
    assert float(r.grad[5:].abs().max()) == 0.0


def test_self_adversarial_k1_is_negative_sampling():
    rng = np.random.default_rng(3)
    codes, relt = tables(500, 30, 4, seed=3, scale=0.05)
    X = layout(rng, 30, 4, 50, 1)
    c, r, Xd = ops.hole_transform(codes.to(DEV)), ops.hole_transform(relt.to(DEV)), torch.as_tensor(X, device=DEV)
    L, reg, e = ops.self_adversarial_loss(c, r, Xd, 1, 1.0, "hole")
    Y = torch.cat([torch.ones(50), torch.zeros(50)]).to(DEV)
    e_ns, L_ns, reg_ns = ops.hole_score(c, r, Xd, Y)
    assert torch.equal(e, e_ns)
    assert rel(L, L_ns) < 1e-6 and rel(reg, reg_ns) < 1e-6


def one_to_n_case(V, d, n, R=5, seed=0):
    g = torch.Generator().manual_seed(seed)
    scale = 1.0 / np.sqrt(d)
    codes = (torch.randn(V, d, generator=g) * scale).float()
    relt = (torch.randn(R + 2, d, generator=g) * scale).float()   # rows R.. are never queried
    rng = np.random.default_rng(seed)
    qs = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, 2, n)], 1).astype(np.int32)
    qs = qs[np.lexsort((qs[:, 0], qs[:, 1], qs[:, 2]))]
    y = (rng.random((n, V)) < 0.05).astype(np.float64)
    return codes, relt, qs, y


def run_one_to_n(codes, relt, qs, y, eps, R=5):
    c = codes.to(DEV).requires_grad_(True)
    r = relt.to(DEV).requires_grad_(True)
    loss, reg = ops.one_to_n_loss(ops.hole_transform(c), ops.hole_transform(r), qs,
                                  torch.as_tensor(oo.bits(y), device=DEV), eps, "hole", R)
    (loss + REG_WEIGHT * reg).backward()
    return loss.detach(), reg.detach(), c.grad, r.grad


@pytest.mark.parametrize("V,d,n", [(129, 4, 65), (129, 12, 65), (700, 24, 300), (1000, 500, 1000)])
@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_one_to_n_matches_float64(V, d, n, eps, monkeypatch):
    codes, relt, qs, y = one_to_n_case(V, d, n, seed=V + d)
    c = codes.double().requires_grad_(True)
    r = relt.double().requires_grad_(True)
    L, reg = ho.one_to_n_loss(c, r, qs, torch.as_tensor(y), eps)
    (L + REG_WEIGHT * reg).backward()
    whole = run_one_to_n(codes, relt, qs, y, eps)
    for name, a, b in zip(("loss", "reg", "dcodes", "drel"), whole, (L, reg, c.grad, r.grad)):
        assert torch.isfinite(a).all() and rel(a, b) < TOL, (name, rel(a, b))
    monkeypatch.setattr(ops, "ONE_TO_N_CHUNK_BYTES", (V + 4 * d) * 4 * 37)   # 37 queries per pass
    chunked = run_one_to_n(codes, relt, qs, y, eps)
    # the gradients are accumulated by atomic adds, whose order is not fixed: equal to float32 rounding
    for a, b in zip(chunked, whole):
        assert rel(a, b) < 1e-5


# ---- entity ranks and top-k ----
def exact_tables(d, V, R, seed=0, Vrel=None):
    """tables already in the basis with zero DC and Nyquist columns, nonzero only on a few frequency pairs: entity
    entries in {-1/2, 0, 1/2}, relation entries in {-1/w, 0, 1/w} with w = sqrt(d/2), an integer (a power of two) at
    these widths.  Every query row w (h r) is then a multiple of 1/4 (or 1/2) and every energy a multiple of 1/4 with
    |E| <= 6: exact in float32, and where the float32 sigmoid the ranks compare is strictly increasing (integer
    entries would give energies in steps of w, which saturate the sigmoid at d = 512).  Rows R..Vrel-1 of the relation
    table are 2 rel[0]: they would tie with relation 0 if they were ever scored."""
    w = np.sqrt(d / 2)
    assert w.is_integer()
    rng = np.random.default_rng(seed)
    cols = np.arange(2, min(d, 14))

    def rows(n):
        t = np.zeros((n, d), np.float32)
        for v in range(n):
            pick = rng.choice(cols, min(4, len(cols)), replace=False)
            t[v, pick] = rng.choice([-1.0, 1.0], len(pick))
        return t
    codes = rows(V) * 0.5
    relt = np.zeros((Vrel or R, d), np.float32)
    relt[:R] = rows(R) / np.float32(w)
    relt[R:] = 2 * relt[0]
    return torch.as_tensor(codes), torch.as_tensor(relt)


def exact_energies(S):
    return torch.equal(4 * S, (4 * S).round()) and float(S.abs().max()) <= 6


def _known(rng, gold, C, extra=3):
    return [sorted({int(g)} | set(rng.integers(0, C, extra).tolist())) for g in gold]


def _excl(rng, n, C, dense_rows=3):
    """random exclusions, plus rows that leave fewer than k (or no) eligible candidates"""
    lists = [sorted(set(rng.integers(0, C, rng.integers(0, 6)).tolist())) for _ in range(n)]
    for t in range(min(dense_rows, n)):
        keep = set(rng.integers(0, C, t).tolist())
        lists[t] = [v for v in range(C) if v not in keep]
    return lists


def test_query_rows_match_float64():
    codes, relt = tables(500, 100, 9, seed=2)
    X = layout(np.random.default_rng(2), 100, 9, 77, 0)
    for side in (0, 1):
        Q = ops.hole_query_rows(codes.to(DEV), relt.to(DEV), torch.as_tensor(X, device=DEV), side)
        assert rel(Q, ho.queries(codes.double(), relt.double(), X, side)[0]) < 1e-6


@pytest.mark.parametrize("V", [1, 127, 129, 300])
@pytest.mark.parametrize("d", [8, 32, 128, 512])
def test_entity_ranks_and_top_k_are_exact(V, d):
    rng = np.random.default_rng(V * d)
    codes, relt = exact_tables(d, V, 7, seed=V + d)
    if V > 10:
        codes[V - 1] = codes[3]            # duplicated rows tie exactly, across tile boundaries
    X = layout(rng, V, 7, 200, 0)
    ranker = ops.HolERanker(codes.to(DEV), relt.to(DEV))
    Xd = torch.as_tensor(X, device=DEV)
    for side in (0, 1):
        S, Sg, gold = ho.scores(codes, relt, X, side)
        assert exact_energies(S)
        known = _known(rng, gold.numpy(), V)
        raw, filt = ranker.rank(Xd, side, torch.as_tensor(mask_of(known, V), device=DEV))
        ref_raw, ref_filt = ho.ranks(S, gold, known)
        np.testing.assert_array_equal(raw.cpu().numpy(), ref_raw)
        np.testing.assert_array_equal(filt.cpu().numpy(), ref_filt)
        raw_only, none = ranker.rank(Xd, side)
        assert none is None and torch.equal(raw_only, raw)
        for k in (1, 10, 128):
            excl = _excl(rng, len(X), V)
            ids, en = ranker.top_k(Xd, side, k, torch.as_tensor(mask_of(excl, V), device=DEV))
            ref_ids, ref_en = ho.top_k(S, k, excl)
            np.testing.assert_array_equal(ids.cpu().numpy(), ref_ids)
            np.testing.assert_array_equal(en.cpu().numpy(), ref_en.astype(np.float32))


@pytest.mark.parametrize("R", [1, 31, 32, 33, 237])
@pytest.mark.parametrize("d", [8, 128])
def test_relation_ranks_and_top_k_are_exact(R, d):
    rng = np.random.default_rng(R + d)
    V = 300
    codes, relt = exact_tables(d, V, R, seed=R + d, Vrel=V)    # the [V, d] relation table of the R-GCN encoders
    if R > 2:
        relt[R - 1] = relt[0]
    X = layout(rng, V, R, 150, 0)
    ranker = ops.HolERanker(codes.to(DEV), relt.to(DEV), R)
    Xd = torch.as_tensor(X, device=DEV)
    S, Sg, gold = ho.scores(codes, relt, X, "relation", R)
    assert exact_energies(S)
    known = _known(rng, gold.numpy(), R, 2)
    for mask in (None, known):
        raw, filt = ranker.rank_relations(Xd, None if mask is None else torch.as_tensor(mask_of(mask, R), device=DEV))
        ref_raw, ref_filt = ho.ranks(S, gold, mask)
        np.testing.assert_array_equal(raw.cpu().numpy(), ref_raw)
        if mask is not None:
            np.testing.assert_array_equal(filt.cpu().numpy(), ref_filt)
    for k in (1, 10, 128):
        for excl in (None, _excl(rng, len(X), R)):
            ids, en = ranker.top_k_relations(Xd, k, None if excl is None else torch.as_tensor(mask_of(excl, R),
                                                                                             device=DEV))
            ref_ids, ref_en = ho.top_k(S, k, excl)
            np.testing.assert_array_equal(ids.cpu().numpy(), ref_ids)
            np.testing.assert_array_equal(en.cpu().numpy(), ref_en.astype(np.float32))


@pytest.mark.parametrize("V", [127, 14541])
def test_entity_ranks_of_random_tables_match_float64(V):
    """raw rows through the library's transform, against float64 scores of the exactly transformed rows"""
    d = 500 if V > 1000 else 64
    rng = np.random.default_rng(V)
    codes, relt = tables(d, V, 11, seed=V, scale=1.0 / np.sqrt(d))
    X = layout(rng, V, 11, 300, 0)
    ranker = ops.HolERanker(ops.hole_transform(codes.to(DEV)), ops.hole_transform(relt.to(DEV)))
    ct, rt = ho.transform(codes.double().to(DEV)), ho.transform(relt.double().to(DEV))
    for side in (0, 1):
        S, _, gold = ho.scores(ct, rt, X, side)
        known = _known(rng, gold.cpu().numpy(), V)
        raw, filt = ranker.rank(torch.as_tensor(X, device=DEV), side, torch.as_tensor(mask_of(known, V), device=DEV))
        ref_raw, ref_filt = ho.ranks(S, gold, known)
        for got, ref in ((raw, ref_raw), (filt, ref_filt)):
            got = got.cpu().numpy()
            # the gold's score is a float32 dot product, the candidates' the 3xTF32 GEMM's: near-ties may flip
            off = np.abs(got - ref)
            assert (off == 0).mean() >= 0.9 and (off <= 3).mean() >= 0.99, (off.max(), (off > 0).sum())
            assert abs(np.mean(1.0 / got) - np.mean(1.0 / ref)) < 1e-3


def test_relation_ranks_of_random_tables_match_float64():
    rng = np.random.default_rng(9)
    V, R, d = 400, 237, 500
    codes, relt = tables(d, V, V, seed=9, scale=1.0 / np.sqrt(d))
    X = layout(rng, V, R, 300, 0)
    ranker = ops.HolERanker(ops.hole_transform(codes.to(DEV)), ops.hole_transform(relt.to(DEV)), R)
    S, _, gold = ho.scores(ho.transform(codes.double().to(DEV)), ho.transform(relt.double().to(DEV)), X, "relation", R)
    raw, _ = ranker.rank_relations(torch.as_tensor(X, device=DEV))
    ref_raw, _ = ho.ranks(S, gold)
    got = raw.cpu().numpy()
    assert (got == ref_raw).mean() >= 0.97 and abs(np.mean(1.0 / got) - np.mean(1.0 / ref_raw)) < 1e-3


def test_chunked_calls_equal_one_call(monkeypatch):
    rng = np.random.default_rng(5)
    V, R = 400, 40
    codes, relt = tables(64, V, V, seed=5)
    X = torch.as_tensor(layout(rng, V, R, 500, 0), device=DEV)
    em = torch.as_tensor(mask_of(_excl(rng, 500, V), V), device=DEV)
    rm = torch.as_tensor(mask_of(_excl(rng, 500, R), R), device=DEV)

    def run():
        ranker = ops.HolERanker(codes.to(DEV), relt.to(DEV), R)
        out = [ranker.top_k(X, 1, 10, em), ranker.rank_relations(X, rm), ranker.top_k_relations(X, 7, rm),
               ranker.rank_relations(X, rm)]
        return [t for r in out for t in r]
    whole = run()
    monkeypatch.setattr(ops.HolERanker, "TOPK_CHUNK_BYTES", 64 * 1024)
    chunked = run()
    assert all(torch.equal(a, b) for a, b in zip(whole, chunked))


# ---- the kernels the HolE paths launch ----
VENDOR_GEMM = re.compile(r"cublas|cutlass|xmma|sgemm|gemv|gemmSN", re.I)


def test_launched_kernels_are_the_librarys():
    V, R = 300, 9
    rng = np.random.default_rng(1)
    X = torch.as_tensor(layout(rng, V, R, 40, 2), device=DEV)
    qs = np.array([[3, 0, 0], [5, 1, 1], [1, 2, 1]], np.int32)   # ordered by side, relation, anchor
    labels = torch.as_tensor(oo.bits(np.zeros((3, V))), device=DEV)

    def run(d):
        codes, relt = tables(d, V, R, seed=1)
        c = codes.to(DEV).requires_grad_(True)
        r = relt.to(DEV).requires_grad_(True)
        ct, rt = ops.hole_transform(c), ops.hole_transform(r)
        e, L, reg = ops.hole_score(ct, rt, X[:40], torch.ones(40, device=DEV))
        L2, reg2, _ = ops.self_adversarial_loss(ct, rt, X, 2, 1.0, "hole")
        L3, reg3 = ops.one_to_n_loss(ct, rt, qs, labels, 0.1, "hole", R)
        (L + reg + L2 + reg2 + L3 + reg3).backward()
        with torch.no_grad():
            ranker = ops.HolERanker(ct.detach(), rt.detach(), R)
            ranker.rank(X, 1)
            ranker.top_k(X, 0, 5)
            ranker.rank_relations(X)
            ranker.top_k_relations(X, 3)
            ops.hole_query_rows(ct.detach(), rt.detach(), X, 1)
        torch.cuda.synchronize()
    # warm up every path and the profiler itself, so that the first launches of the traced run are recorded; the
    # traced run uses a width no other test builds, so its basis is built inside the trace
    run(40)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]):
        run(40)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        run(44)
    names = {e.name for e in prof.events() if e.device_type == DeviceType.CUDA}
    hole = {m.group(0) for n in names for m in [re.search(r"k_hole_\w+", n)] if m}
    assert hole == {"k_hole_basis", "k_hole_fwd", "k_hole_finalize", "k_hole_bwd", "k_hole_rank_prepare",
                    "k_hole_relation_prepare", "k_hole_query_bwd"}, sorted(hole)
    assert any("k_selfadv_fwd" in n and "HolERows" in n for n in names), sorted(names)
    assert any("k_gemm_tf32x3" in n for n in names) and any("k_split_b" in n for n in names), sorted(names)
    # every name that mentions HolE is one of the kernels above; no vendor GEMM runs on these paths
    assert all(re.search(r"k_hole_\w+|k_selfadv_fwd", n) for n in names if re.search(r"hole", n, re.I)), sorted(names)
    assert not [n for n in names if VENDOR_GEMM.search(n)], sorted(names)


# ---- end to end on Toy ----
def _toy_exp(toy, tmp_path, objective="NegativeSampling", encoder=None):
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    text = TOY_EXP.format(layers=1, concat="No").replace(
        "Name=bilinear-diag", "Name=hole\n\tTrainingObjective=%s" % objective)
    if encoder:
        text = text.replace("Name=gcn_basis", encoder)
    exp.write_text(text)
    return exp


@pytest.mark.parametrize("objective", ["NegativeSampling", "SelfAdversarial", "1-N"])
def test_toy_gcn_basis_training_with_relation_metrics(toy, tmp_path, capsys, objective):
    exp = _toy_exp(toy, tmp_path, objective)
    assert "Name=gcn_basis" in exp.read_text()
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--no-save", "--no-early-stopping", "--final-eval", "0", "--relation-metrics"])
    out = capsys.readouterr().out
    losses = [float(l.split(":")[-1]) for l in out.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and all(np.isfinite(losses)) and losses[-1] < losses[0]
    assert "Relation prediction:" in out
    line = json.loads([l for l in out.splitlines() if l.startswith("{")][-1])
    assert 0.0 < line["relation"]["filtered"]["MRR"] <= 1.0 and 0.0 < line["filtered"]["MRR"] <= 1.0
    assert type(model).__name__ == "HolE"
    # the Scorer's fused ranks against float64 ranks of the raw test codes, transformed exactly
    test = np.array(toy["test"])
    fused = scorer.compute_scores(test)
    model._feed_test(getattr(model, "test_graph", None), test[:1])
    with torch.no_grad():
        codes, relt = [ho.transform(t.detach().double()) for t in model.next_component.get_all_codes(mode='test')[:2]]
    raw = [ho.ranks(*ho.scores(codes, relt, test, side)[::2])[0] for side in (0, 1)]
    assert (np.array(fused.raw_ranks) == np.concatenate(raw)).mean() >= 0.97


def test_predict_command_answers_entity_and_relation_queries(toy, tmp_path, capsys):
    exp = _toy_exp(toy, tmp_path)
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "40",
                                 "--no-save", "--no-early-stopping"])
    model.save(str(tmp_path / "Toy"))
    ckpt = sorted(tmp_path.glob("Toy-*.pt"))[-1]
    ent = {int(k): v for k, v in toy["entities"].items()}
    rl = {int(k): v for k, v in toy["relations"].items()}
    tri = np.array(toy["test"])[:8]
    lines = []
    for s_, r_, o_ in tri.tolist():
        lines += ["%s\t?\t%s" % (ent[s_], ent[o_]), "%s\t%s\t?" % (ent[s_], rl[r_]), "?\t%s\t%s" % (rl[r_], ent[o_])]
    (tmp_path / "queries.tsv").write_text("\n".join(lines) + "\n")
    out = tmp_path / "answers.tsv"
    R = int(model.relation_count)
    k = min(4, R)
    predict_cmd.main(["--settings", str(exp), "--dataset", str(tmp_path), "--checkpoint", str(ckpt),
                      "--queries", str(tmp_path / "queries.tsv"), "--k", str(k), "--out", str(out)])
    rows = [l.split("\t") for l in out.read_text().splitlines()]
    assert {int(r[0]) for r in rows} == set(range(len(lines)))
    for q in range(len(lines)):
        got = [r for r in rows if int(r[0]) == q]
        assert [int(r[1]) for r in got] == list(range(1, len(got) + 1)) and 0 < len(got) <= k
        scores = [float(r[3]) for r in got]
        assert scores == sorted(scores, reverse=True) and all(0.0 <= s <= 1.0 for s in scores)
    # the relation queries answer with relation names, the object queries agree with the Scorer's fused top-k
    assert all(r[2] in rl.values() for r in rows if int(r[0]) % 3 == 0)
    ids, _, _ = scorer.predict_top_k(tri, k, 1, filtered=True)
    obj = [(int(a), int(b), c) for a, b, c, _ in rows if int(a) % 3 == 1]
    assert obj == [(3 * j + 1, p + 1, ent[int(ids[j, p])]) for j in range(len(tri)) for p in range(k) if ids[j, p] >= 0]


def test_compgcn_hole_chain_trains_and_evaluates(toy, tmp_path, capsys):
    exp = _toy_exp(toy, tmp_path, "1-N", "Name=compgcn\n\tComposition=mult")
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "80",
                                 "--no-save", "--no-early-stopping", "--final-eval", "0", "--relation-metrics"])
    out = capsys.readouterr().out
    losses = [float(l.split(":")[-1]) for l in out.splitlines() if l.startswith("Average train loss")]
    assert len(losses) == 4 and all(np.isfinite(losses))
    line = json.loads([l for l in out.splitlines() if l.startswith("{")][-1])
    assert 0.0 < line["filtered"]["MRR"] <= 1.0 and 0.0 < line["relation"]["filtered"]["MRR"] <= 1.0
    assert type(model).__name__ == "HolE"
