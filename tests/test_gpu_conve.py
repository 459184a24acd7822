"""ConvE decoder on the GPU: query rows, the 1-N loss and its seven gradients against the float64 restatement
(conve_oracle.py), bitwise repeatability, fused ranks and top-k against float64 ranks, and Toy training runs."""
import json

import numpy as np
import pytest
import torch

import conve_oracle as co
from relationprediction_b200 import ops
from relationprediction_b200 import train as driver
from test_gpu_train import TOY_EXP, write_toy

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4


def rel(a, b):
    a, b = torch.as_tensor(a).detach(), torch.as_tensor(b).detach()
    return float((a.double() - b.double().to(a.device)).abs().max() / max(float(b.double().abs().max()), 1e-30))


def net_tables(V, R, h, w, C, seed=0):
    """codes, rel, rel_inv, filters, conv_bias, W_fc, b_fc (float32, CPU) with moderate energies"""
    d = h * w
    F = C * (2 * h - 2) * (w - 2)
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(V, d, generator=g) * 0.5).float(), (torch.randn(R, d, generator=g) * 0.5).float(),
            (torch.randn(R, d, generator=g) * 0.5).float(), (torch.randn(C, 3, 3, generator=g) * 0.5).float(),
            (torch.randn(C, generator=g) * 0.1).float(), (torch.randn(F, d, generator=g) / np.sqrt(F)).float(),
            (torch.randn(d, generator=g) * 0.1).float()]


def queries_both_sides(rng, V, R, n):
    """n distinct queries, the subject queries first (as ops.one_to_n_queries sorts them)"""
    q = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), (np.arange(n) >= n // 3).astype(np.int64)], 1)
    return q[np.argsort(q[:, 2], kind="stable")].astype(np.int32)


def label_bits(labels):
    n, V = labels.shape
    words = (V + 31) // 32
    bits = np.zeros((n, words), np.uint32)
    rows, cols = np.nonzero(labels)
    np.bitwise_or.at(bits, (rows, cols >> 5), np.left_shift(np.uint32(1), (cols & 31).astype(np.uint32)))
    return torch.as_tensor(bits.view(np.int32), device=DEV)


def make_masks(n, d, C, on, seed=1):
    if not on:
        return None, (1.0, 1.0, 1.0)
    keeps = (0.8, 0.75, 0.7)
    g = torch.Generator(device=DEV).manual_seed(seed)
    ms = tuple((torch.rand(n, wd, device=DEV, generator=g) < k).to(torch.uint8)
               for wd, k in zip((2 * d, C, d), keeps))
    return ms, keeps


def run_lib(tabs, h, q, bits, eps, masks, keeps, g=(1.0, 0.3)):
    ts = [t.to(DEV).requires_grad_(True) for t in tabs]
    weights = ops.ConvEWeights(*ts[2:], h=h)
    loss, reg = ops.conve_one_to_n_loss(ts[0], ts[1], weights, q, bits, eps, masks, keeps)
    (g[0] * loss + g[1] * reg).backward()
    return [loss.detach(), reg.detach()] + [t.grad for t in ts]


def run_oracle(tabs, h, q, labels, eps, masks, keeps, g=(1.0, 0.3)):
    ts = [t.to(DEV).double().requires_grad_(True) for t in tabs]
    loss, reg = co.one_to_n_loss(*ts, h, q, torch.as_tensor(labels, device=DEV), eps, masks, keeps)
    (g[0] * loss + g[1] * reg).backward()
    return [loss.detach(), reg.detach()] + [t.grad for t in ts]


NAMES = ("loss", "reg", "dcodes", "drel", "drel_inv", "dfilters", "dconv_bias", "dW_fc", "db_fc")

# (h, w, C) shapes; n crossing the 8-row padding and, with a small chunk budget, the chunk boundaries
CASES = [(2, 4, 1, 13, 0.0, False), (3, 4, 3, 40, 0.1, True), (5, 4, 2, 9, 0.1, False), (10, 20, 8, 70, 0.0, True),
         (20, 25, 32, 33, 0.1, True), (4, 4, 5, 1, 0.0, True)]


@pytest.mark.parametrize("h,w,C,n,eps,masked", CASES)
@pytest.mark.parametrize("small_chunks", [False, True])
def test_loss_and_gradients_match_float64(monkeypatch, h, w, C, n, eps, masked, small_chunks):
    V, R, d = 150, 7, h * w
    if small_chunks:   # a few queries per internal pass: chunks of 3-20 rows
        F = C * (2 * h - 2) * (w - 2)
        monkeypatch.setattr(ops, "ONE_TO_N_CHUNK_BYTES", 11 * (V + 6 * d + 3 * ((F + 3) // 4 * 4)) * 4)
    rng = np.random.default_rng(h * 100 + n)
    tabs = net_tables(V, R, h, w, C, seed=n)
    q = queries_both_sides(rng, V, R, n)
    labels = rng.random((n, V)) < 0.05
    masks, keeps = make_masks(n, d, C, masked)
    got = run_lib(tabs, h, q, label_bits(labels), eps, masks, keeps)
    ref = run_oracle(tabs, h, q, labels, eps, masks, keeps)
    for name, a, b in zip(NAMES, got, ref):
        assert torch.isfinite(a).all(), name
        assert rel(a, b) < TOL, (name, rel(a, b))


def test_dropped_elements_get_zero_gradient():
    h, w, C, n, V, R = 4, 5, 4, 50, 90, 5
    d = h * w
    rng = np.random.default_rng(3)
    tabs = net_tables(V, R, h, w, C, seed=3)
    q = queries_both_sides(rng, V, R, n)
    bits = label_bits(rng.random((n, V)) < 0.1)
    masks, keeps = make_masks(n, d, C, True)
    masks[1][:, 2] = 0     # filter 2 dropped for every query
    masks[2][:, 7] = 0     # hidden unit 7 dropped for every query
    got = run_lib(tabs, h, q, bits, 0.0, masks, keeps)
    assert torch.count_nonzero(got[5][2]) == 0 and float(got[6][2]) == 0.0
    assert torch.count_nonzero(got[7][:, 7]) == 0 and float(got[8][7]) == 0.0


def test_loss_and_network_gradients_are_bitwise_repeatable(monkeypatch):
    h, w, C, n, V, R = 10, 20, 8, 300, 2000, 11
    monkeypatch.setattr(ops, "ONE_TO_N_CHUNK_BYTES", 100 * (V + 6 * 200 + 3 * 8 * 18 * 18) * 4)
    rng = np.random.default_rng(5)
    tabs = net_tables(V, R, h, w, C, seed=5)
    q = queries_both_sides(rng, V, R, n)
    bits = label_bits(rng.random((n, V)) < 0.01)
    masks, keeps = make_masks(n, h * w, C, True)
    a = run_lib(tabs, h, q, bits, 0.1, masks, keeps)
    b = run_lib(tabs, h, q, bits, 0.1, masks, keeps)
    for i in (0, 1, 5, 6, 7, 8):
        assert torch.equal(a[i], b[i]), NAMES[i]


def test_query_rows_match_float64():
    h, w, C, V, R, n = 20, 25, 32, 300, 9, 77
    tabs = net_tables(V, R, h, w, C, seed=7)
    rng = np.random.default_rng(7)
    X = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, V, n)], 1).astype(np.int32)
    gt = [t.to(DEV) for t in tabs]
    weights = ops.ConvEWeights(*gt[2:], h=h)
    t64 = [t.to(DEV).double() for t in tabs]
    Xl = torch.as_tensor(X, device=DEV).long()
    for side in (0, 1):
        Q = ops.conve_query_rows(gt[0], gt[1], weights, torch.as_tensor(X, device=DEV), side)
        anchors = Xl[:, 0] if side == 1 else Xl[:, 2]
        ref = co.query_rows(*t64, h, anchors, Xl[:, 1], torch.full((n,), side, device=DEV))
        assert rel(Q, ref) < TOL


def integer_tables(V, R, h, w, C, seed):
    """small-integer tables: every conv output, FC output and energy is an exact float32 integer, in fp32 and in the
    3xTF32 GEMMs alike, so equal energies are exact ties"""
    d = h * w
    F = C * (2 * h - 2) * (w - 2)
    rng = np.random.default_rng(seed)
    ints = lambda shape, p: torch.as_tensor(rng.integers(-1, 2, shape) * (rng.random(shape) < p), dtype=torch.float32)
    return [ints((V, d), 0.05), ints((R, d), 0.5), ints((R, d), 0.5), ints((C, 3, 3), 0.5), ints((C,), 0.5),
            ints((F, d), 2.0 / F), ints((d,), 0.5)]


def gpu_sigmoid(E):
    """the float32 sigmoid the rank epilogue compares, 1 / (1 + exp(-E))"""
    E = E.float()
    return 1.0 / (1.0 + torch.exp(-E))


def oracle_energies(tabs, h, X, side):
    t64 = [t.to(DEV).double() for t in tabs]
    Xl = torch.as_tensor(X, device=DEV).long()
    anchors = Xl[:, 0] if side == 1 else Xl[:, 2]
    Q = co.query_rows(*t64, h, anchors, Xl[:, 1], torch.full((len(X),), side, device=DEV))
    return Q @ t64[0].T, Xl[:, 2] if side == 1 else Xl[:, 0]


def rank_case(V, R, n, seed):
    rng = np.random.default_rng(seed)
    X = np.stack([rng.integers(0, V, n), rng.integers(0, R, n), rng.integers(0, V, n)], 1).astype(np.int32)
    X[:5, 0], X[5:10, 2] = np.arange(5), np.arange(5)   # golds with a duplicated row (below)
    known = torch.as_tensor(rng.random((n, V)) < 0.01, device=DEV)
    known[np.arange(10), V - 5 + np.arange(10) % 5] = True   # ... whose twin is a known entity
    return X, known


@pytest.mark.parametrize("V,h,w,C", [(300, 4, 5, 3), (14541, 20, 25, 32), (14541, 10, 20, 8)])
def test_integer_tables_give_exact_ranks_and_top_k_with_ties(V, h, w, C):
    R, n = 13, 150
    tabs = integer_tables(V, R, h, w, C, seed=V + h)
    tabs[0][V - 5:] = tabs[0][:5]   # duplicated entity rows: exact ties
    X, known = rank_case(V, R, n, V)
    gt = [t.to(DEV) for t in tabs]
    ranker = ops.ConvERanker(gt[0], gt[1], ops.ConvEWeights(*gt[2:], h=h))
    Xd = torch.as_tensor(X, device=DEV)
    for side in (0, 1):
        E, gold = oracle_energies(tabs, h, X, side)
        oraw, ofilt = co.ranks(gpu_sigmoid(E), gold, known)
        raw, filt = ranker.rank(Xd, side, label_bits(known.cpu().numpy()))
        assert torch.equal(raw.long(), oraw) and torch.equal(filt.long(), ofilt), side
        raw2, none = ranker.rank(Xd, side)
        assert none is None and torch.equal(raw2.long(), oraw)
        ids, en = ranker.top_k(Xd, side, 10, label_bits(known.cpu().numpy()))
        order = torch.sort(-E.masked_fill(known, float("-inf")), dim=1, stable=True)
        assert torch.equal(ids.long(), order.indices[:, :10]) and torch.equal(en.double(), -order.values[:, :10])


@pytest.mark.parametrize("V,h,w,C", [(300, 4, 5, 3), (14541, 20, 25, 32), (14541, 10, 20, 8)])
def test_float_tables_match_float64_up_to_near_ties(V, h, w, C):
    """Random float tables: the ranks and top-k against float64 scores of the library's own query rows (the rows
    themselves are held to float64 by test_query_rows_match_float64; an F-wide fp32 FC layer moves energies by ~1e-5
    relative, which alone reorders near-equal candidates), and the filtered MRR against the float64 network."""
    R, n = 13, 300
    tabs = net_tables(V, R, h, w, C, seed=V)
    tabs[0] = tabs[0] * 0.2   # energies of a few units: float32 sigmoid scores away from saturation
    X, known = rank_case(V, R, n, V + 1)
    gt = [t.to(DEV) for t in tabs]
    weights = ops.ConvEWeights(*gt[2:], h=h)
    ranker = ops.ConvERanker(gt[0], gt[1], weights)
    Xd = torch.as_tensor(X, device=DEV)
    for side in (0, 1):
        gold = Xd[:, 2].long() if side == 1 else Xd[:, 0].long()
        E = ops.conve_query_rows(gt[0], gt[1], weights, Xd, side).double() @ gt[0].double().T
        oraw, ofilt = co.ranks(gpu_sigmoid(E), gold, known)
        raw, filt = ranker.rank(Xd, side, label_bits(known.cpu().numpy()))
        # fp32 rounding can swap entities whose scores agree to ~1e-7; nothing else may move (as test_gpu_rank.py)
        for got, ref in ((raw, oraw), (filt, ofilt)):
            dr = (got.long() - ref).abs()
            assert (dr == 0).float().mean() > 0.97 and dr.max() <= 3, (side, (dr == 0).float().mean(), dr.max())
        E64, _ = oracle_energies(tabs, h, X, side)
        _, ofilt64 = co.ranks(torch.sigmoid(E64), gold, known)
        assert abs(float((1.0 / filt.double()).mean() - (1.0 / ofilt64.double()).mean())) < 1e-3
        ids, en = ranker.top_k(Xd, side, 10)
        assert rel(en, torch.topk(E, 10, dim=1).values) < TOL


# ---- the driver on Toy, one run per encoder family ----
CONVE_EXP = TOY_EXP.replace("Name=bilinear-diag", "Name=conve\n\tEmbeddingHeight=4\n\tConvFilters=4").replace(
    "[General]\n", "[General]\n\tTrainingObjective=1-N\n")


@pytest.mark.parametrize("encoder", ["gcn_basis", "embedding"])
def test_toy_training(toy, tmp_path, capsys, encoder):
    write_toy(toy, tmp_path)
    exp = tmp_path / "toy.exp"
    exp.write_text(CONVE_EXP.format(layers=1, concat="No").replace("Name=gcn_basis", "Name=%s" % encoder))
    np.random.seed(0)
    torch.manual_seed(0)
    model, scorer = driver.main(["--settings", str(exp), "--dataset", str(tmp_path), "--max-iterations", "200",
                                 "--save-path", str(tmp_path / "ckpt" / "Toy"), "--final-eval", "0"])
    text = capsys.readouterr().out
    losses = [float(l.split(":")[-1]) for l in text.splitlines() if l.startswith("Average train loss")]
    assert len(losses) >= 4 and all(np.isfinite(losses)) and losses[-1] < losses[0]
    line = json.loads(text.strip().splitlines()[-1])
    assert 0.0 < line["filtered"]["MRR"] <= 1.0
