"""Test-side restatement of the per-relation normaliser (NormalizationMode=relation), the 'local' branch of the
reference's incidence matrices (extras/graph_representations.py:94-107, :134-147): a softmax over a row of ones grouped
by (relation, receiver) for the forward matrix and by (relation, sender) for the backward one, i.e.

    norm_f[k] = 1 / #{k' : o_k' = o_k, r_k' = r_k},    norm_b[k] = 1 / #{k' : s_k' = s_k, r_k' = r_k}

(the R-GCN paper's c_{i,r}; duplicate triples count as often as they occur).

oracle/rgcn_oracle.py states the per-direction norms of the 'global' branch and is left as it is; `graph_norms` below
answers mode "relation" here and hands every other mode to it.  `install(monkeypatch)` puts it in the oracle module's
place for one test, so the existing float64 chains (encoder_forward, the highway / gcn_diag / times_diag / one-hot
oracles, OracleGraph of the host-chain tests), which look the function up there, run in relation mode too."""
import numpy as np

from oracle import rgcn_oracle as oracle

_per_direction = oracle.graph_norms


def relation_norms(triples, norm_dtype=np.float32):
    """(norm_f[E], norm_b[E]) of the 'local' branch, computed in norm_dtype (float32 like the library by default)."""
    t = np.asarray(triples, dtype=np.int64).reshape(-1, 3)
    s, r, o = t[:, 0], t[:, 1], t[:, 2]
    n_rel = int(r.max()) + 1 if r.size else 1

    def per_relation(rows):
        _, inv, counts = np.unique(rows * n_rel + r, return_inverse=True, return_counts=True)
        return (norm_dtype(1.0) / counts[inv.reshape(-1)].astype(norm_dtype)).astype(norm_dtype)
    return per_relation(o), per_relation(s)


def graph_norms(triples, n_vertices, mode="canonical", norm_dtype=np.float32):
    if mode == "relation":
        return relation_norms(triples, norm_dtype)
    return _per_direction(triples, n_vertices, mode, norm_dtype)


def install(monkeypatch):
    monkeypatch.setattr(oracle, "graph_norms", graph_norms)
