"""Golden vectors of the per-relation normaliser (NormalizationMode=relation: c_{i,r} = |N_i^r|) produced by RUNNING
THE REFERENCE'S OWN MODEL CODE (needs /root/reference; run HERE):

  python tests/golden/make_relation_norm_golden.py        ->  tests/golden/reference_relation_norm_golden.npz

Same machinery as make_reference_golden.py (its run_case, over tests/golden/tf1_shim.py).  The reference's layers
hard-code normalization=('global', ...) (gcn_basis.py:75-76 and the other layers) and no setting reaches the
'local' branch of MessageGraph.forward_incidence_matrix / backward_incidence_matrix
(extras/graph_representations.py:94-107, :134-147).  This generator wraps those two methods so that 'global'
becomes 'local'; the reference's own 'local' code then runs unmodified: a sparse_softmax over a [2R, V, E] all-ones
tensor indexed (relation, receiver | sender, message), followed by sparse_reduce_sum_sparse over axis 0.  The shim
lacks that op, so it is installed here (TF 1.4 semantics: sum the entries that agree on every other index; here every
(row, message) pair occurs once, so the sum only drops the relation axis).  Only the canonical sparse_softmax grouping
is recorded: the 'local' branch was never run under TF 1.x.

Importing make_gcn_diag_golden and make_times_diag_golden installs what those encoders need (tf.mul, tf.slice,
T.__rsub__, the Complex / HighwayLayer cache resets, the GraphSplitSize parse).

Cases (the keys below; per case the arrays are those of make_reference_golden.run_case): Toy block (s = 5) and basis
at small widths, the skewed synthetic graph of make_reference_golden.py (block, s = 8), UseInputTransform=No,
DiagonalCoefficients=Yes, Name=gcn_diag, SkipConnections=Highway and a ComplEx decoder."""
import os

import numpy as np
import torch

import make_gcn_diag_golden  # noqa: F401  (installs tf.mul, and through make_complex_golden tf.slice)
import make_times_diag_golden  # noqa: F401  (installs T.__rsub__, the highway resets, the parse_settings fix)
import make_reference_golden as mrg
from extras.graph_representations import MessageGraph  # noqa: E402  (reference module)

# case -> (settings file, overrides {key: value}, decoder name or None, graph: "toy" / "syn", seed)
CASES = {
    "relation_block_toy_s5": ("gcn_block.exp", {"InternalEncoderDimension": "40", "CodeDimension": "40",
                                                "NumberOfBasisFunctions": "8"}, None, "toy", 81),
    "relation_block_syn_s8": ("gcn_block.exp", {"InternalEncoderDimension": "32", "CodeDimension": "32",
                                                "NumberOfBasisFunctions": "4"}, None, "syn", 82),
    "relation_basis_toy": ("gcn_basis.exp", {"InternalEncoderDimension": "24", "CodeDimension": "24",
                                             "NumberOfBasisFunctions": "5"}, None, "toy", 83),
    "relation_onehot_toy": ("gcn_basis.exp", {"InternalEncoderDimension": "24", "CodeDimension": "24",
                                              "NumberOfBasisFunctions": "5", "UseInputTransform": "No"},
                            None, "toy", 84),
    "relation_times_diag_toy": ("gcn_basis.exp", {"InternalEncoderDimension": "16", "CodeDimension": "16",
                                                  "NumberOfBasisFunctions": "3", "DiagonalCoefficients": "Yes"},
                                None, "toy", 85),
    "relation_gcn_diag_toy": ("gcn_basis.exp", {"Name": "gcn_diag", "InternalEncoderDimension": "16",
                                                "CodeDimension": "16"}, None, "toy", 86),
    "relation_highway_block_toy": ("gcn_block.exp", {"InternalEncoderDimension": "20", "CodeDimension": "20",
                                                     "NumberOfBasisFunctions": "4", "SkipConnections": "Highway"},
                                   None, "toy", 87),
    "relation_block_complex_toy": ("gcn_block.exp", {"InternalEncoderDimension": "40", "CodeDimension": "40",
                                                     "NumberOfBasisFunctions": "8"}, "complex", "toy", 88),
}


def _sparse_reduce_sum_sparse(sp, axis):
    idx, vals = sp.indices, sp.values
    keep = [k for k in range(idx.shape[1]) if k != axis]
    rest = idx[:, keep]
    uniq, inv = torch.unique(rest, dim=0, return_inverse=True)
    out = torch.zeros(uniq.shape[0], dtype=vals.dtype).index_add(0, inv, vals)
    return mrg.tf1_shim.SparseTensor(uniq, out, sp.dense_shape[keep])


mrg.tf1_shim.sparse_reduce_sum_sparse = _sparse_reduce_sum_sparse
_forward_base = MessageGraph.forward_incidence_matrix
_backward_base = MessageGraph.backward_incidence_matrix


def _local(normalization):
    return ("local",) + tuple(normalization[1:]) if normalization[0] == "global" else normalization


MessageGraph.forward_incidence_matrix = lambda self, normalization: _forward_base(self, _local(normalization))
MessageGraph.backward_incidence_matrix = lambda self, normalization: _backward_base(self, _local(normalization))


def overrides_of(overrides, decoder):
    o = [('Shared' if k == 'CodeDimension' else 'Encoder', k, v) for k, v in overrides.items()]
    return o + ([('Decoder', 'Name', decoder)] if decoder else [])


def main():
    toy = os.path.join(mrg.REF, "data", "Toy")
    ent, rel = os.path.join(toy, "entities.dict"), os.path.join(toy, "relations.dict")
    toy_train = np.array(mrg.io.read_triplets_as_list(os.path.join(toy, "train.txt"), ent, rel))
    toy_test = np.array(mrg.io.read_triplets_as_list(os.path.join(toy, "test.txt"), ent, rel))
    tV, tR = len(mrg.io.read_dictionary(ent)), len(mrg.io.read_dictionary(rel))
    rng = np.random.RandomState(11)      # the skewed synthetic graph of make_reference_golden.py
    sV, sR, sE = 120, 6, 900
    syn = np.stack([rng.randint(0, sV, sE), rng.randint(0, sR, sE), (rng.zipf(1.6, sE) - 1) % sV], 1)
    syn_test = syn[rng.choice(sE, 12, replace=False)]
    graphs = {"toy": (toy_train, toy_test, tV, tR), "syn": (syn, syn_test, sV, sR)}

    out = {}
    for name, (settings_file, overrides, decoder, graph, seed) in CASES.items():
        train, test, V, R = graphs[graph]
        mrg.run_case(name, settings_file, overrides_of(overrides, decoder), train, test, V, R, seed, "canonical",
                     out)
    path = os.path.join(mrg.HERE, "reference_relation_norm_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%d arrays, %d bytes)" % (path, len(out), os.path.getsize(path)))


if __name__ == "__main__":
    main()
