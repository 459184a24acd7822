"""Golden vectors of the basis layer with per-channel sigmoid coefficients (DiagonalCoefficients=Yes: every layer is
encoders/message_gcns/gcn_basis_times_diag.py's BasisGcnTimesDiag) produced by RUNNING THE REFERENCE'S OWN MODEL CODE
(needs /root/reference; run HERE):

  python tests/golden/make_times_diag_golden.py        ->  tests/golden/reference_times_diag_golden.npz

Same machinery as make_reference_golden.py (its run_case, over tests/golden/tf1_shim.py): the reference's
model_builder picks BasisGcnTimesDiag unmodified (model_builder.py:285-294).  Importing make_highway_golden adds the
operator and the cache resets the highway case needs.

Cases: settings/gcn_basis.exp with the flag on Toy (both sparse_softmax groupings), 1 layer (the only layer is linear),
3 layers, UseOutputTransform=Yes, the skewed synthetic graph of make_reference_golden.py, SkipConnections=Highway, and
settings/gcn_block.exp with the flag (Concatenation=Yes is overridden by the flag; small d and B).  Per case the arrays
are those of make_reference_golden.run_case."""
import os

import numpy as np

import make_highway_golden  # noqa: F401  (installs T.__rsub__ and the HighwayLayer cache resets)
import make_reference_golden as mrg
from encoders.message_gcns.gcn_basis_times_diag import BasisGcnTimesDiag  # noqa: E402  (reference module)


def _parse_settings(self):
    """BasisGcnTimesDiag.parse_settings (:10-14) reads GraphSplitSize with int(), which raises on the shipped settings'
    0.5.  The attribute is only stored (and reset by local_set_variable), never read by the computation, so it is
    parsed as a float here; everything else is the reference's own line."""
    self.dropout_keep_probability = float(self.settings['DropoutKeepProbability'])
    self.graph_split_size = float(self.settings['GraphSplitSize'])
    self.n_coefficients = int(self.settings['NumberOfBasisFunctions'])


BasisGcnTimesDiag.parse_settings = _parse_settings


def widths(d, B, code=None, **extra):
    w = [('Encoder', 'InternalEncoderDimension', str(d)), ('Shared', 'CodeDimension', str(code or d)),
         ('Encoder', 'NumberOfBasisFunctions', str(B)), ('Encoder', 'DiagonalCoefficients', 'Yes')]
    return w + [('Encoder', k, v) for k, v in extra.items()]


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

    out = {}
    for grouping in ("tf_kernel", "canonical"):
        mrg.run_case("times_diag_basis_toy_" + grouping, "gcn_basis.exp", widths(16, 3), toy_train, toy_test, tV, tR,
                     61, grouping, out)
    mrg.run_case("times_diag_basis_toy_1layer_canonical", "gcn_basis.exp", widths(12, 2, NumberOfLayers='1'),
                 toy_train, toy_test, tV, tR, 62, "canonical", out)
    mrg.run_case("times_diag_basis_toy_3layer_canonical", "gcn_basis.exp", widths(12, 2, NumberOfLayers='3'),
                 toy_train, toy_test, tV, tR, 63, "canonical", out)
    mrg.run_case("times_diag_basis_toy_outproj_canonical", "gcn_basis.exp",
                 widths(16, 2, code=12, UseOutputTransform='Yes'), toy_train, toy_test, tV, tR, 64, "canonical", out)
    mrg.run_case("times_diag_basis_syn_canonical", "gcn_basis.exp", widths(16, 4), syn, syn_test, sV, sR, 65,
                 "canonical", out)
    mrg.run_case("times_diag_highway_toy_canonical", "gcn_basis.exp", widths(16, 2, SkipConnections='Highway'),
                 toy_train, toy_test, tV, tR, 66, "canonical", out)
    mrg.run_case("times_diag_block_toy_canonical", "gcn_block.exp", widths(12, 3), toy_train, toy_test, tV, tR, 67,
                 "canonical", out)
    path = os.path.join(mrg.HERE, "reference_times_diag_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%d arrays, %d bytes)" % (path, len(out), os.path.getsize(path)))


if __name__ == "__main__":
    main()
