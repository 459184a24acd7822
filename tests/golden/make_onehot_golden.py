"""Golden vectors of the featureless gcn_basis encoder (UseInputTransform=No: layer 0 is BasisGcn with one-hot input)
produced by RUNNING THE REFERENCE'S OWN MODEL CODE (needs /root/reference; run HERE):

  python tests/golden/make_onehot_golden.py        ->  tests/golden/reference_onehot_golden.npz

Same machinery as make_reference_golden.py (its run_case, over tests/golden/tf1_shim.py): the reference's
model_builder wires Representation -> BasisGcn(onehot_input=True) -> ... unmodified (model_builder.py:140-168,
:277-283), and the one-hot layer's lookups (dot_or_lookup = tf.nn.embedding_lookup of the reshaped tables and of
W_self with tf.range(V)) run on ops the shim already has.  Cases: settings/gcn_basis.exp with UseInputTransform=No on
Toy (2 layers, both sparse_softmax groupings; 1 layer, where the only layer is both one-hot and linear), on the skewed
synthetic graph of make_reference_golden.py (2 layers), and on Toy with UseOutputTransform=Yes.  Per case the arrays
are those of make_reference_golden.run_case."""
import os

import numpy as np

import make_reference_golden as mrg


def widths(d, B, code=None):
    return [('Encoder', 'InternalEncoderDimension', str(d)), ('Shared', 'CodeDimension', str(code or d)),
            ('Encoder', 'NumberOfBasisFunctions', str(B)), ('Encoder', 'UseInputTransform', 'No')]


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
        mrg.run_case("onehot_toy_" + grouping, "gcn_basis.exp", widths(24, 5), toy_train, toy_test, tV, tR, 31,
                     grouping, out)
    mrg.run_case("onehot_toy_1layer_canonical", "gcn_basis.exp", widths(16, 2) + [('Encoder', 'NumberOfLayers', '1')],
                 toy_train, toy_test, tV, tR, 32, "canonical", out)
    mrg.run_case("onehot_syn_canonical", "gcn_basis.exp", widths(20, 3), syn, syn_test, sV, sR, 33, "canonical", out)
    mrg.run_case("onehot_toy_outproj_canonical", "gcn_basis.exp",
                 widths(20, 4, code=12) + [('Encoder', 'UseOutputTransform', 'Yes')], toy_train, toy_test, tV, tR,
                 34, "canonical", out)
    path = os.path.join(mrg.HERE, "reference_onehot_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%d arrays, %d bytes)" % (path, len(out), os.path.getsize(path)))


if __name__ == "__main__":
    main()
