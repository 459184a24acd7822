"""Golden vectors of the diagonal R-GCN encoder (Encoder Name=gcn_diag: model_builder.py:71-119 with every layer
encoders/message_gcns/gcn_diag.py's DiagGcn) produced by RUNNING THE REFERENCE'S OWN MODEL CODE (needs
/root/reference; run HERE):

  python tests/golden/make_gcn_diag_golden.py        ->  tests/golden/reference_gcn_diag_golden.npz

Same machinery as make_reference_golden.py (its run_case, over tests/golden/tf1_shim.py): the reference's
model_builder, DiagGcn, AffineTransform, RelationEmbedding and decoders run unmodified.  DiagGcn.compute_messages
(:35-36) spells the element-wise product `tf.mul`, which TensorFlow removed in 1.0 (TF 1.4 raises AttributeError
there), so this generator installs `mul` on the shim as the element-wise product `tf.multiply` -- the intent of the
line and what the port computes.  Importing make_complex_golden adds tf.slice and the Complex cache resets.

The reference ships no settings file for this encoder: every case is settings/gcn_basis.exp with Name=gcn_diag.
Cases: Toy under both sparse_softmax groupings, 1 layer (the only layer is linear), 3 layers, UseOutputTransform=Yes
with CodeDimension != d, the skewed synthetic graph of make_reference_golden.py, Decoder Name=complex, and one case
with UseInputTransform=No, SkipConnections=Highway, Concatenation=Yes and DiagonalCoefficients=Yes, flags the branch
never reads (the recorded chain is the plain one).  Per case the arrays are those of make_reference_golden.run_case."""
import os

import numpy as np

import make_complex_golden  # noqa: F401  (installs tf.slice and the Complex cache resets)
import make_reference_golden as mrg


def _mul(x, y):
    return mrg.tf1_shim.T(mrg.tf1_shim._raw(x) * mrg.tf1_shim._raw(y))


mrg.tf.mul = _mul


def widths(d, code=None, decoder=None, **extra):
    w = [('Encoder', 'Name', 'gcn_diag'), ('Encoder', 'InternalEncoderDimension', str(d)),
         ('Shared', 'CodeDimension', str(code or d))]
    if decoder:
        w.append(('Decoder', 'Name', decoder))
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
        mrg.run_case("gcn_diag_toy_" + grouping, "gcn_basis.exp", widths(16), toy_train, toy_test, tV, tR, 71,
                     grouping, out)
    mrg.run_case("gcn_diag_toy_1layer_canonical", "gcn_basis.exp", widths(12, NumberOfLayers='1'), toy_train,
                 toy_test, tV, tR, 72, "canonical", out)
    mrg.run_case("gcn_diag_toy_3layer_canonical", "gcn_basis.exp", widths(12, NumberOfLayers='3'), toy_train,
                 toy_test, tV, tR, 73, "canonical", out)
    mrg.run_case("gcn_diag_toy_outproj_canonical", "gcn_basis.exp", widths(16, code=12, UseOutputTransform='Yes'),
                 toy_train, toy_test, tV, tR, 74, "canonical", out)
    mrg.run_case("gcn_diag_syn_canonical", "gcn_basis.exp", widths(20), syn, syn_test, sV, sR, 75, "canonical", out)
    mrg.run_case("gcn_diag_complex_toy_canonical", "gcn_basis.exp", widths(16, decoder='complex'), toy_train,
                 toy_test, tV, tR, 76, "canonical", out)
    mrg.run_case("gcn_diag_ignored_flags_toy_canonical", "gcn_basis.exp",
                 widths(16, UseInputTransform='No', SkipConnections='Highway', Concatenation='Yes',
                        DiagonalCoefficients='Yes'), toy_train, toy_test, tV, tR, 77, "canonical", out)
    path = os.path.join(mrg.HERE, "reference_gcn_diag_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%d arrays, %d bytes)" % (path, len(out), os.path.getsize(path)))


if __name__ == "__main__":
    main()
