"""Golden vectors of the ComplEx decoder produced by RUNNING THE REFERENCE'S OWN MODEL CODE (needs /root/reference;
run HERE):

  python tests/golden/make_complex_golden.py        ->  tests/golden/reference_complex_golden.npz

Same machinery as make_reference_golden.py (its run_case, over tests/golden/tf1_shim.py): the reference's
model_builder builds decoders/complex.py's Complex unmodified.  Complex is the only reference class that calls
tf.slice (extract_real_and_imaginary, :71-75), so this generator adds that one op to the shim at run time
(`_slice` below, TF 1.4 semantics: size[i] = -1 takes the rest of dimension i).  The reference memoises
Complex.encoder_cache in a class-level dict, so it is reset wherever BilinearDiag.encoder_cache is.  Cases: settings/complex.exp (graph-less
embedding encoder) on Toy and on the skewed synthetic graph, and settings/gcn_block.exp with Decoder.Name=complex
(both sparse_softmax groupings).  Per case the arrays are those of make_reference_golden.run_case."""
import os

import numpy as np

import make_reference_golden as mrg
from decoders.complex import Complex  # noqa: E402  (reference module, importable once mrg set up the path)


def _slice(x, begin, size):
    r = mrg.tf1_shim._raw(x)
    idx = tuple(slice(int(b), None if int(n) == -1 else int(b) + int(n)) for b, n in zip(begin, size))
    return mrg.tf1_shim.T(r[idx])


mrg.tf.slice = _slice
_reset_bilinear = mrg.reset_class_level_caches
_feed_bilinear = mrg.EagerScoringAdapter._feed


def reset_class_level_caches():
    _reset_bilinear()
    Complex.encoder_cache = {'train': None, 'test': None}


def _feed(self, triplets):
    Complex.encoder_cache['test'] = None
    _feed_bilinear(self, triplets)


mrg.reset_class_level_caches = reset_class_level_caches
mrg.EagerScoringAdapter._feed = _feed


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
    mrg.run_case("complex_toy_canonical", "complex.exp", [('Shared', 'CodeDimension', '24')], toy_train, toy_test,
                 tV, tR, 21, "canonical", out)
    mrg.run_case("complex_syn_canonical", "complex.exp", [('Shared', 'CodeDimension', '16')], syn, syn_test,
                 sV, sR, 22, "canonical", out)
    block = [('Encoder', 'InternalEncoderDimension', '40'), ('Shared', 'CodeDimension', '40'),
             ('Encoder', 'NumberOfBasisFunctions', '8'), ('Decoder', 'Name', 'complex')]
    for grouping in ("tf_kernel", "canonical"):
        mrg.run_case("block_complex_toy_" + grouping, "gcn_block.exp", block, toy_train, toy_test, tV, tR, 23,
                     grouping, out)
    path = os.path.join(mrg.HERE, "reference_complex_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%d arrays, %d bytes)" % (path, len(out), os.path.getsize(path)))


if __name__ == "__main__":
    main()
