"""Golden vectors of the highway skip connection (SkipConnections=Highway: every feature-input R-GCN layer wrapped in
extras/highway_layer.py's HighwayLayer) produced by RUNNING THE REFERENCE'S OWN MODEL CODE (needs /root/reference;
run HERE):

  python tests/golden/make_highway_golden.py        ->  tests/golden/reference_highway_golden.npz

Same machinery as make_reference_golden.py (its run_case, over tests/golden/tf1_shim.py): the reference's
model_builder wraps the layers unmodified (model_builder.py:296-307).  HighwayLayer computes `1 - gates`, so this
generator adds the one operator the shim lacks (T.__rsub__) at run time.  The reference memoises
HighwayLayer.vertex_embedding_function in a class-level dict, so it is reset wherever the MessageGcn and BilinearDiag
caches are (case start and every test feed); otherwise test-mode scores would come from the stale train-mode cache.

Cases: settings/gcn_block.exp with Highway on Toy (both sparse_softmax groupings), settings/gcn_basis.exp with Highway,
1 layer (the only layer is linear and wrapped), 3 layers, UseOutputTransform=Yes, the skewed synthetic graph of
make_reference_golden.py, and gcn_basis.exp with UseInputTransform=No, recorded only to document that the reference's
gate is dead there (its W and b gradients are exactly zero).  Per case the arrays are those of
make_reference_golden.run_case."""
import os

import numpy as np

import make_reference_golden as mrg
from extras.highway_layer import HighwayLayer  # noqa: E402  (reference module, importable once mrg set up the path)


def _rsub(self, o):
    return mrg.tf1_shim.T(mrg.tf1_shim._raw(o) - mrg.tf1_shim._raw(self))


mrg.tf1_shim.T.__rsub__ = _rsub
_reset_base = mrg.reset_class_level_caches
_feed_base = mrg.EagerScoringAdapter._feed


def reset_class_level_caches():
    _reset_base()
    HighwayLayer.vertex_embedding_function = {'train': None, 'test': None}


def _feed(self, triplets):
    HighwayLayer.vertex_embedding_function['test'] = None
    _feed_base(self, triplets)


mrg.reset_class_level_caches = reset_class_level_caches
mrg.EagerScoringAdapter._feed = _feed


def widths(d, B, code=None, **extra):
    w = [('Encoder', 'InternalEncoderDimension', str(d)), ('Shared', 'CodeDimension', str(code or d)),
         ('Encoder', 'NumberOfBasisFunctions', str(B)), ('Encoder', 'SkipConnections', 'Highway')]
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
    for grouping in ("tf_kernel", "canonical"):      # d = 20, B = 4: block size s = 5
        mrg.run_case("highway_block_toy_" + grouping, "gcn_block.exp", widths(20, 4), toy_train, toy_test, tV, tR,
                     41, grouping, out)
    mrg.run_case("highway_basis_toy_canonical", "gcn_basis.exp", widths(16, 3), toy_train, toy_test, tV, tR, 42,
                 "canonical", out)
    mrg.run_case("highway_block_toy_1layer_canonical", "gcn_block.exp", widths(16, 4, NumberOfLayers='1'),
                 toy_train, toy_test, tV, tR, 43, "canonical", out)
    mrg.run_case("highway_block_toy_3layer_canonical", "gcn_block.exp", widths(16, 2, NumberOfLayers='3'),
                 toy_train, toy_test, tV, tR, 44, "canonical", out)
    mrg.run_case("highway_block_toy_outproj_canonical", "gcn_block.exp",
                 widths(20, 4, code=12, UseOutputTransform='Yes'), toy_train, toy_test, tV, tR, 45, "canonical", out)
    mrg.run_case("highway_block_syn_canonical", "gcn_block.exp", widths(16, 4), syn, syn_test, sV, sR, 46,
                 "canonical", out)
    mrg.run_case("highway_onehot_toy_canonical", "gcn_basis.exp", widths(16, 2, UseInputTransform='No'),
                 toy_train, toy_test, tV, tR, 47, "canonical", out)
    path = os.path.join(mrg.HERE, "reference_highway_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%d arrays, %d bytes)" % (path, len(out), os.path.getsize(path)))


if __name__ == "__main__":
    main()
