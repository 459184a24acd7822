"""Golden vectors of the variational encoders (Encoder Name=variational_embedding, model_builder.py:43-69, and
Name=variational_gcn_basis, :186-254, both built on extras/variational_encoding.py's VariationalEncoding and
split_model.py's SplitModel) produced by RUNNING THE REFERENCE'S OWN MODEL CODE (needs /root/reference; run HERE):

  python tests/golden/make_variational_golden.py        ->  tests/golden/reference_variational_golden.npz

Same machinery as make_reference_golden.py (its run_case, over tests/golden/tf1_shim.py).  This generator adds the
ops VariationalEncoding calls to the shim: exp, multiply, pow, and random_normal, which draws float32 N(0, 1) values
from a per-case numpy stream and records every draw (as _dropout records its masks) so the CUDA path can replay them.
Importing make_times_diag_golden adds the highway operator, the Complex and HighwayLayer cache resets and the
BasisGcnTimesDiag settings fix; make_complex_golden adds tf.slice.

Eager quirks handled here:
  * VariationalEncoding memoises z in a CLASS-level dict: it is reset before each case, or a case silently reuses the
    previous case's z.  In test mode z is computed once (one eps draw) and shared by predict, all subjects, all
    objects and the ranking.  Each train case therefore records exactly two draws: eps0 (train) and eps1 (test).
  * SplitModel has no next_component, so the chain walk that drops the frozen graph before test mode descends into
    both branches.
  * get_weights() is list(set(...)) under the split, so its order is a set's order: every weight is stored with a
    name (`w_names`), the path of the component that owns it plus its index in that component's local_get_weights().

Cases: variational_embedding on settings/distmult.exp (Toy, both groupings: the encoder has no graph, so the two are
the same model) and variational_gcn_basis on settings/gcn_basis.exp: Toy under both groupings, 1 and 3 layers,
UseInputTransform=No, UseOutputTransform=Yes, the skewed synthetic graph, DiagonalCoefficients=Yes,
SkipConnections=Highway, settings/gcn_block.exp (Concatenation=Yes) and the ComplEx decoder."""
import os

import numpy as np
import torch

import make_complex_golden  # noqa: F401  (installs tf.slice and the Complex cache resets)
import make_times_diag_golden  # noqa: F401  (highway operator and cache resets, BasisGcnTimesDiag settings fix)
import make_reference_golden as mrg
from extras.variational_encoding import VariationalEncoding  # noqa: E402  (reference module)

shim = mrg.tf1_shim
normal_rng = np.random.RandomState(0)
normal_draws = []
gradient_xs = []


def _random_normal(shape, name=None):
    e = normal_rng.standard_normal(size=tuple(int(s) for s in shape)).astype(np.float32)
    normal_draws.append(e)
    return shim.T(torch.from_numpy(e.astype(np.float64)))


mrg.tf.exp = lambda x: shim.T(torch.exp(shim._raw(x)))
mrg.tf.multiply = lambda x, y: shim.T(shim._raw(x) * shim._raw(y))
mrg.tf.pow = lambda x, y: shim.T(shim._raw(x) ** shim._raw(y))
mrg.tf.random_normal = _random_normal
_gradients = mrg.tf.gradients


def _recording_gradients(ys, xs):
    gradient_xs[:] = list(xs)
    return _gradients(ys, xs)


mrg.tf.gradients = _recording_gradients
_reset_base = mrg.reset_class_level_caches


def reset_class_level_caches():
    _reset_base()
    VariationalEncoding.vertex_embedding_function = {'train': None, 'test': None}


mrg.reset_class_level_caches = reset_class_level_caches


def chain(model):
    while model is not None:
        yield model
        if hasattr(model, 'next_components'):
            for branch in model.next_components:
                yield from chain(branch)
            return
        model = model.next_component


mrg.chain = chain


def weight_names(model):
    """id(weight) -> name: the class path from the top of the chain, the split's branches as /mu and /sigma (a shared
    trunk is named along /mu), then '#' and the index in the owner's local_get_weights()."""
    names = {}

    def walk(comp, path):
        while comp is not None:
            path = path + "/" + comp.__class__.__name__
            if hasattr(comp, 'local_get_weights'):
                for i, w in enumerate(comp.local_get_weights()):
                    names.setdefault(id(w), "%s#%d" % (path, i))
            if hasattr(comp, 'next_components'):
                walk(comp.mu_network, path + "/mu")
                walk(comp.sigma_network, path + "/sigma")
                return
            comp = comp.next_component
    walk(model, "")
    return names


_build = mrg.build
built = []


def _recording_build(*a, **k):
    model, general = _build(*a, **k)
    built[:] = [model]
    return model, general


mrg.build = _recording_build


def run_case(name, settings_file, overrides, train, test, V, R, seed, grouping, out):
    global normal_rng
    normal_rng = np.random.RandomState(seed + 4)
    del normal_draws[:]
    mrg.run_case(name, settings_file, overrides, train, test, V, R, seed, grouping, out)
    names = weight_names(built[0])
    p = name + "/"
    out[p + "w_names"] = np.array([names[id(w)] for w in gradient_xs])
    assert len(normal_draws) == 2, len(normal_draws)
    out[p + "eps0"], out[p + "eps1"] = normal_draws
    print("    %d eps draws of %s, weights %s" % (len(normal_draws), normal_draws[0].shape,
                                                 ", ".join(out[p + "w_names"])))


def widths(name, d, code=None, decoder=None, **extra):
    w = [('Encoder', 'Name', name), ('Shared', 'CodeDimension', str(code or d))]
    if name == "variational_gcn_basis":
        w += [('Encoder', 'InternalEncoderDimension', str(d)), ('Encoder', 'NumberOfBasisFunctions', '3')]
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
    ve, vg = "variational_embedding", "variational_gcn_basis"

    out = {}
    for grouping in ("tf_kernel", "canonical"):
        run_case("var_emb_toy_" + grouping, "distmult.exp", widths(ve, 16), toy_train, toy_test, tV, tR, 81,
                 grouping, out)
        run_case("var_gcn_toy_" + grouping, "gcn_basis.exp", widths(vg, 16), toy_train, toy_test, tV, tR, 82,
                 grouping, out)
    run_case("var_gcn_toy_1layer_canonical", "gcn_basis.exp", widths(vg, 12, NumberOfLayers='1'), toy_train,
             toy_test, tV, tR, 83, "canonical", out)
    run_case("var_gcn_toy_3layer_canonical", "gcn_basis.exp", widths(vg, 12, NumberOfLayers='3'), toy_train,
             toy_test, tV, tR, 84, "canonical", out)
    run_case("var_gcn_toy_onehot_canonical", "gcn_basis.exp", widths(vg, 16, UseInputTransform='No'), toy_train,
             toy_test, tV, tR, 85, "canonical", out)
    run_case("var_gcn_toy_outproj_canonical", "gcn_basis.exp", widths(vg, 16, UseOutputTransform='Yes'), toy_train,
             toy_test, tV, tR, 86, "canonical", out)
    run_case("var_gcn_syn_canonical", "gcn_basis.exp", widths(vg, 20), syn, syn_test, sV, sR, 87, "canonical", out)
    run_case("var_gcn_toy_diagcoef_canonical", "gcn_basis.exp", widths(vg, 16, DiagonalCoefficients='Yes'),
             toy_train, toy_test, tV, tR, 88, "canonical", out)
    run_case("var_gcn_toy_highway_canonical", "gcn_basis.exp", widths(vg, 16, SkipConnections='Highway'), toy_train,
             toy_test, tV, tR, 89, "canonical", out)
    run_case("var_gcn_block_toy_canonical", "gcn_block.exp", widths(vg, 16, NumberOfBasisFunctions='4'), toy_train, toy_test, tV, tR, 90,
             "canonical", out)
    run_case("var_gcn_complex_toy_canonical", "gcn_basis.exp", widths(vg, 16, decoder='complex'), toy_train,
             toy_test, tV, tR, 91, "canonical", out)
    path = os.path.join(mrg.HERE, "reference_variational_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%d arrays, %d bytes)" % (path, len(out), os.path.getsize(path)))


if __name__ == "__main__":
    main()
