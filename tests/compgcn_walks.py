"""The walks of the CompGCN layer (Encoder Name=compgcn) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

One row per (d_in, composition) that reaches a distinct set of walk kernels.  The dispatch lives in csrc/compgcn.cu:
the forward walk k_compgcn_fwd<NV, OP> and the backward walk k_compgcn_bwd<NV, OP> both take quads per lane
NV = min(ceil(d_in / 128), 4), with column slabs of NV * 128 columns (d_in > 512 runs several slabs of NV = 4), and
OP = 0 for Composition=mult, 1 for sub.  Besides the walks the layer launches shared helpers (split-row zeroing,
gradient prologue, db column sums) and the 3xTF32 GEMMs, which are not `k_compgcn_*`.
tests/test_compgcn_walk_table_host.py checks the rows against these rules and that the table names every
`k_compgcn_*` instantiation of the built library; tests/test_gpu_compgcn.py runs every row and checks both the
kernels launched and the numbers they produce.  Names are canonical: `k_compgcn_bwd<4,1>`."""
import block_walks

PREFIX = "k_compgcn_"
COMPOSITIONS = ("mult", "sub")


def nv_rule(d):
    return min((d + 127) // 128, 4)


def slabs(d, nv):
    return (d + nv * 128 - 1) // (nv * 128)


class Row(object):
    def __init__(self, d, nv, composition):
        self.d, self.nv, self.composition = d, nv, composition
        op = COMPOSITIONS.index(composition)
        self.name = "compgcn-%s-d%d" % (composition, d)
        self.fwd = ("k_compgcn_fwd<%d,%d>" % (nv, op),)
        self.bwd = ("k_compgcn_bwd<%d,%d>" % (nv, op),)

    @property
    def kernels(self):
        return frozenset(self.fwd + self.bwd)

    def __repr__(self):
        return self.name


ROWS = [Row(d, nv, c) for c in COMPOSITIONS for d, nv in ((24, 1), (200, 2), (300, 3), (516, 4))]
BY_NAME = {r.name: r for r in ROWS}


def table_kernels():
    return frozenset().union(*(r.kernels for r in ROWS))


def canonical(name):
    """`k_compgcn_*<...>` of a demangled kernel name in the table's spelling (either demangler); None otherwise."""
    return block_walks.canonical(name, PREFIX)
