"""The walks of the diagonal R-GCN layer (Encoder Name=gcn_diag) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

One row per d that reaches a distinct set of walk kernels.  The dispatch lives in csrc/gcn_diag.cu: the forward walk
k_diaggcn_fwd<NV> and the backward walk k_diaggcn_bwd<NV> both take quads per lane NV = min(ceil(d / 128), 4), with
column slabs of NV * 128 columns (d > 512 runs several slabs of NV = 4).  Besides the walks the backward launches the
shared helpers in HELPERS (gradient prologue, db column sums) and the 3xTF32 GEMMs, which are not `k_diaggcn_*`.
tests/test_gcn_diag_walk_table_host.py checks the rows against these rules and that the table names every
`k_diaggcn_*` instantiation of the built library; tests/test_gpu_gcn_diag.py runs every row and checks both the
kernels launched and the numbers they produce.  Names are canonical: `k_diaggcn_bwd<4>`."""
import block_walks

PREFIX = "k_diaggcn_"
HELPERS = ()


def nv_rule(d):
    return min((d + 127) // 128, 4)


def slabs(d, nv):
    return (d + nv * 128 - 1) // (nv * 128)


class Row(object):
    def __init__(self, d, nv):
        self.d, self.nv = d, nv
        self.name = "gcn-diag-d%d" % d
        self.fwd = ("k_diaggcn_fwd<%d>" % nv,)
        self.bwd = ("k_diaggcn_bwd<%d>" % nv,)

    @property
    def kernels(self):
        return frozenset(self.fwd + self.bwd)

    def __repr__(self):
        return self.name


ROWS = [
    Row(24, 1),
    Row(200, 2),
    Row(300, 3),
    Row(516, 4),      # 512 + 4 columns: two slabs, the second one quad wide
]
BY_NAME = {r.name: r for r in ROWS}


def table_kernels():
    return frozenset().union(*(r.kernels for r in ROWS))


def canonical(name):
    """`k_diaggcn_*<...>` of a demangled kernel name in the table's spelling (either demangler); None otherwise."""
    return block_walks.canonical(name, PREFIX)
