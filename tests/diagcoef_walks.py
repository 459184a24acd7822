"""The walks of the basis layer with per-channel sigmoid coefficients (DiagonalCoefficients=Yes) -- TEST
INFRASTRUCTURE, NOT PRODUCT CODE.

One row per (B, d) that reaches a distinct set of walk kernels.  The dispatch lives in csrc/basis_diagcoef.cu:
  - forward  k_diagcoef_fwd<NV>: quads per lane NV = min(ceil(d / 128), 4), column slabs ceil(d / (NV * 128));
  - backward k_diagcoef_dp<BC,NVB> (source-major dP walk) and k_diagcoef_dc<BC,NVB> (weight-id-major dC walk): bases
    per pass BC = B for B in {1, 2, 5}, else 4 (ceil(B / 4) passes); NVB = min(ceil(d / 128), 2).
Besides the walks the layer launches the helpers in HELPERS (sigmoid table, bias + activation epilogue, db column sums;
the last only in the backward).  tests/test_diagcoef_walk_table_host.py checks the rows against these rules and that
the table names every `k_diagcoef_*` instantiation of the built library; tests/test_gpu_times_diag.py runs every row
and checks both the kernels launched and the numbers they produce.  Names are canonical: `k_diagcoef_dp<4,2>`."""
import block_walks

PREFIX = "k_diagcoef_"
HELPERS = ("k_diagcoef_sigmoid", "k_diagcoef_bias_act", "k_diagcoef_colsum")


def bc_rule(B):
    return B if B in (1, 2, 5) else 4


def nv_rule(d, cap=4):
    return min((d + 127) // 128, cap)


def slabs(d, nv):
    return (d + nv * 128 - 1) // (nv * 128)


class Row(object):
    def __init__(self, B, d, bc, nv, nvb):
        self.B, self.d, self.bc, self.nv, self.nvb = B, d, bc, nv, nvb
        self.name = "diag-B%d-d%d" % (B, d)
        self.fwd = ("k_diagcoef_fwd<%d>" % nv,)
        self.bwd = ("k_diagcoef_dp<%d,%d>" % (bc, nvb), "k_diagcoef_dc<%d,%d>" % (bc, nvb))

    @property
    def passes(self):
        return -(-self.B // self.bc)

    @property
    def kernels(self):
        return frozenset(self.fwd + self.bwd)

    def __repr__(self):
        return self.name


ROWS = [
    Row(1, 24, 1, 1, 1),
    Row(1, 516, 1, 4, 2),      # forward 512 + 4 columns, backward 256 + 256 + 4
    Row(2, 8, 2, 1, 1),
    Row(2, 200, 2, 2, 2),
    Row(5, 128, 5, 1, 1),
    Row(5, 500, 5, 4, 2),      # the FB15k-237 shape
    Row(3, 40, 4, 1, 1),       # one partial pass
    Row(6, 300, 4, 3, 2),      # a full pass and a partial one; backward 256 + 44
    Row(8, 512, 4, 4, 2),      # two exact passes
    Row(100, 24, 4, 1, 1),     # gcn_block.exp's B at a small width: 25 passes
]
BY_NAME = {r.name: r for r in ROWS}


def table_kernels():
    return frozenset().union(*(r.kernels for r in ROWS))


def canonical(name):
    """`k_diagcoef_*<...>` of a demangled kernel name in the table's spelling (either demangler); None otherwise."""
    return block_walks.canonical(name, PREFIX)
