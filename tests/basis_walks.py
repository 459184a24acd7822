"""The aggregation walks of the basis layer -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

One row per (layer kind, B, d) that reaches a distinct set of walk kernels.  The dispatch lives in
`launch_basis_agg_b` / `launch_basis_agg_t` / `launch_basis_dc` (csrc/rgcn_kernels.cu) and
`launch_basis_onehot_push` (csrc/basis_onehot.cu):
  - bases per pass BC = B for B in {1, 2, 5}, else 4 (ceil(B / 4) passes over the bases);
  - quads per lane NV = min(ceil(d / 128), 4), capped at 2 for the fused one-hot backward (`DC = true`);
  - column slabs on grid.y: ceil(d / (NV * 128)).
A row states BC and NV explicitly; tests/test_basis_walk_table_host.py checks them against these rules and checks
that the table names every `k_basis_*` instantiation of the built library; tests/test_gpu_basis_walks.py runs every
row and checks both the kernels launched and the numbers they produce.

Kernels per forward + backward:
  feature input ("feat", rgcn_basis_forward / _backward): k_basis_agg<BC,NV,0,false> forward;
      k_basis_dc<BC,NV> and k_basis_agg<BC,NV,1,false> backward;
  one-hot input ("onehot", rgcn_basis_onehot_forward / _backward): k_basis_onehot_push<NV> forward;
      k_basis_agg<BC,min(NV,2),1,true> backward.

Kernel names are canonical: `k_basis_agg<4,2,1,true>` -- no spaces, bools as true/false."""
import block_walks

PREFIX = "k_basis_"

# kernels the basis paths launch besides the walks: row clearing of split rows, dropout / ReLU, the gradient prologue,
# and the 3xTF32 GEMMs with their operand split
NON_WALK = ("k_zero_rows", "k_mask_relu", "k_grad_prologue", "k_gemm_tf32x3", "k_gemm_tn_tf32x3", "k_split_b")


def _b(x):
    return "true" if x else "false"


def agg(bc, nv, layout, dc):
    return "k_basis_agg<%d,%d,%d,%s>" % (bc, nv, layout, _b(dc))


def dc(bc, nv):
    return "k_basis_dc<%d,%d>" % (bc, nv)


def push(nv):
    return "k_basis_onehot_push<%d>" % nv


def bc_rule(B):
    """bases per pass of launch_basis_agg_b / launch_basis_dc"""
    return B if B in (1, 2, 5) else 4


def nv_rule(d, dc_variant=False):
    """quads per lane of launch_basis_agg_t / launch_basis_dc_t / launch_basis_onehot_push"""
    nv = min((d + 127) // 128, 4)
    return min(nv, 2) if dc_variant else nv


def slabs(d, nv):
    return (d + nv * 128 - 1) // (nv * 128)


class Row(object):
    """kind 'feat' or 'onehot'; bc / nv as the dispatch picks them for the walks (for one-hot rows: nv of the push,
    nv_dc of the fused backward walk)."""

    def __init__(self, kind, B, d, bc, nv, nv_dc=None):
        self.kind, self.B, self.d, self.bc, self.nv, self.nv_dc = kind, B, d, bc, nv, nv_dc
        self.name = "%s-B%d-d%d" % (kind, B, d)
        if kind == "feat":
            self.fwd, self.bwd = (agg(bc, nv, 0, False),), (dc(bc, nv), agg(bc, nv, 1, False))
        else:
            self.fwd, self.bwd = (push(nv),), (agg(bc, nv_dc, 1, True),)

    @property
    def onehot(self):
        return self.kind == "onehot"

    @property
    def passes(self):
        return -(-self.B // self.bc)

    @property
    def kernels(self):
        return frozenset(self.fwd + self.bwd)

    def __repr__(self):
        return self.name


def _rows():
    R = []
    feat = lambda B, d, bc, nv: R.append(Row("feat", B, d, bc, nv))
    onehot = lambda B, d, bc, nv, nv_dc: R.append(Row("onehot", B, d, bc, nv, nv_dc))
    # ---- feature input: every (BC, NV) pair, narrow tails and exact widths, one and two slabs -------------------------
    feat(1, 24, 1, 1)
    feat(1, 200, 1, 2)
    feat(1, 300, 1, 3)
    feat(1, 516, 1, 4)      # two slabs: 512 + 4 columns
    feat(2, 8, 2, 1)
    feat(2, 256, 2, 2)
    feat(2, 384, 2, 3)
    feat(2, 1024, 2, 4)     # two full slabs
    feat(5, 128, 5, 1)
    feat(5, 200, 5, 2)
    feat(5, 300, 5, 3)
    feat(5, 500, 5, 4)
    feat(5, 640, 5, 4)      # two slabs: 512 + 128
    feat(3, 40, 4, 1)       # one partial pass
    feat(4, 252, 4, 2)
    feat(4, 640, 4, 4)      # two slabs
    feat(6, 300, 4, 3)      # a full pass and a partial one
    feat(8, 512, 4, 4)      # two exact passes
    feat(9, 1000, 4, 4)     # three passes (the last holds one basis), two slabs: 512 + 488
    # ---- one-hot input: the 8 fused-dC pairs and every push width ------------------------------------------------------
    onehot(1, 24, 1, 1, 1)
    onehot(1, 300, 1, 3, 2)    # backward: two slabs of 256 + 44
    onehot(2, 128, 2, 1, 1)
    onehot(2, 1024, 2, 4, 2)   # push: two slabs; backward: four
    onehot(5, 40, 5, 1, 1)
    onehot(5, 200, 5, 2, 2)
    onehot(3, 516, 4, 4, 2)    # partial pass; push 512 + 4, backward 256 + 256 + 4
    onehot(9, 120, 4, 1, 1)    # three passes
    return R


ROWS = _rows()
BY_NAME = {r.name: r for r in ROWS}


def table_kernels():
    return frozenset().union(*(r.kernels for r in ROWS))


def canonical(name):
    """`k_basis_*<...>` of a demangled kernel name in the table's spelling (either demangler); None otherwise."""
    return block_walks.canonical(name, PREFIX)
