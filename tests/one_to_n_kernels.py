"""The kernels of 1-N training (ops.one_to_n_loss, ops.OneToNLabels.rows) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

One row per call: the exact kernels one library call launches, in launch order, for queries of both sides sorted by
side (two runs) that fit one internal pass.  "loss" is a forward that needs no gradient (the loss only); "fwd" is a
forward whose inputs need gradients (the whole pass with the gradient GEMMs, for the loss alone); "bwd" scales that
gradient and adds the L2 term (rgcn_one_to_n_finish, the same for both decoders).  csrc/onen.cu holds the `k_onen_*`
kernels; the rows also name the rank prepare kernels, the codes split and the GEMMs of gemm_tf32x3.cu
(`k_gemm_tf32x3<5>` is the BCE epilogue).  tests/test_one_to_n_kernel_table_host.py checks that the table names every
`k_onen_*` kernel of the built library and that the others exist; tests/test_gpu_one_to_n.py checks with the profiler
that each row launches exactly these."""
import block_walks

PREFIX = "k_onen_"


def _row(prepare, query_bwd, backward):
    head = ("k_split_b", "k_onen_reg", prepare, prepare, "k_gemm_tf32x3<5>")
    if backward:
        head += ("k_gemm_tn_tf32x3", "k_split_b", "k_gemm_tf32x3<0>", query_bwd, query_bwd)
    return head + ("k_onen_loss_reduce",)


FINISH = ("k_onen_scale", "k_onen_scale", "k_onen_query_bwd", "k_onen_query_bwd")
ROWS = {
    ("labels", "loss"): ("k_onen_labels", "k_onen_labels"),
    ("distmult", "loss"): _row("k_rank_prepare", None, False),
    ("distmult", "fwd"): _row("k_rank_prepare", "k_onen_query_bwd", True),
    ("distmult", "bwd"): FINISH,
    ("complex4", "loss"): _row("k_complex_rank_prepare<4>", None, False),
    ("complex4", "fwd"): _row("k_complex_rank_prepare<4>", "k_onen_complex_query_bwd<4>", True),
    ("complex4", "bwd"): FINISH,
    ("complex2", "loss"): _row("k_complex_rank_prepare<2>", None, False),
    ("complex2", "fwd"): _row("k_complex_rank_prepare<2>", "k_onen_complex_query_bwd<2>", True),
    ("complex2", "bwd"): FINISH,
}
# kernels of other families the rows name (they must exist in the library, but are not checked for completeness)
SHARED = ("k_split_b", "k_rank_prepare", "k_complex_rank_prepare<4>", "k_complex_rank_prepare<2>", "k_gemm_tf32x3<5>",
          "k_gemm_tn_tf32x3", "k_gemm_tf32x3<0>")


def table_kernels():
    return frozenset(k for row in ROWS.values() for k in row if k.startswith(PREFIX))


def canonical(name, prefix=PREFIX):
    """`<prefix>*<...>` of a demangled kernel name in the table's spelling (either demangler); None otherwise."""
    return block_walks.canonical(name, prefix)
