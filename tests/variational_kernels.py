"""The kernels of the variational head (ops.variational) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

One row per variant and direction: the exact kernels one call launches, in launch order.  csrc/variational.cu holds
the `k_var_*` kernels; the gcn variant also runs the interleaving weight split `k_split_b_interleave` and the GEMMs of
gemm_tf32x3.cu (`k_gemm_tf32x3<3>` is the variational epilogue).  tests/test_variational_kernel_table_host.py checks
that the table names every `k_var_*` kernel of the built library and that the others exist; tests/test_gpu_variational.py
checks with the profiler that each row launches exactly these kernels."""
import block_walks

PREFIX = "k_var_"

ROWS = {
    ("embedding", "fwd"): ("k_var_emb_fwd", "k_var_kl_reduce"),
    ("embedding", "bwd"): ("k_var_emb_bwd",),
    ("gcn", "fwd"): ("k_split_b_interleave", "k_gemm_tf32x3<3>", "k_var_kl_reduce"),
    ("gcn", "bwd"): ("k_var_prologue", "k_var_colsum_finish", "k_gemm_tn_tf32x3", "k_var_deinterleave",
                     "k_split_b_interleave", "k_gemm_tf32x3<0>"),
}
# kernels of other families the rows name (they must exist in the library, but are not checked for completeness)
SHARED = ("k_split_b_interleave", "k_gemm_tf32x3<3>", "k_gemm_tn_tf32x3", "k_gemm_tf32x3<0>")


def table_kernels():
    return frozenset(k for row in ROWS.values() for k in row if k.startswith(PREFIX))


def canonical(name, prefix=PREFIX):
    """`<prefix>*<...>` of a demangled kernel name in the table's spelling (either demangler); None otherwise."""
    return block_walks.canonical(name, prefix)
