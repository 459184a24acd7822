"""The kernels of the 3xTF32 GEMM library (csrc/gemm_tf32x3.cu) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

One row per kernel the file builds: the canonical kernel name and the public entry point that reaches it.
tests/test_gemm_kernel_table_host.py checks that the rows name exactly the `k_gemm_*` and `k_split_*` kernels of the
built library; tests/test_gpu_gemm_epilogues.py runs every row against float64 at the GEMM's tile, k-block,
stage-ring and persistent-walk boundaries and checks with the profiler that each row's entry point launched its
kernel.

Kernel names are canonical (block_walks.canonical after the namespace qualifiers are dropped):
`k_gemm_tf32x3<5>`, `k_gemm_ensemble<EnsRankEpi>`."""
import re

import block_walks

PREFIXES = ("k_gemm_", "k_split_")

# kernel -> the public entry point that launches it
ROWS = {
    "k_gemm_tf32x3<0>": "rgcn_gemm_tf32x3 / ops.gemm_tf32x3 (StoreEpi)",
    "k_gemm_tf32x3<1>": "DistMultRanker / ComplexRanker .rank and .rank_relations (RankEpi)",
    "k_gemm_tf32x3<2>": "ops.highway (HighwayEpi)",
    "k_gemm_tf32x3<3>": "ops.variational (VarEpi)",
    "k_gemm_tf32x3<4>": "DistMultRanker / ComplexRanker .top_k and .top_k_relations (TopKEpi)",
    "k_gemm_tf32x3<5>": "ops.one_to_n_loss (BceEpi)",
    "k_gemm_tf32x3<6>": "ops.compgcn_layer (BiasActEpi)",
    "k_gemm_tn_tf32x3": "rgcn_gemm_tn_tf32x3 / ops.gemm_tn_tf32x3",
    "k_gemm_ensemble<EnsRankEpi>": "EnsembleRanker.rank / .rank_relations",
    "k_gemm_ensemble<EnsTopKEpi>": "EnsembleRanker.top_k / .top_k_relations",
    "k_split_b": "ops.gemm_tf32x3 (the pre-split of B, both orientations)",
    "k_split_b_interleave": "ops.variational (the pre-split of [W_mu, W_sigma] interleaved)",
    "k_split_trunc": "EnsembleRanker.rank / .top_k (the in-place split of the query rows)",
}

# Boundaries of a kernel that no public entry point can reach, and why.  The GPU tests cover what is reachable.
UNREACHABLE = {
    "k_gemm_tf32x3<0> with K = 0": "rgcn_gemm_tf32x3 refuses K <= 0 before any launch; the launcher's memset path "
                                   "for an empty contraction serves no public caller",
    "k_gemm_tf32x3<5> Gt padding (ldgt > M)": "Gt is workspace of the 1-N body (ldgt = M rounded up to 8), never "
                                              "returned: it is checked through dcodes / drel, which the padding "
                                              "columns would corrupt if written",
    "k_gemm_tf32x3<5> g_scale null with Gt": "ops.one_to_n_loss passes g_scale on the device exactly when it asks for "
                                             "Gt, and neither for the loss alone",
    "k_gemm_tf32x3<2>/<3> padded leading dimensions": "the highway and variational launchers take contiguous "
                                                       "[M, d] / [M, 2w] operands only",
}

_QUALIFIER = re.compile(r"(\(anonymous namespace\)|<unnamed>)::")


def canonical(name):
    """`k_gemm_*<...>` / `k_split_*` of a demangled kernel name (either demangler), None for other kernels."""
    name = _QUALIFIER.sub("", name)
    for p in PREFIXES:
        c = block_walks.canonical(name, p)
        if c is not None:
            return c
    return None


def table_kernels():
    return frozenset(ROWS)
