"""The message-walk kernels of the block-diagonal layer -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

One row per configuration the dispatch can reach: `use_rel_major` / `use_staged` and the dW-fusion decision in
csrc/api.cu, `launch_block_stg` (csrc/block_staged.cu), `launch_block_rel`, `launch_block_agg` and
`launch_block_dw` (csrc/rgcn_kernels.cu).  A row names the block_algo option, the environment knobs, the block size
s, a representative width d, and the walk kernels (with their template arguments) that one forward and one backward
of the layer launch.  tests/test_block_walk_table_host.py checks that the table and UNREACHABLE together name every
`k_block_*` instantiation of the built library; tests/test_gpu_block_walks.py runs every row and checks both the
kernels launched and the numbers they produce.

Kernel names are canonical: `k_block_team<8,1,true,true,4,3,2,8>` -- no spaces, bools as true/false."""
import re

# kernels that every layer call launches (weight-table re-layouts) or that belong to the slice-norm pass, not to a walk
LAYOUT = ("k_block_relayout", "k_block_unlayout")
NON_WALK = LAYOUT + ("k_block_sqnorm", "k_block_slice_sumsq")


def _b(x):
    return "true" if x else "false"


def team(s, fuse, tail):
    """k_block_team<S, NV=1, FUSE, TAIL, T=4, NTEAMS, NG, GS=8>: forward 4 teams x 3 groups, backward 3 x 2."""
    nteams, ng = (3, 2) if fuse else (4, 3)
    return "k_block_team<%d,1,%s,%s,4,%d,%d,8>" % (s, _b(fuse), _b(tail), nteams, ng)


def stg(s, nv, fuse, tail, nw, ng, gs, mode):
    return "k_block_stg<%d,%d,%s,%s,%d,%d,%d,%d>" % (s, nv, _b(fuse), _b(tail), nw, ng, gs, mode)


def rel(s, nv, fuse):
    return "k_block_rel<%d,%d,%s>" % (s, nv, _b(fuse))


def relg(g, fuse):
    return "k_block_relg<5,%d,%s>" % (g, _b(fuse))


def agg(s, nv):
    return "k_block_agg<%d,%d>" % (s, nv)


def dw(s, jc, nv):
    return "k_block_dw<%d,%d,%d>" % (s, jc, nv)


# the k_block_stg configurations of launch_block_stg, without TAIL: (S, NV, FUSE, NW, NG, GS, MODE)
S4_FWD, S4_BWD = (4, 1, False, 16, 3, 8, 1), (4, 1, True, 12, 2, 8, 1)
S8_FWD_CP, S8_FWD_TMA, S8_FWD_NV2 = (8, 1, False, 16, 3, 8, 1), (8, 1, False, 16, 3, 8, 0), (8, 2, False, 12, 2, 8, 0)
S8_BWD_CP, S8_BWD_TMA, S8_BWD_NV2 = (8, 1, True, 12, 2, 8, 1), (8, 1, True, 12, 2, 8, 0), (8, 2, True, 8, 2, 4, 0)
S16_FWD, S16_BWD = (16, 1, False, 16, 3, 8, 1), (16, 1, True, 8, 2, 8, 1)


def st(cfg, d):
    """the k_block_stg instantiation `cfg` launches at width d (TAIL: the last slab is narrower than NV*128)."""
    s, nv, fuse, nw, ng, gs, mode = cfg
    return stg(s, nv, fuse, d % (nv * 128) != 0, nw, ng, gs, mode)


class Row(object):
    def __init__(self, name, algo, env, s, d, fwd, bwd):
        self.name, self.algo, self.env, self.s, self.d = name, algo, dict(env), s, d
        self.fwd, self.bwd = tuple(fwd), tuple(bwd)

    @property
    def B(self):
        return self.d // self.s

    @property
    def kernels(self):
        return frozenset(self.fwd + self.bwd)

    @property
    def staged(self):
        """persistent TMA / cp.async-staged kernels (one CTA per SM, dynamic work distribution)"""
        return any(k.startswith(("k_block_team", "k_block_stg")) for k in self.kernels)

    def __repr__(self):
        return self.name


def _rows():
    R = []
    add = lambda *a: R.append(Row(*a))
    # ---- block_algo = -1 (the default): TMA-staged kernels for s in {4, 8, 16} -------------------------------------
    # team kernels: 384 < d <= 512, s in {4, 8}, no RGCN_STG_FWD / _BWD for that direction
    add("team-s8", -1, {}, 8, 512, [team(8, 0, 0)], [team(8, 1, 0)])
    add("team-s8-tail", -1, {}, 8, 400, [team(8, 0, 1)], [team(8, 1, 1)])
    add("team-s4", -1, {}, 4, 512, [team(4, 0, 0)], [team(4, 1, 0)])
    add("team-s4-tail", -1, {}, 4, 500, [team(4, 0, 1)], [team(4, 1, 1)])
    add("team-s8-unfused", -1, {"RGCN_NO_FUSE_DW": "1"}, 8, 512, [team(8, 0, 0)], [team(8, 0, 0), dw(8, 8, 2)])
    add("team-off-s8-tail", -1, {"RGCN_STG_TEAM": "0"}, 8, 448, [st(S8_FWD_CP, 448)], [st(S8_BWD_CP, 448)])
    # a forward knob turns the team kernel off for the forward only
    add("team-bwd-only-s4", -1, {"RGCN_STG_FWD": "2"}, 4, 512, [st(S4_FWD, 512)], [team(4, 1, 0)])
    # per-warp rings, s = 8
    add("stg-s8", -1, {}, 8, 256, [st(S8_FWD_CP, 256)], [st(S8_BWD_CP, 256)])
    add("stg-s8-tail", -1, {}, 8, 264, [st(S8_FWD_CP, 264)], [st(S8_BWD_CP, 264)])
    add("stg-s8-d640", -1, {}, 8, 640, [st(S8_FWD_CP, 640)], [st(S8_BWD_CP, 640)])
    add("stg-s8-d128", -1, {}, 8, 128, [st(S8_FWD_TMA, 128)], [st(S8_BWD_CP, 128)])   # d <= 128: TMA forward
    add("stg-s8-d64", -1, {}, 8, 64, [st(S8_FWD_TMA, 64)], [st(S8_BWD_CP, 64)])
    add("stg-s8-d128-bwd3", -1, {"RGCN_STG_BWD": "3"}, 8, 128, [st(S8_FWD_TMA, 128)], [st(S8_BWD_CP, 128)])
    add("stg-s8-fwd2-bwd0", -1, {"RGCN_STG_FWD": "2", "RGCN_STG_BWD": "0"}, 8, 512,
        [st(S8_FWD_TMA, 512)], [st(S8_BWD_TMA, 512)])
    add("stg-s8-fwd2-bwd0-tail", -1, {"RGCN_STG_FWD": "2", "RGCN_STG_BWD": "0"}, 8, 264,
        [st(S8_FWD_TMA, 264)], [st(S8_BWD_TMA, 264)])
    add("stg-s8-fwd0-bwd3", -1, {"RGCN_STG_FWD": "0", "RGCN_STG_BWD": "3"}, 8, 512,
        [st(S8_FWD_NV2, 512)], [st(S8_BWD_NV2, 512)])
    add("stg-s8-fwd0-bwd3-tail", -1, {"RGCN_STG_FWD": "0", "RGCN_STG_BWD": "3"}, 8, 264,
        [st(S8_FWD_NV2, 264)], [st(S8_BWD_NV2, 264)])
    add("stg-s8-fwd3-bwd1", -1, {"RGCN_STG_FWD": "3", "RGCN_STG_BWD": "1"}, 8, 512,
        [st(S8_FWD_CP, 512)], [st(S8_BWD_CP, 512)])
    add("stg-s8-tail-unfused", -1, {"RGCN_NO_FUSE_DW": "1"}, 8, 264,
        [st(S8_FWD_CP, 264)], [st(S8_FWD_CP, 264), dw(8, 8, 2)])
    # s = 4 and s = 16
    add("stg-s4", -1, {}, 4, 256, [st(S4_FWD, 256)], [st(S4_BWD, 256)])
    add("stg-s4-tail", -1, {}, 4, 260, [st(S4_FWD, 260)], [st(S4_BWD, 260)])
    add("stg-s16", -1, {}, 16, 512, [st(S16_FWD, 512)], [st(S16_BWD, 512)])
    add("stg-s16-tail", -1, {}, 16, 144, [st(S16_FWD, 144)], [st(S16_BWD, 144)])
    add("stg-s16-d1024", -1, {}, 16, 1024, [st(S16_FWD, 1024)], [st(S16_BWD, 1024)])
    # ---- s = 5 (gcn_block.exp): weight-id major with the rows in registers -----------------------------------------
    add("relg4", -1, {}, 5, 500, [relg(4, 0)], [relg(4, 1)])
    add("relg2", -1, {"RGCN_REL_GROUP": "2"}, 5, 500, [relg(2, 0)], [relg(2, 1)])
    add("relg4-s5-unfused", -1, {"RGCN_FUSE_DW_S5": "0"}, 5, 500, [relg(4, 0)], [relg(4, 0), dw(5, 5, 4)])
    add("relg4-unfused", -1, {"RGCN_NO_FUSE_DW": "1"}, 5, 500, [relg(4, 0)], [relg(4, 0), dw(5, 5, 4)])
    for d, nv in ((120, 1), (240, 2), (380, 3), (500, 4)):   # one warp per slab: no fused form, dW in its own walk
        add("rel-s5-group1-d%d" % d, -1, {"RGCN_REL_GROUP": "1"}, 5, d, [rel(5, nv, 0)], [rel(5, nv, 0), dw(5, 5, nv)])
    # ---- block_algo = 1: weight-id major with the rows in registers (the fused backward forces NV = 1) -----------
    add("rel-s8", 1, {}, 8, 512, [rel(8, 2, 0)], [rel(8, 1, 1)])
    add("rel-s8-tail", 1, {}, 8, 264, [rel(8, 2, 0)], [rel(8, 1, 1)])
    add("rel-s8-d128", 1, {}, 8, 128, [rel(8, 1, 0)], [rel(8, 1, 1)])
    add("rel-s8-nv1", 1, {"RGCN_REL_NV": "1"}, 8, 512, [rel(8, 1, 0)], [rel(8, 1, 1)])
    add("rel-s8-unfused", 1, {"RGCN_NO_FUSE_DW": "1"}, 8, 512, [rel(8, 2, 0)], [rel(8, 2, 0), dw(8, 8, 2)])
    add("rel-s4", 1, {}, 4, 512, [rel(4, 4, 0)], [rel(4, 1, 1)])
    add("rel-s4-tail", 1, {}, 4, 260, [rel(4, 3, 0)], [rel(4, 1, 1)])
    for nv in (1, 2, 3):
        add("rel-s4-nv%d" % nv, 1, {"RGCN_REL_NV": str(nv)}, 4, 512, [rel(4, nv, 0)], [rel(4, 1, 1)])
    add("rel-s4-unfused", 1, {"RGCN_NO_FUSE_DW": "1"}, 4, 256, [rel(4, 2, 0)], [rel(4, 2, 0), dw(4, 4, 2)])
    add("rel-s16", 1, {}, 16, 512, [rel(16, 1, 0)], [rel(16, 1, 1)])
    add("rel-s16-tail", 1, {}, 16, 144, [rel(16, 1, 0)], [rel(16, 1, 1)])
    add("relg4-algo1", 1, {}, 5, 500, [relg(4, 0)], [relg(4, 1)])
    # ---- block_algo = 0: destination-major (NV = min(4, ceil(d / 128)) quads per lane) -------------------------------
    for s, dws in ((4, ((128, 1), (256, 2), (384, 3), (512, 4))), (5, ((120, 1), (240, 2), (380, 3), (500, 4))),
                   (8, ((128, 1), (256, 2), (384, 3), (1024, 4))), (16, ((128, 1), (144, 2), (384, 3), (512, 4)))):
        for d, nv in dws:
            jc_nv = {4: (4, nv), 5: (5, nv), 8: (8, 1 if nv == 1 else 2), 16: (16, 1)}[s]
            add("agg-s%d-d%d" % (s, d), 0, {}, s, d, [agg(s, nv)], [agg(s, nv), dw(s, *jc_nv)])
    # ---- block sizes without a dedicated kernel (here s = 6): destination-major under every block_algo -------------
    for d, nv in ((24, 1), (192, 2), (384, 3), (504, 4)):
        add("agg-generic-s6-d%d" % d, -1, {}, 6, d, [agg(0, nv)], [agg(0, nv), dw(0, 4, nv)])
    return R


ROWS = _rows()
BY_NAME = {r.name: r for r in ROWS}

# compiled, but no dispatch decision leads to them
UNREACHABLE = {
    rel(4, 2, 1): "the fused backward forces NV = 1 and RGCN_REL_NV can only lower it",
    rel(4, 3, 1): "the fused backward forces NV = 1 and RGCN_REL_NV can only lower it",
    rel(4, 4, 1): "the fused backward forces NV = 1 and RGCN_REL_NV can only lower it",
    rel(8, 2, 1): "the fused backward forces NV = 1 and RGCN_REL_NV can only lower it",
}


def table_kernels():
    return frozenset().union(*(r.kernels for r in ROWS))


def canonical(name, prefix="k_block_"):
    """`<prefix>*<...>` of a demangled kernel name, in the table's spelling: cu++filt writes `<(int)8, (bool)0>`,
    the CUDA profiler `<8, false>`.  None when the name is not a kernel of that family (default: the block
    layer's)."""
    m = re.search(r"\b(%s\w+)(<[^<>]*>)?" % re.escape(prefix), name)
    if not m:
        return None
    if not m.group(2):
        return m.group(1)
    args = []
    for a in m.group(2)[1:-1].split(","):
        a = a.strip()
        if a.startswith("(bool)"):
            a = "true" if a[6:] not in ("0", "false") else "false"
        elif a.startswith("("):
            a = a[a.index(")") + 1:]
        args.append(a)
    return "%s<%s>" % (m.group(1), ",".join(args))
