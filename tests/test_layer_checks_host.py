"""Argument checks of the layer, block aggregate and slice-norm entry points without a GPU: the exact return code of
every bad argument, one at a time, and of valid arguments on a host-only graph.

The block and basis entry points check the graph first, so on a host-only graph every argument error after a null
graph reads RGCN_ERR_NODEVICE.  The one-hot, per-channel and diagonal entry points check shape, pointers and workspace
first, so those errors are reported as such even for a host-only graph."""
import ctypes

import numpy as np
import pytest

from relationprediction_b200 import _lib, ops

INVALID, WORKSPACE, NODEVICE = -1, -4, -5

# argument kinds: g graph, d width, B blocks, P required pointer, O optional pointer (passed as NULL), k keep,
# r relu (passed as 1, so `out` is read), a accumulate flag, w workspace, n workspace bytes, s stream
ENTRIES = {
    # name: (argument kinds, pointer names, workspace bytes function, takes `backward`, checks the graph first)
    "rgcn_block_forward": ("gdBPPPPOkrPwns", "H Wf Wb Wself out", "rgcn_block_workspace_bytes", 0, True),
    "rgcn_block_backward": ("gdBPPPPOkrPPPPPPwns", "H Wf Wb Wself out dOut dH dWf dWb dWself",
                            "rgcn_block_workspace_bytes", 1, True),
    "rgcn_basis_forward": ("gdBPPPPPPOkrPPwns", "H Vf Vb Cf Cb Wself out saved", "rgcn_basis_workspace_bytes", 0,
                           True),
    "rgcn_basis_backward": ("gdBPPPPPPOkrPPPPPPPPPwns", "H Vf Vb Cf Cb Wself out saved dOut dH dVf dVb dCf dCb dWself",
                            "rgcn_basis_workspace_bytes", 1, True),
    "rgcn_basis_onehot_forward": ("gdBPPPPPOkrPwns", "Wf Wb Cf Cb Wself out", "rgcn_basis_onehot_workspace_bytes", 0,
                                  False),
    "rgcn_basis_onehot_backward": ("gdBPPPPOkrPPPPPPPwns", "Wf Wb Cf Cb out dOut dWf dWb dCf dCb dWself",
                                   "rgcn_basis_onehot_workspace_bytes", 1, False),
    "rgcn_basis_diagcoef_forward": ("gdBPPPPPPPOkrPPwns", "H Vf Vb Cf Cb Wself b out saved",
                                    "rgcn_basis_diagcoef_workspace_bytes", 0, False),
    "rgcn_basis_diagcoef_backward": ("gdBPPPPPPOkrPPPPPPPPPPwns",
                                     "H Vf Vb Cf Cb Wself out saved dOut dH dVf dVb dCf dCb dWself db",
                                     "rgcn_basis_diagcoef_workspace_bytes", 1, False),
    "rgcn_diag_forward": ("gdPPPPPOkrPwns", "H Df Db Wself b out", "rgcn_diag_workspace_bytes", 0, False),
    "rgcn_diag_backward": ("gdPPPPOkrPPPPPPPOwns", "H Df Db Wself out dOut dH dDf dDb dWself db",
                           "rgcn_diag_workspace_bytes", 1, False),
    "rgcn_block_aggregate": ("gdBPPPPwns", "X Wf Wb out", "rgcn_block_aggregate_workspace_bytes", 0, True),
    "rgcn_block_aggregate_backward": ("gdBPPPPPPPawns", "X Wf Wb G dX dWf dWb",
                                      "rgcn_block_aggregate_workspace_bytes", 1, True),
    "rgcn_block_slice_sumsq": ("gdBPPPwns", "H G sumsq2", "rgcn_block_slice_sumsq_workspace_bytes", None, True),
}
BLOCK = {"rgcn_block_forward", "rgcn_block_backward", "rgcn_block_aggregate", "rgcn_block_aggregate_backward",
         "rgcn_block_slice_sumsq"}
D, B = 8, 2


@pytest.fixture(scope="module")
def host_graph():
    rng = np.random.RandomState(0)
    V, R, E = 12, 3, 40
    tri = np.stack([rng.randint(0, V, E), rng.randint(0, R, E), rng.randint(0, V, E)], 1).astype(np.int32)
    return ops.Graph(tri, V, R)   # host-only graph


def _workspace_bytes(lib, name, g, d=D, b=B):
    kinds, _, ws_fn, backward, _ = ENTRIES[name]
    args = [g, d] + ([b] if "B" in kinds else []) + ([] if backward is None else [backward])
    return getattr(lib, ws_fn)(*args)


def _call(lib, name, g, buf, d=D, b=B, keep=1.0, null=None, ws_bytes=None, graph=True):
    kinds, pointers, _, _, _ = ENTRIES[name]
    pointers = pointers.split()
    if ws_bytes is None:
        ws_bytes = _workspace_bytes(lib, name, g)
    args, p = [], 0
    for kind in kinds:
        if kind == "g":
            args.append(g if graph else None)
        elif kind == "d":
            args.append(d)
        elif kind == "B":
            args.append(b)
        elif kind == "P":
            args.append(None if pointers[p] == null else buf)
            p += 1
        elif kind == "O":
            args.append(None)
        elif kind == "k":
            args.append(keep)
        elif kind in "ra":
            args.append(1)
        elif kind == "w":
            args.append(None if null == "workspace" else buf)
        elif kind == "n":
            args.append(ws_bytes)
        elif kind == "s":
            args.append(None)
    assert p == len(pointers)
    return getattr(lib, name)(*args)


@pytest.mark.parametrize("name", sorted(ENTRIES))
def test_workspace_bytes_reject_bad_arguments(name, host_graph):
    lib = _lib.load()
    kinds = ENTRIES[name][0]
    g = host_graph.handle
    assert _workspace_bytes(lib, name, g) > 0
    assert _workspace_bytes(lib, name, None) == INVALID
    assert _workspace_bytes(lib, name, g, d=0) == INVALID
    if "B" in kinds:
        assert _workspace_bytes(lib, name, g, b=0) == INVALID
    if name in BLOCK:
        assert _workspace_bytes(lib, name, g, d=12, b=8) == INVALID   # d % B != 0


@pytest.mark.parametrize("name", sorted(ENTRIES))
def test_entry_points_return_exact_codes(name, host_graph):
    lib = _lib.load()
    kinds, pointers, _, _, graph_first = ENTRIES[name]
    g = host_graph.handle
    need = _workspace_bytes(lib, name, g)
    buf = ctypes.create_string_buffer(max(need, 1 << 16))
    # on a host-only graph, the graph-first entry points stop at the device check
    arg_error = NODEVICE if graph_first else INVALID
    cases = [(dict(graph=False), INVALID), (dict(d=0), arg_error), (dict(d=6, b=1 if "B" in kinds else B), arg_error),
             (dict(null="workspace"), arg_error), (dict(ws_bytes=need - 1), NODEVICE if graph_first else WORKSPACE),
             ({}, NODEVICE)]
    if "B" in kinds:
        cases.append((dict(b=0), arg_error))
    if name in BLOCK:
        cases.append((dict(d=12, b=8), arg_error))   # d % B != 0
    if "k" in kinds:
        cases += [(dict(keep=0.0), arg_error), (dict(keep=-1.0), arg_error)]
    cases += [(dict(null=p), arg_error) for p in pointers.split()]
    for kw, expected in cases:
        assert _call(lib, name, g, buf, **kw) == expected, (kw, lib.rgcn_last_error())
        if expected == NODEVICE:
            assert b"host-only" in lib.rgcn_last_error()
