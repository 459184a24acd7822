"""Host-side operators over the C-ABI: graph handle + autograd Functions.

PyTorch is used for storage (CUDA tensors), streams and autograd bookkeeping only: every
forward/backward below is ONE call into librgcn_b200.so (include/rgcn_b200.h).  There is no CPU or
eager-torch fallback: tensors that are not CUDA fp32 raise.
"""
import ctypes
import os

import numpy as np
import torch

from . import _lib

_NORM = {"canonical": _lib.RGCN_NORM_CANONICAL, "explicit": _lib.RGCN_NORM_EXPLICIT,
         "none": _lib.RGCN_NORM_NONE, "relation": _lib.RGCN_NORM_RELATION}


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _np_ptr(a):
    return ctypes.c_void_p(a.ctypes.data) if a is not None else ctypes.c_void_p(0)


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _check_cuda_f32(name, t, shape=None):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32):
        raise _lib.RgcnError("%s must be a CUDA float32 tensor (no CPU fallback exists)" % name)
    if not t.is_contiguous():
        raise _lib.RgcnError("%s must be contiguous" % name)
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise _lib.RgcnError("%s has shape %s, expected %s" % (name, tuple(t.shape), tuple(shape)))


class Graph:
    """Prepared message-passing graph (opaque C handle).

    Replaces Representation/MessageGraph (extras/graph_representations.py): triples [E,3] (s,r,o)
    -> 2E messages, per-direction 1/in-degree normalisation, three sorted views + warp work lists.
    norm_mode: "canonical" (1 / #messages of the direction into the destination), "relation" (1 / #messages with
    the same destination and weight id: the paper's c_{i,r}), "explicit" (norm_f / norm_b given) or "none".
    `device=None` builds the host structure only (used by the CPU tests of the index work).
    """

    def __init__(self, triples, n_entities, n_relations, norm_mode="canonical", norm_f=None,
                 norm_b=None, device=None, _handle=None):
        self._lib = _lib.load()
        self._h = ctypes.c_void_p(0)
        self.device = device
        if _handle is not None:
            self._h = _handle
        else:
            tri = np.ascontiguousarray(np.asarray(triples, dtype=np.int32).reshape(-1, 3))
            nf = None if norm_f is None else np.ascontiguousarray(norm_f, dtype=np.float32)
            nb = None if norm_b is None else np.ascontiguousarray(norm_b, dtype=np.float32)
            dev = -1 if device is None else int(device)
            st = _stream(device) if device is not None else ctypes.c_void_p(0)
            rc = self._lib.rgcn_graph_create(_np_ptr(tri), tri.shape[0], int(n_entities),
                                             int(n_relations), _NORM[norm_mode], _np_ptr(nf),
                                             _np_ptr(nb), dev, st, ctypes.byref(self._h))
            _lib.check(rc, "rgcn_graph_create")
        info = self.info()
        self.M, self.V_dst, self.V_src, self.n_relw = info[0], info[1], info[2], info[3]

    @classmethod
    def from_messages(cls, dst, src, relw, norm, V_dst, V_src, n_relw, device=None):
        lib = _lib.load()
        dst = np.ascontiguousarray(dst, dtype=np.int32)
        src = np.ascontiguousarray(src, dtype=np.int32)
        relw = np.ascontiguousarray(relw, dtype=np.int32)
        norm = np.ascontiguousarray(norm, dtype=np.float32)
        h = ctypes.c_void_p(0)
        dev = -1 if device is None else int(device)
        st = _stream(device) if device is not None else ctypes.c_void_p(0)
        rc = lib.rgcn_graph_create_messages(_np_ptr(dst), _np_ptr(src), _np_ptr(relw), _np_ptr(norm),
                                            dst.shape[0], int(V_dst), int(V_src), int(n_relw), dev,
                                            st, ctypes.byref(h))
        _lib.check(rc, "rgcn_graph_create_messages")
        return cls(None, 0, 0, device=device, _handle=h)

    @staticmethod
    def _dev_i32(name, t, n=None):
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.int32 and t.is_contiguous()):
            raise _lib.RgcnError("%s must be a contiguous CUDA int32 tensor" % name)
        if n is not None and t.numel() != n:
            raise _lib.RgcnError("%s has %d elements, expected %d" % (name, t.numel(), n))
        return t

    @classmethod
    def from_device_triples(cls, triples, n_entities, n_relations, norm_mode="canonical", norm_f=None, norm_b=None):
        """Graph from an int32 [E,3] (s,r,o) tensor that already lives on the GPU (rgcn_graph_create_device):
        the edge list never visits the host."""
        lib = _lib.load()
        tri = cls._dev_i32("triples", triples)
        if tri.dim() != 2 or tri.shape[1] != 3:
            raise _lib.RgcnError("triples must be [E,3]")
        for nm, t in (("norm_f", norm_f), ("norm_b", norm_b)):
            if t is not None:
                _check_cuda_f32(nm, t, (tri.shape[0],))
        dev = tri.device.index if tri.device.index is not None else torch.cuda.current_device()
        h = ctypes.c_void_p(0)
        rc = lib.rgcn_graph_create_device(_ptr(tri), tri.shape[0], int(n_entities), int(n_relations),
                                          _NORM[norm_mode], _ptr(norm_f), _ptr(norm_b), dev, _stream(tri.device),
                                          ctypes.byref(h))
        _lib.check(rc, "rgcn_graph_create_device")
        return cls(None, 0, 0, device=dev, _handle=h)

    @classmethod
    def from_device_messages(cls, dst, src, relw, norm, V_dst, V_src, n_relw):
        """Graph from message arrays resident on the GPU (rgcn_graph_create_messages_device)."""
        lib = _lib.load()
        M = dst.numel()
        cls._dev_i32("dst", dst)
        cls._dev_i32("src", src, M)
        cls._dev_i32("relw", relw, M)
        _check_cuda_f32("norm", norm, (M,))
        dev = dst.device.index if dst.device.index is not None else torch.cuda.current_device()
        h = ctypes.c_void_p(0)
        rc = lib.rgcn_graph_create_messages_device(_ptr(dst), _ptr(src), _ptr(relw), _ptr(norm), M, int(V_dst),
                                                   int(V_src), int(n_relw), dev, _stream(dst.device),
                                                   ctypes.byref(h))
        _lib.check(rc, "rgcn_graph_create_messages_device")
        return cls(None, 0, 0, device=dev, _handle=h)

    def info(self):
        arr = (ctypes.c_int64 * 16)()
        _lib.check(self._lib.rgcn_graph_info(self._h, arr), "rgcn_graph_info")
        return [int(x) for x in arr]

    def export(self, which):
        n = self._lib.rgcn_graph_export_bytes(self._h, which)
        if n < 0:
            _lib.check(int(n), "rgcn_graph_export_bytes")
        dtype = np.float32 if which in (_lib.X_DST_NORM, _lib.X_SRC_NORM, _lib.X_REL_NORM,
                                        _lib.X_MSG_NORM, _lib.X_REL2_NORM) else np.int32
        out = np.empty(n // 4, dtype=dtype)
        _lib.check(self._lib.rgcn_graph_export(self._h, which, _np_ptr(out), n), "rgcn_graph_export")
        return out

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            if self.device is not None and os.environ.get("RGCN_ASYNC_FREE") == "1":
                # opt-in (not yet validated on a GPU): stream-ordered frees on the current stream, no device sync
                self._lib.rgcn_graph_destroy_async(self._h, _stream(self.device))
            else:
                self._lib.rgcn_graph_destroy(self._h)
            self._h = ctypes.c_void_p(0)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h


# ---- tf.clip_by_global_norm sees IndexedSlices -----------------------------------------------------------------
# Variables the reference reads through tf.nn.embedding_lookup (block tables, relation table) get un-aggregated
# per-edge / per-triple gradient slices, and the global clipping norm is taken over those slice values.  When enabled,
# the backward passes below also produce sum |slice|^2 on the device and park it on the parameter tensor as
# `_slice_sumsq`; optim.ClippedAdam uses it in place of the dense gradient's sum of squares.
_SLICE_NORMS = False


def set_slice_norms(enabled):
    global _SLICE_NORMS
    _SLICE_NORMS = bool(enabled)


def _add_slice_sumsq(param, value):
    # a table made by an orthogonal transform (hole_transform) has the slice norms of the table it was made from
    param = getattr(param, "_slice_source", param)
    prev = getattr(param, "_slice_sumsq", None)
    param._slice_sumsq = value if prev is None else prev + value


def _workspace(nbytes, device):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)


def _call(entry, workspace_fn, workspace_args, args, device):
    """lib.entry(*args, workspace, workspace_bytes, stream) with a workspace of lib.workspace_fn(*workspace_args) bytes
    on `device` and its current stream; a negative size or a non-zero return code raises RgcnError."""
    lib = _lib.load()
    nb = getattr(lib, workspace_fn)(*workspace_args)
    if nb < 0:
        _lib.check(int(nb), workspace_fn)
    ws = _workspace(nb, device)
    _lib.check(getattr(lib, entry)(*args, _ptr(ws), ws.numel(), _stream(device)), entry)


def _mask_arg(mask, V, d):
    if mask is None:
        return None
    if not (mask.is_cuda and mask.dtype == torch.uint8 and mask.is_contiguous()
            and tuple(mask.shape) == (V, d)):
        raise _lib.RgcnError("drop_mask must be a contiguous CUDA uint8 [V_dst, d] keep-mask")
    return mask


class _BlockLayerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, H, Wf, Wb, Wself, graph, n_blocks, drop_mask, keep, relu):
        d = H.shape[1]
        R = graph.n_relw // 2
        s = d // n_blocks
        _check_cuda_f32("H", H, (graph.V_src, d))
        _check_cuda_f32("W_forward", Wf, (R, n_blocks, s, s))
        _check_cuda_f32("W_backward", Wb, (R, n_blocks, s, s))
        _check_cuda_f32("W_self", Wself, (d, d))
        mask = _mask_arg(drop_mask, graph.V_dst, d)
        dev = H.device
        out = torch.empty(graph.V_dst, d, dtype=torch.float32, device=dev)
        _call("rgcn_block_forward", "rgcn_block_workspace_bytes", (graph.handle, d, n_blocks, 0),
              (graph.handle, d, n_blocks, _ptr(H), _ptr(Wf), _ptr(Wb), _ptr(Wself), _ptr(mask), float(keep),
               int(bool(relu)), _ptr(out)), dev)
        ctx.graph, ctx.n_blocks, ctx.keep, ctx.relu = graph, n_blocks, float(keep), bool(relu)
        ctx.mask = mask
        ctx.params = (Wf, Wb)   # the caller's tensor objects (slice norms are parked on them)
        ctx.save_for_backward(H, Wf, Wb, Wself, out)
        return out

    @staticmethod
    def backward(ctx, dOut):
        H, Wf, Wb, Wself, out = ctx.saved_tensors
        graph, B = ctx.graph, ctx.n_blocks
        d = H.shape[1]
        dOut = dOut.contiguous()
        _check_cuda_f32("dOut", dOut, (graph.V_dst, d))
        dev = H.device
        dH = torch.empty_like(H)
        dWf, dWb, dWself = torch.empty_like(Wf), torch.empty_like(Wb), torch.empty_like(Wself)
        _call("rgcn_block_backward", "rgcn_block_workspace_bytes", (graph.handle, d, B, 1),
              (graph.handle, d, B, _ptr(H), _ptr(Wf), _ptr(Wb), _ptr(Wself), _ptr(ctx.mask), ctx.keep, int(ctx.relu),
               _ptr(out), _ptr(dOut), _ptr(dH), _ptr(dWf), _ptr(dWb), _ptr(dWself)), dev)
        if _SLICE_NORMS:
            G = ((dOut * (out > 0)) if ctx.relu else dOut).contiguous()
            ss = torch.empty(2, dtype=torch.float32, device=dev)
            _call("rgcn_block_slice_sumsq", "rgcn_block_slice_sumsq_workspace_bytes", (graph.handle, d, B),
                  (graph.handle, d, B, _ptr(H), _ptr(G), _ptr(ss)), dev)
            _add_slice_sumsq(ctx.params[0], ss[0])
            _add_slice_sumsq(ctx.params[1], ss[1])
        return dH, dWf, dWb, dWself, None, None, None, None, None


def block_layer(H, W_forward, W_backward, W_self, graph, n_blocks, drop_mask=None, keep=1.0,
                relu=True):
    """Block-diagonal R-GCN layer (ConcatGcn, gcn_basis_concat.py:35-83), differentiable."""
    return _BlockLayerFn.apply(H, W_forward, W_backward, W_self, graph, int(n_blocks), drop_mask,
                               keep, relu)


class _BasisLayerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, H, Vf, Vb, Cf, Cb, Wself, graph, drop_mask, keep, relu):
        d = H.shape[1]
        R = graph.n_relw // 2
        B = Cf.shape[1]
        _check_cuda_f32("H", H, (graph.V_src, d))
        _check_cuda_f32("W_forward", Vf, (d, B, d))
        _check_cuda_f32("W_backward", Vb, (d, B, d))
        _check_cuda_f32("C_forward", Cf, (R, B))
        _check_cuda_f32("C_backward", Cb, (R, B))
        _check_cuda_f32("W_self", Wself, (d, d))
        mask = _mask_arg(drop_mask, graph.V_dst, d)
        dev = H.device
        out = torch.empty(graph.V_dst, d, dtype=torch.float32, device=dev)
        saved = torch.empty(graph.V_dst, 2 * d * B, dtype=torch.float32, device=dev)
        _call("rgcn_basis_forward", "rgcn_basis_workspace_bytes", (graph.handle, d, B, 0),
              (graph.handle, d, B, _ptr(H), _ptr(Vf), _ptr(Vb), _ptr(Cf), _ptr(Cb), _ptr(Wself), _ptr(mask),
               float(keep), int(bool(relu)), _ptr(out), _ptr(saved)), dev)
        ctx.graph, ctx.keep, ctx.relu, ctx.mask = graph, float(keep), bool(relu), mask
        ctx.save_for_backward(H, Vf, Vb, Cf, Cb, Wself, out, saved)
        return out

    @staticmethod
    def backward(ctx, dOut):
        H, Vf, Vb, Cf, Cb, Wself, out, saved = ctx.saved_tensors
        graph = ctx.graph
        d, B = H.shape[1], Cf.shape[1]
        dOut = dOut.contiguous()
        dev = H.device
        dH = torch.empty_like(H)
        dVf, dVb = torch.empty_like(Vf), torch.empty_like(Vb)
        dCf, dCb, dWself = torch.empty_like(Cf), torch.empty_like(Cb), torch.empty_like(Wself)
        _call("rgcn_basis_backward", "rgcn_basis_workspace_bytes", (graph.handle, d, B, 1),
              (graph.handle, d, B, _ptr(H), _ptr(Vf), _ptr(Vb), _ptr(Cf), _ptr(Cb), _ptr(Wself), _ptr(ctx.mask),
               ctx.keep, int(ctx.relu), _ptr(out), _ptr(saved), _ptr(dOut), _ptr(dH), _ptr(dVf), _ptr(dVb), _ptr(dCf),
               _ptr(dCb), _ptr(dWself)), dev)
        return dH, dVf, dVb, dCf, dCb, dWself, None, None, None, None


def basis_layer(H, W_forward, W_backward, C_forward, C_backward, W_self, graph, drop_mask=None,
                keep=1.0, relu=True):
    """Basis-decomposition R-GCN layer (BasisGcn, gcn_basis.py:39-88), differentiable."""
    return _BasisLayerFn.apply(H, W_forward, W_backward, C_forward, C_backward, W_self, graph,
                               drop_mask, keep, relu)


class _BasisOnehotLayerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, Wf, Wb, Cf, Cb, Wself, graph, drop_mask, keep, relu):
        if not (isinstance(Wf, torch.Tensor) and Wf.dim() == 3):
            raise _lib.RgcnError("W_forward must be a [V, B, d] tensor")
        _, B, d = Wf.shape
        R = graph.n_relw // 2
        _check_cuda_f32("W_forward", Wf, (graph.V_src, B, d))
        _check_cuda_f32("W_backward", Wb, (graph.V_src, B, d))
        _check_cuda_f32("C_forward", Cf, (R, B))
        _check_cuda_f32("C_backward", Cb, (R, B))
        _check_cuda_f32("W_self", Wself, (graph.V_dst, d))
        mask = _mask_arg(drop_mask, graph.V_dst, d)
        dev = Wf.device
        out = torch.empty(graph.V_dst, d, dtype=torch.float32, device=dev)
        _call("rgcn_basis_onehot_forward", "rgcn_basis_onehot_workspace_bytes", (graph.handle, d, B, 0),
              (graph.handle, d, B, _ptr(Wf), _ptr(Wb), _ptr(Cf), _ptr(Cb), _ptr(Wself), _ptr(mask), float(keep),
               int(bool(relu)), _ptr(out)), dev)
        ctx.graph, ctx.keep, ctx.relu, ctx.mask = graph, float(keep), bool(relu), mask
        ctx.save_for_backward(Wf, Wb, Cf, Cb, Wself, out)
        return out

    @staticmethod
    def backward(ctx, dOut):
        Wf, Wb, Cf, Cb, Wself, out = ctx.saved_tensors
        graph = ctx.graph
        B, d = Wf.shape[1], Wf.shape[2]
        dOut = dOut.contiguous()
        _check_cuda_f32("dOut", dOut, (graph.V_dst, d))
        dev = Wf.device
        dWf, dWb = torch.empty_like(Wf), torch.empty_like(Wb)
        dCf, dCb, dWself = torch.empty_like(Cf), torch.empty_like(Cb), torch.empty_like(Wself)
        _call("rgcn_basis_onehot_backward", "rgcn_basis_onehot_workspace_bytes", (graph.handle, d, B, 1),
              (graph.handle, d, B, _ptr(Wf), _ptr(Wb), _ptr(Cf), _ptr(Cb), _ptr(ctx.mask), ctx.keep, int(ctx.relu),
               _ptr(out), _ptr(dOut), _ptr(dWf), _ptr(dWb), _ptr(dCf), _ptr(dCb), _ptr(dWself)), dev)
        return dWf, dWb, dCf, dCb, dWself, None, None, None, None


def basis_onehot_layer(W_forward, W_backward, C_forward, C_backward, W_self, graph, drop_mask=None, keep=1.0,
                       relu=True):
    """Featureless first basis layer (BasisGcn with onehot_input=True, gcn_basis.py:15-71): the input is the
    identity, so the basis terms of a message are rows W_dir[source] of the [V, B, d] tables.  Differentiable in
    every weight; there is no input gradient."""
    return _BasisOnehotLayerFn.apply(W_forward, W_backward, C_forward, C_backward, W_self, graph, drop_mask, keep,
                                     relu)


class _BasisDiagcoefLayerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, H, Vf, Vb, Cf, Cb, Wself, b, graph, drop_mask, keep, relu):
        if not (isinstance(Cf, torch.Tensor) and Cf.dim() == 3):
            raise _lib.RgcnError("C_forward must be a [R, B, d] tensor")
        d = H.shape[1]
        R = graph.n_relw // 2
        B = Cf.shape[1]
        _check_cuda_f32("H", H, (graph.V_src, d))
        _check_cuda_f32("W_forward", Vf, (d, B, d))
        _check_cuda_f32("W_backward", Vb, (d, B, d))
        _check_cuda_f32("C_forward", Cf, (R, B, d))
        _check_cuda_f32("C_backward", Cb, (R, B, d))
        _check_cuda_f32("W_self", Wself, (d, d))
        _check_cuda_f32("b", b, (d,))
        mask = _mask_arg(drop_mask, graph.V_dst, d)
        dev = H.device
        out = torch.empty(graph.V_dst, d, dtype=torch.float32, device=dev)
        saved = torch.empty(graph.V_src, 2 * B * d, dtype=torch.float32, device=dev)
        _call("rgcn_basis_diagcoef_forward", "rgcn_basis_diagcoef_workspace_bytes", (graph.handle, d, B, 0),
              (graph.handle, d, B, _ptr(H), _ptr(Vf), _ptr(Vb), _ptr(Cf), _ptr(Cb), _ptr(Wself), _ptr(b), _ptr(mask),
               float(keep), int(bool(relu)), _ptr(out), _ptr(saved)), dev)
        ctx.graph, ctx.keep, ctx.relu, ctx.mask = graph, float(keep), bool(relu), mask
        ctx.save_for_backward(H, Vf, Vb, Cf, Cb, Wself, out, saved)
        return out

    @staticmethod
    def backward(ctx, dOut):
        H, Vf, Vb, Cf, Cb, Wself, out, saved = ctx.saved_tensors
        graph = ctx.graph
        d, B = H.shape[1], Cf.shape[1]
        dOut = dOut.contiguous()
        _check_cuda_f32("dOut", dOut, (graph.V_dst, d))
        dev = H.device
        dH = torch.empty_like(H)
        dVf, dVb = torch.empty_like(Vf), torch.empty_like(Vb)
        dCf, dCb, dWself = torch.empty_like(Cf), torch.empty_like(Cb), torch.empty_like(Wself)
        db = torch.empty(d, dtype=torch.float32, device=dev)
        _call("rgcn_basis_diagcoef_backward", "rgcn_basis_diagcoef_workspace_bytes", (graph.handle, d, B, 1),
              (graph.handle, d, B, _ptr(H), _ptr(Vf), _ptr(Vb), _ptr(Cf), _ptr(Cb), _ptr(Wself), _ptr(ctx.mask),
               ctx.keep, int(ctx.relu), _ptr(out), _ptr(saved), _ptr(dOut), _ptr(dH), _ptr(dVf), _ptr(dVb), _ptr(dCf),
               _ptr(dCb), _ptr(dWself), _ptr(db)), dev)
        return dH, dVf, dVb, dCf, dCb, dWself, db, None, None, None, None


def basis_diagcoef_layer(H, W_forward, W_backward, C_forward, C_backward, W_self, b, graph, drop_mask=None, keep=1.0,
                         relu=True):
    """Basis R-GCN layer with per-channel sigmoid coefficients (BasisGcnTimesDiag, gcn_basis_times_diag.py, feature
    input): m = sum_b sigmoid(C_dir[r, b, :]) * (H[s] @ V_dir[:, b, :]), out = act(A_f m_f + A_b m_b +
    dropout(H @ W_self) + b).  C tables are [R, B, d]; differentiable in H and every weight, b included."""
    return _BasisDiagcoefLayerFn.apply(H, W_forward, W_backward, C_forward, C_backward, W_self, b, graph, drop_mask,
                                       keep, relu)


class _DiagLayerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, H, Df, Db, Wself, b, graph, drop_mask, keep, relu):
        if not (isinstance(H, torch.Tensor) and H.dim() == 2):
            raise _lib.RgcnError("H must be a [V_src, d] tensor")
        d = H.shape[1]
        R = graph.n_relw // 2
        _check_cuda_f32("H", H, (graph.V_src, d))
        _check_cuda_f32("D_types_forward", Df, (R, d))
        _check_cuda_f32("D_types_backward", Db, (R, d))
        _check_cuda_f32("W_self", Wself, (d, d))
        _check_cuda_f32("b", b, (d,))
        mask = _mask_arg(drop_mask, graph.V_dst, d)
        dev = H.device
        out = torch.empty(graph.V_dst, d, dtype=torch.float32, device=dev)
        _call("rgcn_diag_forward", "rgcn_diag_workspace_bytes", (graph.handle, d, 0),
              (graph.handle, d, _ptr(H), _ptr(Df), _ptr(Db), _ptr(Wself), _ptr(b), _ptr(mask), float(keep),
               int(bool(relu)), _ptr(out)), dev)
        ctx.graph, ctx.keep, ctx.relu, ctx.mask = graph, float(keep), bool(relu), mask
        ctx.params = (Df, Db)   # the caller's tensor objects (slice norms are parked on them)
        ctx.save_for_backward(H, Df, Db, Wself, out)
        return out

    @staticmethod
    def backward(ctx, dOut):
        H, Df, Db, Wself, out = ctx.saved_tensors
        graph = ctx.graph
        d = H.shape[1]
        dOut = dOut.contiguous()
        _check_cuda_f32("dOut", dOut, (graph.V_dst, d))
        dev = H.device
        dH = torch.empty_like(H)
        dDf, dDb, dWself = torch.empty_like(Df), torch.empty_like(Db), torch.empty_like(Wself)
        db = torch.empty(d, dtype=torch.float32, device=dev)
        ss = torch.empty(2, dtype=torch.float32, device=dev) if _SLICE_NORMS else None
        _call("rgcn_diag_backward", "rgcn_diag_workspace_bytes", (graph.handle, d, 1),
              (graph.handle, d, _ptr(H), _ptr(Df), _ptr(Db), _ptr(Wself), _ptr(ctx.mask), ctx.keep, int(ctx.relu),
               _ptr(out), _ptr(dOut), _ptr(dH), _ptr(dDf), _ptr(dDb), _ptr(dWself), _ptr(db), _ptr(ss)), dev)
        if ss is not None:
            _add_slice_sumsq(ctx.params[0], ss[0])
            _add_slice_sumsq(ctx.params[1], ss[1])
        return dH, dDf, dDb, dWself, db, None, None, None, None


def diag_layer(H, D_forward, D_backward, W_self, b, graph, drop_mask=None, keep=1.0, relu=True):
    """Diagonal R-GCN layer (DiagGcn, gcn_diag.py): a message s -> o of relation r is D_dir[r] * H[s] (element-wise),
    out = act(A_f m_f + A_b m_b + dropout(H @ W_self) + b).  D tables are [R, d]; differentiable in H and every
    weight, b included.  With set_slice_norms(True) the backward also parks the IndexedSlices sum of squares of the
    D gradients on D_forward / D_backward."""
    return _DiagLayerFn.apply(H, D_forward, D_backward, W_self, b, graph, drop_mask, keep, relu)


COMPOSITIONS = ("mult", "sub")   # the composition codes of the library: RGCN_COMPOSITION_MULT = 0, _SUB = 1


class _CompGcnLayerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, H, Z, z_loop, W_cat, W_rel, b, graph, op, drop_mask, keep, relu):
        if not (isinstance(H, torch.Tensor) and H.dim() == 2 and isinstance(W_cat, torch.Tensor) and W_cat.dim() == 2):
            raise _lib.RgcnError("H must be a [V_src, d_in] tensor and W_cat a [3 d_in, d_out] tensor")
        d_in, d_out = H.shape[1], W_cat.shape[1]
        _check_cuda_f32("H", H, (graph.V_src, d_in))
        _check_cuda_f32("Z", Z, (graph.n_relw, d_in))
        _check_cuda_f32("z_loop", z_loop, (d_in,))
        _check_cuda_f32("W_cat", W_cat, (3 * d_in, d_out))
        _check_cuda_f32("W_rel", W_rel, (d_in, d_out))
        _check_cuda_f32("b", b, (d_out,))
        mask = _mask_arg(drop_mask, graph.V_dst, 2 * d_in)
        dev = H.device
        Cat = torch.empty(graph.V_dst, 3 * d_in, dtype=torch.float32, device=dev)
        out = torch.empty(graph.V_dst, d_out, dtype=torch.float32, device=dev)
        Z_next = torch.empty(graph.n_relw, d_out, dtype=torch.float32, device=dev)
        _call("rgcn_compgcn_forward", "rgcn_compgcn_workspace_bytes", (graph.handle, d_in, d_out, 0),
              (graph.handle, d_in, d_out, op, _ptr(H), _ptr(Z), _ptr(z_loop), _ptr(W_cat), _ptr(W_rel), _ptr(b),
               _ptr(mask), float(keep), int(bool(relu)), _ptr(Cat), _ptr(out), _ptr(Z_next)), dev)
        ctx.graph, ctx.op, ctx.keep, ctx.relu, ctx.mask = graph, op, float(keep), bool(relu), mask
        ctx.save_for_backward(H, Z, z_loop, W_cat, W_rel, Cat, out)
        return out, Z_next

    @staticmethod
    def backward(ctx, dOut, dZ_next):
        H, Z, z_loop, W_cat, W_rel, Cat, out = ctx.saved_tensors
        graph = ctx.graph
        d_in, d_out = H.shape[1], W_cat.shape[1]
        dOut, dZ_next = dOut.contiguous(), dZ_next.contiguous()
        _check_cuda_f32("dOut", dOut, (graph.V_dst, d_out))
        _check_cuda_f32("dZ_next", dZ_next, (graph.n_relw, d_out))
        dev = H.device
        dH, dZ, dz_loop = torch.empty_like(H), torch.empty_like(Z), torch.empty_like(z_loop)
        dW_cat, dW_rel = torch.empty_like(W_cat), torch.empty_like(W_rel)
        db = torch.empty(d_out, dtype=torch.float32, device=dev)
        _call("rgcn_compgcn_backward", "rgcn_compgcn_workspace_bytes", (graph.handle, d_in, d_out, 1),
              (graph.handle, d_in, d_out, ctx.op, _ptr(H), _ptr(Z), _ptr(z_loop), _ptr(W_cat), _ptr(W_rel),
               _ptr(ctx.mask), ctx.keep, int(ctx.relu), _ptr(Cat), _ptr(out), _ptr(dOut), _ptr(dZ_next), _ptr(dH),
               _ptr(dZ), _ptr(dz_loop), _ptr(dW_cat), _ptr(dW_rel), _ptr(db)), dev)
        return dH, dZ, dz_loop, dW_cat, dW_rel, db, None, None, None, None, None


def compgcn_layer(H, Z, z_loop, W_cat, W_rel, b, graph, composition="mult", drop_mask=None, keep=1.0, relu=True):
    """CompGCN layer (Vashishth et al., ICLR 2020) as one library call each way.  A message s -> o of weight id w
    (forward relation r: w = r, its inverse: w = R + r) is norm * phi(H[s], Z[w]) with phi = h * z ("mult") or
    h - z ("sub"); with A_f / A_b the two directions' sums, L = phi(H[:V_dst], z_loop) and M the [V_dst, 2 d_in]
    keep-mask,
        out    = act([M * [A_f | A_b] / keep | L] / 3 @ W_cat + b),     W_cat = [W_I; W_O; W_S] : [3 d_in, d_out]
        Z_next = Z @ W_rel.
    Z : [2R, d_in], z_loop : [d_in], W_rel : [d_in, d_out].  Returns (out, Z_next), differentiable in H, Z, z_loop
    and every weight."""
    if composition not in COMPOSITIONS:
        raise ValueError("composition must be one of %s, got %r" % (", ".join(COMPOSITIONS), composition))
    return _CompGcnLayerFn.apply(H, Z, z_loop, W_cat, W_rel, b, graph, COMPOSITIONS.index(composition), drop_mask,
                                 keep, relu)


class _HighwayFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, c1, c2, W, b):
        if not (isinstance(c1, torch.Tensor) and c1.dim() == 2):
            raise _lib.RgcnError("c1 must be a [V, d] tensor")
        V, d = c1.shape
        _check_cuda_f32("c1", c1)
        _check_cuda_f32("c2", c2, (V, d))
        _check_cuda_f32("W", W, (d, d))
        _check_cuda_f32("b", b, (d,))
        dev = c1.device
        out = torch.empty(V, d, dtype=torch.float32, device=dev)
        gate = torch.empty(V, d, dtype=torch.float32, device=dev)
        _call("rgcn_highway_forward", "rgcn_highway_workspace_bytes", (V, d, 0),
              (_ptr(c1), _ptr(c2), _ptr(W), _ptr(b), V, d, _ptr(out), _ptr(gate)), dev)
        ctx.save_for_backward(c1, c2, W, gate)
        return out

    @staticmethod
    def backward(ctx, dOut):
        c1, c2, W, gate = ctx.saved_tensors
        V, d = c1.shape
        dOut = dOut.contiguous()
        _check_cuda_f32("dOut", dOut, (V, d))
        dev = c1.device
        dc1, dc2, dW = torch.empty_like(c1), torch.empty_like(c2), torch.empty_like(W)
        db = torch.empty(d, dtype=torch.float32, device=dev)
        _call("rgcn_highway_backward", "rgcn_highway_workspace_bytes", (V, d, 1),
              (_ptr(c1), _ptr(c2), _ptr(W), _ptr(gate), _ptr(dOut), V, d, _ptr(dc1), _ptr(dc2), _ptr(dW), _ptr(db)),
              dev)
        return dc1, dc2, dW, db


def highway(c1, c2, W, b):
    """Highway skip connection (extras/highway_layer.py:14-38): g = sigmoid(c2 @ W + b), out = g * c1 + (1 - g) * c2,
    with c1 the wrapped layer's output and c2 its input.  One library call each way; differentiable in all four."""
    return _HighwayFn.apply(c1, c2, W, b)


class _VariationalFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, H, W_mu, b_mu, W_sigma, b_sigma, eps):
        if not (isinstance(W_mu, torch.Tensor) and W_mu.dim() == 2):
            raise _lib.RgcnError("W_mu must be a 2-D tensor")
        w = W_mu.shape[1]
        _check_cuda_f32("eps", eps)
        V = eps.shape[0]
        _check_cuda_f32("eps", eps, (V, w))
        if H is None:           # embedding variant: mu = W_mu, log sigma = W_sigma
            d = 0
            _check_cuda_f32("W_mu", W_mu, (V, w))
            _check_cuda_f32("W_sigma", W_sigma, (V, w))
        else:
            d = W_mu.shape[0]
            _check_cuda_f32("H", H, (V, d))
            _check_cuda_f32("W_mu", W_mu, (d, w))
            _check_cuda_f32("W_sigma", W_sigma, (d, w))
            _check_cuda_f32("b_mu", b_mu, (w,))
            _check_cuda_f32("b_sigma", b_sigma, (w,))
        dev = eps.device
        z = torch.empty(V, w, dtype=torch.float32, device=dev)
        kl = torch.empty((), dtype=torch.float32, device=dev)
        P = torch.empty(V, 2 * w, dtype=torch.float32, device=dev) if d else None
        _call("rgcn_variational_forward", "rgcn_variational_workspace_bytes", (V, d, w, 0),
              (_ptr(H), V, d, w, _ptr(W_mu), _ptr(b_mu if d else None), _ptr(W_sigma), _ptr(b_sigma if d else None),
               _ptr(eps), _ptr(z), _ptr(P), _ptr(kl)), dev)
        ctx.d = d
        ctx.save_for_backward(H, W_mu, W_sigma, P, eps)
        return z, kl

    @staticmethod
    def backward(ctx, dz, g_kl):
        H, W_mu, W_sigma, P, eps = ctx.saved_tensors
        d = ctx.d
        V, w = eps.shape
        dev = eps.device
        dz = dz.contiguous()
        _check_cuda_f32("dz", dz, (V, w))
        g_kl = g_kl.reshape(1).contiguous()
        dW_mu, dW_sigma = torch.empty_like(W_mu), torch.empty_like(W_sigma)
        dH = torch.empty_like(H) if d else None
        db_mu = torch.empty(w, dtype=torch.float32, device=dev) if d else None
        db_sigma = torch.empty(w, dtype=torch.float32, device=dev) if d else None
        _call("rgcn_variational_backward", "rgcn_variational_workspace_bytes", (V, d, w, 1),
              (_ptr(H), V, d, w, _ptr(W_mu), _ptr(W_sigma), _ptr(P), _ptr(eps), _ptr(dz), _ptr(g_kl), _ptr(dH),
               _ptr(dW_mu), _ptr(db_mu), _ptr(dW_sigma), _ptr(db_sigma)), dev)
        # the embedding variant's biases are never read: their gradient is None, as in the reference
        return dH, dW_mu, db_mu, dW_sigma, db_sigma, None


def variational(H, W_mu, b_mu, W_sigma, b_sigma, eps):
    """Reparameterised codes and KL term of VariationalEncoding (extras/variational_encoding.py:14-31).  With H None
    (variational_embedding) mu = W_mu and log sigma = W_sigma ([V, w]) and the biases are ignored; otherwise
    mu = H @ W_mu + b_mu and log sigma = H @ W_sigma + b_sigma.  Returns (z, kl): z = mu + exp(log sigma) * eps and
    kl = -0.0005 * sum(1 + 2 log sigma - mu^2 - exp(2 log sigma)).  One library call each way; differentiable in H and
    every weight it reads."""
    return _VariationalFn.apply(H, W_mu, b_mu, W_sigma, b_sigma, eps)


def _triple_forward(ctx, entry, codes, rel, X, Y, extra=()):
    """Forward of a triple scorer entry point with the distmult_forward argument list; `extra` goes after Y (the
    margin of rgcn_rotate_forward)."""
    lib = _lib.load()
    _check_cuda_f32("codes", codes)
    _check_cuda_f32("relation table", rel)
    if not (X.is_cuda and X.dtype == torch.int32 and X.is_contiguous() and X.dim() == 2
            and X.shape[1] == 3):
        raise _lib.RgcnError("X must be a contiguous CUDA int32 [N,3] tensor")
    if Y is not None:
        _check_cuda_f32("Y", Y, (X.shape[0],))
    V, d = codes.shape
    dev = codes.device
    N = X.shape[0]
    energies = torch.empty(N, dtype=torch.float32, device=dev)
    loss2 = torch.empty(2, dtype=torch.float32, device=dev)
    rc = getattr(lib, entry)(_ptr(codes), _ptr(rel), V, rel.shape[0], d, _ptr(X), N, _ptr(Y), *extra,
                             _ptr(energies), _ptr(loss2), _stream(dev))
    _lib.check(rc, entry)
    ctx.has_y = Y is not None
    ctx.extra = extra
    ctx.rel_param = rel
    ctx.save_for_backward(codes, rel, X, Y if Y is not None else torch.empty(0, device=dev),
                          energies)
    return energies, loss2[0], loss2[1]


def _triple_backward(ctx, entry, g_energy, g_loss, g_reg):
    """Backward of a triple scorer entry point with the distmult_backward_slices argument list; the forward's `extra`
    goes after Y."""
    lib = _lib.load()
    codes, rel, X, Y, energies = ctx.saved_tensors
    Y = Y if ctx.has_y else None
    V, d = codes.shape
    dev = codes.device
    dcodes = torch.zeros_like(codes)
    drel = torch.zeros_like(rel)
    ge = None
    if g_energy is not None:
        ge = g_energy.contiguous()
    # upstream scalar gradients stay on the device (no host sync): passed as g_scale_dev[2]
    gs = torch.zeros(2, dtype=torch.float32, device=dev)
    if g_loss is not None:
        gs[0] = g_loss
    if g_reg is not None:
        gs[1] = g_reg
    ss = torch.zeros(1, dtype=torch.float32, device=dev) if _SLICE_NORMS else None
    rc = getattr(lib, entry)(_ptr(codes), _ptr(rel), V, rel.shape[0], d, _ptr(X), X.shape[0],
                             _ptr(Y), *ctx.extra, _ptr(energies), 1.0, 1.0, _ptr(gs), _ptr(ge),
                             _ptr(dcodes), _ptr(drel), _ptr(ss), _stream(dev))
    _lib.check(rc, entry)
    if ss is not None:
        _add_slice_sumsq(ctx.rel_param, ss[0])
    return dcodes, drel, None, None


class _DistMultFn(torch.autograd.Function):
    """Returns (energies[N], loss, reg): loss = mean sigmoid-CE (0 if Y is None), reg = un-scaled L2."""

    @staticmethod
    def forward(ctx, codes, rel, X, Y):
        return _triple_forward(ctx, "distmult_forward", codes, rel, X, Y)

    @staticmethod
    def backward(ctx, g_energy, g_loss, g_reg):
        return _triple_backward(ctx, "distmult_backward_slices", g_energy, g_loss, g_reg)


def distmult(codes, rel, X, Y=None):
    """DistMult energies + sigmoid cross-entropy + L2 term (bilinear_diag.py:14-34,63-69)."""
    return _DistMultFn.apply(codes, rel, X, Y)


class _ComplexFn(torch.autograd.Function):
    """Returns (energies[N], loss, reg) of the ComplEx scorer, same conventions as _DistMultFn."""

    @staticmethod
    def forward(ctx, codes, rel, X, Y):
        return _triple_forward(ctx, "rgcn_complex_forward", codes, rel, X, Y)

    @staticmethod
    def backward(ctx, g_energy, g_loss, g_reg):
        return _triple_backward(ctx, "rgcn_complex_backward", g_energy, g_loss, g_reg)


def complex_score(codes, rel, X, Y=None):
    """ComplEx energies + sigmoid cross-entropy + L2 term (complex.py:31-45,108-114); rows are [real | imaginary]."""
    return _ComplexFn.apply(codes, rel, X, Y)


def _check_gamma(gamma):
    gamma = float(gamma)
    if not np.isfinite(gamma):
        raise ValueError("the margin gamma must be finite, got %r" % (gamma,))
    return gamma


class _RotateFn(torch.autograd.Function):
    """Returns (energies[N], loss, reg) of the RotatE scorer, same conventions as _DistMultFn."""

    @staticmethod
    def forward(ctx, codes, rel, X, Y, gamma):
        return _triple_forward(ctx, "rgcn_rotate_forward", codes, rel, X, Y, (gamma,))

    @staticmethod
    def backward(ctx, g_energy, g_loss, g_reg):
        return _triple_backward(ctx, "rgcn_rotate_backward", g_energy, g_loss, g_reg) + (None,)


def rotate_score(codes, rel, X, Y=None, *, gamma):
    """RotatE energies gamma - sum_k |a_k e^{i theta_k} - c_k| (entity rows [re | im], the phases theta in the first
    d/2 columns of the relation row), the mean sigmoid cross-entropy (0 if Y is None) and the L2 term
    mean(a^2) + mean(c^2) of the gathered entity rows (include/rgcn_b200.h, rgcn_rotate_forward)."""
    return _RotateFn.apply(codes, rel, X, Y, _check_gamma(gamma))


class _TransEFn(torch.autograd.Function):
    """Returns (energies[N], loss, reg) of the TransE scorer, same conventions as _DistMultFn."""

    @staticmethod
    def forward(ctx, codes, rel, X, Y, gamma):
        return _triple_forward(ctx, "rgcn_transe_forward", codes, rel, X, Y, (gamma,))

    @staticmethod
    def backward(ctx, g_energy, g_loss, g_reg):
        return _triple_backward(ctx, "rgcn_transe_backward", g_energy, g_loss, g_reg) + (None,)


def transe_score(codes, rel, X, Y=None, *, gamma):
    """TransE energies gamma - sum_k |h_k + r_k - t_k| (plain real rows, all d columns of the relation row), the mean
    sigmoid cross-entropy (0 if Y is None) and the L2 term mean(h^2) + mean(r^2) + mean(t^2) of the gathered rows
    (include/rgcn_b200.h, rgcn_transe_forward)."""
    return _TransEFn.apply(codes, rel, X, Y, _check_gamma(gamma))


class _QuatEFn(torch.autograd.Function):
    """Returns (energies[N], loss, reg) of the QuatE scorer, same conventions as _DistMultFn."""

    @staticmethod
    def forward(ctx, codes, rel, X, Y):
        return _triple_forward(ctx, "rgcn_quate_forward", codes, rel, X, Y)

    @staticmethod
    def backward(ctx, g_energy, g_loss, g_reg):
        return _triple_backward(ctx, "rgcn_quate_backward", g_energy, g_loss, g_reg)


def quate_score(codes, rel, X, Y=None):
    """QuatE energies sum_k <h_k (x) r_k / max(|r_k|, 1e-12), t_k> (quaternion k of a row: columns 4k..4k+3, (x) the
    Hamilton product), the mean sigmoid cross-entropy (0 if Y is None) and DistMult's L2 term mean(h^2) + mean(r^2) +
    mean(t^2) of the gathered raw rows (include/rgcn_b200.h, rgcn_quate_forward)."""
    return _QuatEFn.apply(codes, rel, X, Y)


# ---- HolE (rgcn_hole_*, include/rgcn_b200.h): the real Fourier basis and the scorer over transformed tables ----
_HOLE_BASES = {}   # (device, d) -> U [d, d]


def hole_basis(d, device):
    """The HolE basis U [d, d] (float32 CUDA, built once per (device, d) by rgcn_hole_transform): the orthonormal real
    DFT basis with columns DC, Nyquist, then (cos, -sin) pairs of frequencies 1 .. d/2 - 1."""
    device = torch.device(device)
    key = (device, int(d))
    U = _HOLE_BASES.get(key)
    if U is None:
        U = torch.empty((d, d), dtype=torch.float32, device=device)
        _call("rgcn_hole_transform", "rgcn_hole_transform_workspace_bytes", (d,),
              (None, 0, d, 0, _ptr(U), 0, None), device)
        _HOLE_BASES[key] = U
    return U


def _hole_apply(x, inverse):
    """x U (inverse False) or x U^T (inverse True) of a CUDA float32 [rows, d] tensor, one library GEMM"""
    _check_cuda_f32("rows to transform", x)
    rows, d = x.shape
    U = hole_basis(d, x.device)
    out = torch.empty_like(x)
    _call("rgcn_hole_transform", "rgcn_hole_transform_workspace_bytes", (d,),
          (_ptr(x), rows, d, int(inverse), _ptr(U), 1, _ptr(out)), x.device)
    return out


class _HolETransformFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, inverse):
        ctx.inverse = inverse
        return _hole_apply(x, inverse)

    @staticmethod
    def backward(ctx, g):
        return _hole_apply(g.contiguous(), not ctx.inverse), None


def hole_transform(x, inverse=False):
    """The rows of x [rows, d] (CUDA float32, d % 4 == 0) in the HolE basis, x U (inverse=True: x U^T, which takes
    them back).  Differentiable: the backward is g U^T (g U).  The result carries the slice norms the HolE backward
    passes leave on it over to x, or to the table x is a row range of, for optim.ClippedAdam: U is orthogonal, so
    they are x's own."""
    out = _HolETransformFn.apply(x, bool(inverse))
    out._slice_source = getattr(x, "_slice_source", x if x._base is None else x._base)
    return out


class _HolEFn(torch.autograd.Function):
    """Returns (energies[N], loss, reg) of the HolE scorer over transformed tables, same conventions as _DistMultFn."""

    @staticmethod
    def forward(ctx, codes, rel, X, Y):
        return _triple_forward(ctx, "rgcn_hole_forward", codes, rel, X, Y)

    @staticmethod
    def backward(ctx, g_energy, g_loss, g_reg):
        return _triple_backward(ctx, "rgcn_hole_backward", g_energy, g_loss, g_reg)


def hole_score(codes, rel, X, Y=None):
    """HolE energies sum_k r_k [h * t]_k (circular correlation) of tables already in the HolE basis (hole_transform),
    the mean sigmoid cross-entropy (0 if Y is None) and DistMult's L2 term mean(h^2) + mean(r^2) + mean(t^2) of the
    gathered rows, which the orthogonal basis leaves unchanged (include/rgcn_b200.h, rgcn_hole_forward)."""
    return _HolEFn.apply(codes, rel, X, Y)


# decoder -> (the decoder kind of rgcn_self_adversarial_forward, or the name of the decoder's own entry point, which
# takes the margin gamma if the decoder is one of MARGIN_DECODERS; the scorer's backward)
SELF_ADVERSARIAL_DECODERS = {"distmult": (_lib.RGCN_DECODER_DISTMULT, "distmult_backward_slices"),
                             "complex": (_lib.RGCN_DECODER_COMPLEX, "rgcn_complex_backward"),
                             "rotate": ("rgcn_rotate_self_adversarial_forward", "rgcn_rotate_backward"),
                             "transe": ("rgcn_transe_self_adversarial_forward", "rgcn_transe_backward"),
                             "quate": ("rgcn_quate_self_adversarial_forward", "rgcn_quate_backward"),
                             "hole": ("rgcn_hole_self_adversarial_forward", "rgcn_hole_backward")}
# the decoders whose energy carries the margin gamma
MARGIN_DECODERS = ("rotate", "transe")


class _SelfAdversarialFn(torch.autograd.Function):
    """Returns (loss, reg, energies) of rgcn_self_adversarial_forward.  The forward also writes each triple's energy
    gradient coefficient; the backward is the scorer's own (Y = NULL) with g_energy = g_loss * coef (+ the upstream
    gradient of the energies) and the L2 term scaled on the device."""

    @staticmethod
    def forward(ctx, codes, rel, X, K, alpha, decoder, gamma):
        kind, bwd = SELF_ADVERSARIAL_DECODERS[decoder]
        V, d = codes.shape
        dev = codes.device
        N = X.shape[0]
        energies = torch.empty(N, dtype=torch.float32, device=dev)
        coef = torch.empty(N, dtype=torch.float32, device=dev)
        loss2 = torch.empty(2, dtype=torch.float32, device=dev)
        rows = (_ptr(codes), _ptr(rel), V, rel.shape[0], d, _ptr(X), N, K, alpha)
        outs = (_ptr(energies), _ptr(coef), _ptr(loss2))
        margin = (gamma,) if gamma is not None else ()
        if isinstance(kind, str):
            _call(kind, "rgcn_self_adversarial_workspace_bytes", (N, K), rows + margin + outs, dev)
        else:
            _call("rgcn_self_adversarial_forward", "rgcn_self_adversarial_workspace_bytes", (N, K),
                  (kind,) + rows + outs, dev)
        ctx.bwd = bwd
        ctx.extra = margin
        ctx.rel_param = rel
        ctx.save_for_backward(codes, rel, X, coef)
        return loss2[0], loss2[1], energies

    @staticmethod
    def backward(ctx, g_loss, g_reg, g_energy):
        lib = _lib.load()
        codes, rel, X, coef = ctx.saved_tensors
        V, d = codes.shape
        dev = codes.device
        ge = None
        if g_loss is not None:
            ge = coef * g_loss
        if g_energy is not None:
            ge = g_energy.contiguous() if ge is None else ge + g_energy
        gs = torch.zeros(2, dtype=torch.float32, device=dev)
        if g_reg is not None:
            gs[1] = g_reg
        dcodes = torch.zeros_like(codes)
        drel = torch.zeros_like(rel)
        ss = torch.zeros(1, dtype=torch.float32, device=dev) if _SLICE_NORMS else None
        rc = getattr(lib, ctx.bwd)(_ptr(codes), _ptr(rel), V, rel.shape[0], d, _ptr(X), X.shape[0], None, *ctx.extra,
                                   None, 0.0, 1.0, _ptr(gs), _ptr(ge), _ptr(dcodes), _ptr(drel), _ptr(ss),
                                   _stream(dev))
        _lib.check(rc, ctx.bwd)
        if ss is not None:
            _add_slice_sumsq(ctx.rel_param, ss[0])
        return dcodes, drel, None, None, None, None, None


def self_adversarial_loss(codes, rel, X, K, alpha, decoder, *, gamma=None):
    """Self-adversarial negative sampling (Sun et al., RotatE, ICLR 2019) over the fed triples X (CUDA int32 [N, 3]) in
    the negative sampler's layout: rows 0..n-1 the positives, row i + n j (j = 1..K) the j-th corruption of positive i,
    N = n (K + 1).  Returns (loss, reg, energies): loss = 1/(2n) sum_i [softplus(-s_i) + sum_j p_ij softplus(s_ij)] with
    p_ij = softmax_j(alpha s_ij) held constant, reg = the decoder's L2 term over all N triples, energies [N].
    decoder is "distmult", "complex", "rotate", "transe", "quate" or "hole" (on tables in the HolE basis); gamma is the
    margin, needed by "rotate" and "transe" only.
    Differentiable in codes and rel."""
    if decoder not in SELF_ADVERSARIAL_DECODERS:
        raise ValueError("self_adversarial_loss: decoder must be one of %s, got %r"
                         % (sorted(SELF_ADVERSARIAL_DECODERS), decoder))
    if (decoder in MARGIN_DECODERS) != (gamma is not None):
        raise ValueError("self_adversarial_loss: the margin gamma goes with decoders 'rotate' and 'transe' only (got "
                         "decoder %r, gamma %r)" % (decoder, gamma))
    if gamma is not None:
        gamma = _check_gamma(gamma)
    K, alpha = int(K), float(alpha)
    if K < 1:
        raise ValueError("self_adversarial_loss: NegativeSampleRate must be >= 1, got %d" % K)
    if not 0.0 <= alpha < float("inf"):
        raise ValueError("self_adversarial_loss: AdversarialTemperature must be finite and >= 0, got %r" % (alpha,))
    _check_cuda_f32("codes", codes)
    _check_cuda_f32("relation table", rel)
    if not (X.is_cuda and X.dtype == torch.int32 and X.is_contiguous() and X.dim() == 2 and X.shape[1] == 3):
        raise _lib.RgcnError("X must be a contiguous CUDA int32 [N,3] tensor")
    if X.shape[0] % (K + 1):
        raise ValueError("self_adversarial_loss: %d fed triples are not n positives with NegativeSampleRate=%d "
                         "corruptions each (N %% (K + 1) != 0)" % (X.shape[0], K))
    return _SelfAdversarialFn.apply(codes, rel, X, K, alpha, decoder, gamma)


def gemm_tf32x3(A, B, b_is_nk=False, out=None, accumulate=False):
    """C = A @ B (B [K,N]) or A @ B.T (B [N,K], b_is_nk=True) on the wgmma tensor cores with the
    3xTF32 split (fp32-level accuracy).  Thin wrapper over rgcn_gemm_tf32x3 (include/rgcn_b200.h)."""
    lib = _lib.load()
    _check_cuda_f32("A", A)
    _check_cuda_f32("B", B)
    M, K = A.shape
    N = B.shape[0] if b_is_nk else B.shape[1]
    if out is None:
        out = torch.empty(M, N, dtype=torch.float32, device=A.device)
    ws = torch.empty(2 * N * K, dtype=torch.float32, device=A.device)
    rc = lib.rgcn_gemm_tf32x3(_ptr(A), A.stride(0), _ptr(B), B.stride(0), int(b_is_nk), _ptr(out),
                              out.stride(0), M, N, K, int(accumulate), _ptr(ws), ws.numel() * 4,
                              _stream(A.device))
    _lib.check(rc, "rgcn_gemm_tf32x3")
    return out


def gemm_tn_tf32x3(A, B, out=None, accumulate=False):
    """C = A.T @ B with A [K,M], B [K,N] (contraction over the slow dimension), wgmma 3xTF32, split-K."""
    lib = _lib.load()
    _check_cuda_f32("A", A)
    _check_cuda_f32("B", B)
    K, M = A.shape
    N = B.shape[1]
    if out is None:
        out = torch.empty(M, N, dtype=torch.float32, device=A.device)
    rc = lib.rgcn_gemm_tn_tf32x3(_ptr(A), A.stride(0), _ptr(B), B.stride(0), _ptr(out), out.stride(0), M, N, K,
                                 int(accumulate), _stream(A.device))
    _lib.check(rc, "rgcn_gemm_tn_tf32x3")
    return out


def rows_add_(dst, rows, src):
    """dst[rows[i]] += src[i] for UNIQUE rows (rgcn_rows_add): the non-atomic unpack of one peer's halo gradients."""
    lib = _lib.load()
    _check_cuda_f32("dst", dst)
    _check_cuda_f32("src", src)
    if not (rows.is_cuda and rows.dtype == torch.int64 and rows.is_contiguous() and rows.numel() == src.shape[0]):
        raise _lib.RgcnError("rows must be a contiguous CUDA int64 tensor with one entry per row of src")
    _lib.check(lib.rgcn_rows_add(_ptr(dst), _ptr(rows), _ptr(src), src.shape[0], dst.shape[1], _stream(dst.device)),
               "rgcn_rows_add")
    return dst


def relu_backward(dOut, out):
    """G = dOut * (out > 0) in one pass (rgcn_relu_backward)."""
    lib = _lib.load()
    dOut = dOut.contiguous()
    _check_cuda_f32("dOut", dOut)
    _check_cuda_f32("out", out, dOut.shape)
    G = torch.empty_like(dOut)
    _lib.check(lib.rgcn_relu_backward(_ptr(dOut), _ptr(out), _ptr(G), dOut.numel(), _stream(dOut.device)),
               "rgcn_relu_backward")
    return G


def rows_gather_to(dst_ptr, src, rows, max_ctas=0):
    """memory at dst_ptr [len(rows), d] = src[rows] (rgcn_rows_gather).  dst_ptr is a raw device address, normally a
    PEER GPU's halo buffer mapped into this process (parallel.PeerHalo): the halo push of the node-sharded path."""
    lib = _lib.load()
    _check_cuda_f32("src", src)
    if not (rows.is_cuda and rows.dtype == torch.int64 and rows.is_contiguous()):
        raise _lib.RgcnError("rows must be a contiguous CUDA int64 tensor")
    _lib.check(lib.rgcn_rows_gather(int(dst_ptr), _ptr(src), _ptr(rows), rows.numel(), src.shape[1], int(max_ctas),
                                    _stream(src.device)), "rgcn_rows_gather")


def block_aggregate_(out, X, W_forward, W_backward, graph, n_blocks):
    """out[dst] += sum_m norm_m W[relw_m] . X[src_m] (messages only, in place; rgcn_block_aggregate)."""
    d = X.shape[1]
    _check_cuda_f32("X", X, (graph.V_src, d))
    _check_cuda_f32("out", out, (graph.V_dst, d))
    _call("rgcn_block_aggregate", "rgcn_block_aggregate_workspace_bytes", (graph.handle, d, n_blocks, 0),
          (graph.handle, d, n_blocks, _ptr(X), _ptr(W_forward), _ptr(W_backward), _ptr(out)), X.device)
    return out


def block_aggregate_backward(X, W_forward, W_backward, G, graph, n_blocks, dWf=None, dWb=None):
    """Returns (dX, dWf, dWb) of block_aggregate_; when dWf/dWb are given they are accumulated into."""
    d = X.shape[1]
    _check_cuda_f32("X", X, (graph.V_src, d))
    _check_cuda_f32("G", G, (graph.V_dst, d))
    acc = dWf is not None
    if not acc:
        dWf, dWb = torch.empty_like(W_forward), torch.empty_like(W_backward)
    dX = torch.empty_like(X)
    _call("rgcn_block_aggregate_backward", "rgcn_block_aggregate_workspace_bytes", (graph.handle, d, n_blocks, 1),
          (graph.handle, d, n_blocks, _ptr(X), _ptr(W_forward), _ptr(W_backward), _ptr(G), _ptr(dX), _ptr(dWf),
           _ptr(dWb), int(acc)), X.device)
    return dX, dWf, dWb


class DistMultRanker(object):
    """Fused all-entity scoring + ranking over one entity code matrix (distmult_rank, include/rgcn_b200.h): the
    hi/lo split of `codes` is made once and reused by every chunk / corruption side, by rank and top_k alike (both
    workspaces start with the split)."""
    _RANK, _WORKSPACE, _TOPK = "distmult_rank", "distmult_rank_workspace_bytes", "distmult_topk"
    _REL_RANK, _REL_TOPK = "distmult_relation_rank", "distmult_relation_topk"
    _REL_RANK_WORKSPACE = "rgcn_relation_rank_workspace_bytes"
    _REL_TOPK_WORKSPACE = "rgcn_relation_topk_workspace_bytes"
    DECODER = _lib.RGCN_DECODER_DISTMULT   # the decoder kind of the ensemble entry point (rgcn_ensemble_rank)
    # device bytes one top_k / top_k_relations / rank_relations call may use beyond the split of its table; more
    # queries than fit go in several calls
    TOPK_CHUNK_BYTES = 1 << 30

    def __init__(self, codes, rel, relation_count=None):
        """relation_count = R, the candidates of the relation queries: rows 0..R-1 of `rel` (default: all rows).
        The R-GCN encoders' relation table has V rows of which only the first R are trained."""
        _check_cuda_f32("codes", codes)
        _check_cuda_f32("relation table", rel)
        self.codes, self.rel = codes, rel
        self.relation_count = rel.shape[0] if relation_count is None else int(relation_count)
        self._ws, self._ws_n, self._split_ready = None, -1, False
        # the relation queries keep their own workspace: its head is the split of rel[0:R], not of `codes`
        self._rel_ws, self._rel_split_ready = None, False

    def _check_rows(self, X, mask, name, count=None, label="V"):
        """X int32 [n,3] CUDA; mask None or int32 [n, ceil(count/32)] CUDA, count the candidates (default: V)."""
        if not (X.is_cuda and X.dtype == torch.int32 and X.is_contiguous() and X.dim() == 2 and X.shape[1] == 3):
            raise _lib.RgcnError("X must be a contiguous CUDA int32 [n,3] tensor")
        words = ((self.codes.shape[0] if count is None else count) + 31) // 32
        if mask is not None and not (mask.is_cuda and mask.dtype == torch.int32
                                     and mask.is_contiguous() and tuple(mask.shape) == (X.shape[0], words)):
            raise _lib.RgcnError("%s must be a contiguous CUDA int32 [n, ceil(%s/32)] tensor (bit masks)"
                                 % (name, label))

    def _chunk_rows(self, n, workspace_bytes, name):
        """(queries per library call, workspace bytes of such a call) for n queries, so that a call's workspace beyond
        the split of its table stays under TOPK_CHUNK_BYTES; workspace_bytes(m) sizes a call of m queries."""
        split_bytes = workspace_bytes(0)
        if split_bytes < 0:
            _lib.check(int(split_bytes), name)
        chunk = max(1, min(n, self.TOPK_CHUNK_BYTES // max(1, workspace_bytes(1) - split_bytes)))
        return chunk, workspace_bytes(chunk)

    def top_k(self, X, side, k, exclude_mask=None):
        """The k entities of highest energy for every triple of X (int32 [n,3] CUDA; side 0 predicts subjects, 1
        objects; the predicted column is not read), energy descending and the smaller id first on ties, never one
        whose bit is set in exclude_mask (uint32 [n, ceil(V/32)] CUDA, as int32, or None).  Returns (ids int32
        [n,k], energies float32 [n,k]) CUDA tensors; rows with fewer than k eligible entities end in (-1, -inf).
        Queries go to the library in chunks whose workspace beyond the split stays under TOPK_CHUNK_BYTES."""
        lib = _lib.load()
        V, d = self.codes.shape
        self._check_rows(X, exclude_mask, "exclude_mask")
        k, n = int(k), X.shape[0]
        chunk, nb = self._chunk_rows(n, lambda m: lib.rgcn_topk_workspace_bytes(V, d, m, k),
                                     "rgcn_topk_workspace_bytes")
        dev = self.codes.device
        if self._ws is None or self._ws.numel() < nb:
            self._ws, self._ws_n, self._split_ready = _workspace(nb, dev), -1, False
        ids = torch.empty((n, k), dtype=torch.int32, device=dev)
        energies = torch.empty((n, k), dtype=torch.float32, device=dev)
        for c0 in range(0, max(n, 1), chunk):
            c1 = min(n, c0 + chunk)
            rc = getattr(lib, self._TOPK)(_ptr(self.codes), _ptr(self.rel), V, self.rel.shape[0], d, _ptr(X[c0:c1]),
                                          c1 - c0, int(side), k,
                                          _ptr(None if exclude_mask is None else exclude_mask[c0:c1]),
                                          int(self._split_ready), _ptr(ids[c0:c1]), _ptr(energies[c0:c1]),
                                          _ptr(self._ws), self._ws.numel(), _stream(dev))
            _lib.check(rc, self._TOPK)
            self._split_ready = True
        return ids, energies

    def rank(self, X, side, known_mask=None):
        """X int32 [n,3] CUDA; side 0 = subjects corrupted, 1 = objects; known_mask uint32 [n, ceil(V/32)] CUDA or None.
        Returns (raw_rank, filtered_rank or None) int32 CUDA tensors."""
        lib = _lib.load()
        V, d = self.codes.shape
        self._check_rows(X, known_mask, "known_mask")
        n = X.shape[0]
        dev = self.codes.device
        if self._ws is None or n > self._ws_n:
            nb = getattr(lib, self._WORKSPACE)(V, d, n)
            if nb < 0:
                _lib.check(int(nb), self._WORKSPACE)
            self._ws, self._ws_n, self._split_ready = _workspace(nb, dev), n, False
        raw = torch.empty(n, dtype=torch.int32, device=dev)
        filt = torch.empty(n, dtype=torch.int32, device=dev) if known_mask is not None else None
        rc = getattr(lib, self._RANK)(_ptr(self.codes), _ptr(self.rel), V, self.rel.shape[0], d, _ptr(X), n,
                                      int(side), _ptr(known_mask), int(self._split_ready), _ptr(raw), _ptr(filt),
                                      _ptr(self._ws), self._ws.numel(), _stream(dev))
        _lib.check(rc, self._RANK)
        self._split_ready = True
        return raw, filt

    # ---- relation queries (h, ?, t) over rel[0:R] (distmult_relation_rank / distmult_relation_topk) ----
    def _relation_calls(self, X, mask, name, workspace_bytes):
        """Checks X and the [n, ceil(R/32)] mask, sizes the relation workspace for chunks of at most
        TOPK_CHUNK_BYTES beyond the split, and yields (c0, c1) per chunk; the split is marked ready after each."""
        self._check_rows(X, mask, name, self.relation_count, "R")
        n = X.shape[0]
        chunk, nb = self._chunk_rows(n, workspace_bytes, "relation workspace bytes")
        if self._rel_ws is None or self._rel_ws.numel() < nb:
            self._rel_ws, self._rel_split_ready = _workspace(nb, self.codes.device), False
        for c0 in range(0, max(n, 1), chunk):
            yield c0, min(n, c0 + chunk)
            self._rel_split_ready = True

    def rank_relations(self, X, known_mask=None):
        """Ranks of the relation X[t, 1] in [0, R) among all R relations for the pair (X[t, 0], X[t, 2]), by the
        rules of rank: raw = #{r : score_r >= gold score}, filtered = raw - #{known r with score >= gold} + 1.
        X int32 [n,3] CUDA; known_mask uint32 [n, ceil(R/32)] CUDA (as int32) or None.  Returns (raw_rank,
        filtered_rank or None) int32 CUDA tensors."""
        lib = _lib.load()
        R, d = self.relation_count, self.codes.shape[1]
        dev = self.codes.device
        n = X.shape[0]
        raw = torch.empty(n, dtype=torch.int32, device=dev)
        filt = torch.empty(n, dtype=torch.int32, device=dev) if known_mask is not None else None
        fn = getattr(lib, self._REL_RANK)
        for c0, c1 in self._relation_calls(X, known_mask, "known_mask",
                                           lambda m: getattr(lib, self._REL_RANK_WORKSPACE)(R, d, m)):
            rc = fn(_ptr(self.codes), _ptr(self.rel), self.codes.shape[0], self.rel.shape[0], R, d, _ptr(X[c0:c1]),
                    c1 - c0, _ptr(None if known_mask is None else known_mask[c0:c1]), int(self._rel_split_ready),
                    _ptr(raw[c0:c1]), _ptr(None if filt is None else filt[c0:c1]), _ptr(self._rel_ws),
                    self._rel_ws.numel(), _stream(dev))
            _lib.check(rc, self._REL_RANK)
        return raw, filt

    def top_k_relations(self, X, k, exclude_mask=None):
        """The k relations of rel[0:R] of highest energy for every pair (X[t, 0], ?, X[t, 2]) (the relation column
        is not read), energy descending and the smaller id first on ties, never one whose bit is set in
        exclude_mask (uint32 [n, ceil(R/32)] CUDA, as int32, or None).  Returns (ids int32 [n,k], energies float32
        [n,k]) CUDA tensors; rows with fewer than k eligible relations end in (-1, -inf)."""
        lib = _lib.load()
        R, d, k = self.relation_count, self.codes.shape[1], int(k)
        dev = self.codes.device
        n = X.shape[0]
        ids = torch.empty((n, k), dtype=torch.int32, device=dev)
        energies = torch.empty((n, k), dtype=torch.float32, device=dev)
        fn = getattr(lib, self._REL_TOPK)
        for c0, c1 in self._relation_calls(X, exclude_mask, "exclude_mask",
                                           lambda m: getattr(lib, self._REL_TOPK_WORKSPACE)(R, d, m, k)):
            rc = fn(_ptr(self.codes), _ptr(self.rel), self.codes.shape[0], self.rel.shape[0], R, d, _ptr(X[c0:c1]),
                    c1 - c0, k, _ptr(None if exclude_mask is None else exclude_mask[c0:c1]),
                    int(self._rel_split_ready), _ptr(ids[c0:c1]), _ptr(energies[c0:c1]), _ptr(self._rel_ws),
                    self._rel_ws.numel(), _stream(dev))
            _lib.check(rc, self._REL_TOPK)
        return ids, energies


class ComplexRanker(DistMultRanker):
    """Fused all-entity scoring + ranking of the ComplEx decoder (rgcn_complex_rank): same interface and split reuse
    as DistMultRanker, the query rows are the complex products of complex.py:77-106."""
    _RANK, _WORKSPACE, _TOPK = "rgcn_complex_rank", "rgcn_complex_rank_workspace_bytes", "rgcn_complex_topk"
    _REL_RANK, _REL_TOPK = "rgcn_complex_relation_rank", "rgcn_complex_relation_topk"
    DECODER = _lib.RGCN_DECODER_COMPLEX


class QuatERanker(object):
    """Fused all-entity and all-relation ranking and top-k of the QuatE decoder (rgcn_quate_rank / _topk /
    _relation_rank / _relation_topk): DistMultRanker's interface, workspaces and split reuse, with QuatE's query rows
    (side 1 h (x) rh, side 0 t (x) conj(rh), relation pairs conj(h) (x) t against the normalised rel[0:R]).  Not a
    DistMultRanker: it is no member of the fused ensemble, whose kernels score DistMult and ComplEx rows only."""
    _RANK, _WORKSPACE, _TOPK = "rgcn_quate_rank", "distmult_rank_workspace_bytes", "rgcn_quate_topk"
    _REL_RANK, _REL_TOPK = "rgcn_quate_relation_rank", "rgcn_quate_relation_topk"
    _REL_RANK_WORKSPACE = "rgcn_quate_relation_rank_workspace_bytes"
    _REL_TOPK_WORKSPACE = "rgcn_quate_relation_topk_workspace_bytes"
    TOPK_CHUNK_BYTES = DistMultRanker.TOPK_CHUNK_BYTES

    __init__ = DistMultRanker.__init__
    _check_rows = DistMultRanker._check_rows
    _chunk_rows = DistMultRanker._chunk_rows
    _relation_calls = DistMultRanker._relation_calls
    rank = DistMultRanker.rank
    top_k = DistMultRanker.top_k
    rank_relations = DistMultRanker.rank_relations
    top_k_relations = DistMultRanker.top_k_relations


def quate_query_rows(codes, rel, X, side):
    """QuatE query rows Q [n, d] of the triples X (int32 [n, 3] CUDA): side 1 h (x) rh (scored against the objects),
    side 0 t (x) conj(rh) (against the subjects); <Q[t], codes[v]> is the energy of the triple with v in the predicted
    column (rgcn_quate_query_rows)."""
    _check_cuda_f32("codes", codes)
    _check_cuda_f32("relation table", rel)
    if not (X.is_cuda and X.dtype == torch.int32 and X.is_contiguous() and X.dim() == 2 and X.shape[1] == 3):
        raise _lib.RgcnError("X must be a contiguous CUDA int32 [n,3] tensor")
    V, d = codes.shape
    n = X.shape[0]
    Q = torch.empty((n, d), dtype=torch.float32, device=codes.device)
    lib = _lib.load()
    rc = lib.rgcn_quate_query_rows(_ptr(codes), _ptr(rel), V, rel.shape[0], d, _ptr(X), n, int(side), _ptr(Q),
                                   _stream(codes.device))
    _lib.check(rc, "rgcn_quate_query_rows")
    return Q


class HolERanker(object):
    """Fused all-entity and all-relation ranking and top-k of the HolE decoder (rgcn_hole_rank / _topk /
    _relation_rank / _relation_topk) over tables in the HolE basis (hole_transform): DistMultRanker's interface,
    workspaces and split reuse, with HolE's query rows (side 1 w (h r), side 0 w conj(r) t, relation pairs
    w conj(h) t against rel[0:R]).  Not a DistMultRanker: it is no member of the fused ensemble, whose kernels score
    DistMult and ComplEx rows only."""
    _RANK, _WORKSPACE, _TOPK = "rgcn_hole_rank", "distmult_rank_workspace_bytes", "rgcn_hole_topk"
    _REL_RANK, _REL_TOPK = "rgcn_hole_relation_rank", "rgcn_hole_relation_topk"
    _REL_RANK_WORKSPACE = DistMultRanker._REL_RANK_WORKSPACE
    _REL_TOPK_WORKSPACE = DistMultRanker._REL_TOPK_WORKSPACE
    TOPK_CHUNK_BYTES = DistMultRanker.TOPK_CHUNK_BYTES

    __init__ = DistMultRanker.__init__
    _check_rows = DistMultRanker._check_rows
    _chunk_rows = DistMultRanker._chunk_rows
    _relation_calls = DistMultRanker._relation_calls
    rank = DistMultRanker.rank
    top_k = DistMultRanker.top_k
    rank_relations = DistMultRanker.rank_relations
    top_k_relations = DistMultRanker.top_k_relations


def hole_query_rows(codes, rel, X, side):
    """HolE query rows Q [n, d] of the triples X (int32 [n, 3] CUDA) over tables in the HolE basis: side 1 w (h r)
    (scored against the objects), side 0 w conj(r) t (against the subjects); <Q[t], codes[v]> is the energy of the
    triple with v in the predicted column (rgcn_hole_query_rows)."""
    _check_cuda_f32("codes", codes)
    _check_cuda_f32("relation table", rel)
    if not (X.is_cuda and X.dtype == torch.int32 and X.is_contiguous() and X.dim() == 2 and X.shape[1] == 3):
        raise _lib.RgcnError("X must be a contiguous CUDA int32 [n,3] tensor")
    V, d = codes.shape
    n = X.shape[0]
    Q = torch.empty((n, d), dtype=torch.float32, device=codes.device)
    lib = _lib.load()
    rc = lib.rgcn_hole_query_rows(_ptr(codes), _ptr(rel), V, rel.shape[0], d, _ptr(X), n, int(side), _ptr(Q),
                                  _stream(codes.device))
    _lib.check(rc, "rgcn_hole_query_rows")
    return Q


class RotateRanker(object):
    """All-entity ranking of the RotatE decoder by distance (rgcn_rotate_rank): rank(X, side, known_mask) as
    DistMultRanker.rank, with D_v = sum_k |q_k - v_k| <= D_gold in place of score >= gold score, so the ranks do not
    depend on the margin.  RotatE has no fused top-k or relation prediction, and is no member of the fused ensemble
    (EnsembleRanker takes DistMultRanker objects only)."""

    def __init__(self, codes, rel, relation_count=None):
        _check_cuda_f32("codes", codes)
        _check_cuda_f32("relation table", rel)
        self.codes, self.rel = codes, rel
        self.relation_count = rel.shape[0] if relation_count is None else int(relation_count)
        self._ws, self._ws_n = None, -1

    _check_rows = DistMultRanker._check_rows

    def rank(self, X, side, known_mask=None):
        """X int32 [n,3] CUDA; side 0 = subjects corrupted, 1 = objects; known_mask uint32 [n, ceil(V/32)] CUDA (as
        int32) or None.  Returns (raw_rank, filtered_rank or None) int32 CUDA tensors."""
        lib = _lib.load()
        V, d = self.codes.shape
        self._check_rows(X, known_mask, "known_mask")
        n = X.shape[0]
        dev = self.codes.device
        if self._ws is None or n > self._ws_n:
            nb = lib.rgcn_rotate_rank_workspace_bytes(V, d, n)
            if nb < 0:
                _lib.check(int(nb), "rgcn_rotate_rank_workspace_bytes")
            self._ws, self._ws_n = _workspace(nb, dev), n
        raw = torch.empty(n, dtype=torch.int32, device=dev)
        filt = torch.empty(n, dtype=torch.int32, device=dev) if known_mask is not None else None
        rc = lib.rgcn_rotate_rank(_ptr(self.codes), _ptr(self.rel), V, self.rel.shape[0], d, _ptr(X), n, int(side),
                                  _ptr(known_mask), _ptr(raw), _ptr(filt), _ptr(self._ws), self._ws.numel(),
                                  _stream(dev))
        _lib.check(rc, "rgcn_rotate_rank")
        return raw, filt

    def top_k(self, X, side, k, exclude_mask=None):
        raise NotImplementedError("the RotatE decoder has no top-k entity prediction")

    def rank_relations(self, X, known_mask=None):
        raise NotImplementedError("the RotatE decoder has no relation prediction")

    def top_k_relations(self, X, k, exclude_mask=None):
        raise NotImplementedError("the RotatE decoder has no relation prediction")


class TransERanker(object):
    """Ranking and top-k of the TransE decoder by L1 distance (rgcn_transe_rank / _topk / _relation_rank /
    _relation_topk), with DistMultRanker's interface: every query ranks the rows of a table by D = sum_k |q_k - v_k|,
    D <= D_gold in place of score >= gold score, so the ranks do not depend on the margin.  top_k / top_k_relations
    return the energies gamma - D of the k smallest D (gamma = 0: -D).  There is no split to reuse; queries go to the
    library in chunks whose workspace stays under TOPK_CHUNK_BYTES.  No member of the fused ensemble."""
    TOPK_CHUNK_BYTES = DistMultRanker.TOPK_CHUNK_BYTES

    def __init__(self, codes, rel, relation_count=None, gamma=0.0):
        _check_cuda_f32("codes", codes)
        _check_cuda_f32("relation table", rel)
        self.codes, self.rel = codes, rel
        self.relation_count = rel.shape[0] if relation_count is None else int(relation_count)
        self.gamma = _check_gamma(gamma)
        self._ws = None

    _check_rows = DistMultRanker._check_rows
    _chunk_rows = DistMultRanker._chunk_rows

    def _calls(self, X, mask, name, relations, workspace_bytes):
        """Checks X and the mask ([n, ceil(V/32)], or [n, ceil(R/32)] for relation queries), sizes the workspace for
        chunks of at most TOPK_CHUNK_BYTES, and yields (c0, c1) per chunk."""
        if relations:
            self._check_rows(X, mask, name, self.relation_count, "R")
        else:
            self._check_rows(X, mask, name)
        n = X.shape[0]
        chunk, nb = self._chunk_rows(n, workspace_bytes, "TransE workspace bytes")
        if self._ws is None or self._ws.numel() < nb:
            self._ws = _workspace(nb, self.codes.device)
        for c0 in range(0, max(n, 1), chunk):
            yield c0, min(n, c0 + chunk)

    # lead: the arguments before X; side: () for relation queries, else (side,), which goes after n
    def _rank(self, entry, X, known_mask, lead, side, workspace_bytes):
        lib = _lib.load()
        dev = self.codes.device
        n = X.shape[0]
        raw = torch.empty(n, dtype=torch.int32, device=dev)
        filt = torch.empty(n, dtype=torch.int32, device=dev) if known_mask is not None else None
        for c0, c1 in self._calls(X, known_mask, "known_mask", not side, workspace_bytes):
            rc = getattr(lib, entry)(*lead, _ptr(X[c0:c1]), c1 - c0, *side,
                                     _ptr(None if known_mask is None else known_mask[c0:c1]), _ptr(raw[c0:c1]),
                                     _ptr(None if filt is None else filt[c0:c1]), _ptr(self._ws), self._ws.numel(),
                                     _stream(dev))
            _lib.check(rc, entry)
        return raw, filt

    def _top_k(self, entry, X, k, exclude_mask, lead, side, workspace_bytes):
        lib = _lib.load()
        dev = self.codes.device
        k, n = int(k), X.shape[0]
        ids = torch.empty((n, k), dtype=torch.int32, device=dev)
        energies = torch.empty((n, k), dtype=torch.float32, device=dev)
        for c0, c1 in self._calls(X, exclude_mask, "exclude_mask", not side, workspace_bytes):
            rc = getattr(lib, entry)(*lead, _ptr(X[c0:c1]), c1 - c0, *side, k,
                                     _ptr(None if exclude_mask is None else exclude_mask[c0:c1]), self.gamma,
                                     _ptr(ids[c0:c1]), _ptr(energies[c0:c1]), _ptr(self._ws), self._ws.numel(),
                                     _stream(dev))
            _lib.check(rc, entry)
        return ids, energies

    def _lead(self, relations):
        V, d = self.codes.shape
        head = (_ptr(self.codes), _ptr(self.rel), V, self.rel.shape[0])
        return head + ((self.relation_count, d) if relations else (d,))

    def rank(self, X, side, known_mask=None):
        """X int32 [n,3] CUDA; side 0 = subjects corrupted (q = t - r), 1 = objects (q = h + r); known_mask uint32
        [n, ceil(V/32)] CUDA (as int32) or None.  Returns (raw_rank, filtered_rank or None) int32 CUDA tensors."""
        lib = _lib.load()
        V, d = self.codes.shape
        return self._rank("rgcn_transe_rank", X, known_mask, self._lead(False), (int(side),),
                          lambda m: lib.rgcn_transe_rank_workspace_bytes(V, d, m))

    def top_k(self, X, side, k, exclude_mask=None):
        """The k entities of smallest distance for every triple of X (side 0 predicts subjects, 1 objects; the
        predicted column is not read), D ascending and the smaller id first on ties, never one whose bit is set in
        exclude_mask (uint32 [n, ceil(V/32)] CUDA, as int32, or None).  Returns (ids int32 [n,k], energies
        gamma - D float32 [n,k]) CUDA tensors; rows with fewer than k eligible entities end in (-1, -inf)."""
        lib = _lib.load()
        V, d = self.codes.shape
        return self._top_k("rgcn_transe_topk", X, k, exclude_mask, self._lead(False), (int(side),),
                           lambda m: lib.rgcn_transe_topk_workspace_bytes(V, d, m, int(k)))

    def rank_relations(self, X, known_mask=None):
        """Ranks of the relation X[t, 1] in [0, R) among rel[0:R] for the pair (X[t, 0], X[t, 2]), q = t - h, by the
        rules of rank; known_mask uint32 [n, ceil(R/32)] CUDA (as int32) or None."""
        lib = _lib.load()
        R, d = self.relation_count, self.codes.shape[1]
        return self._rank("rgcn_transe_relation_rank", X, known_mask, self._lead(True), (),
                          lambda m: lib.rgcn_transe_relation_rank_workspace_bytes(R, d, m))

    def top_k_relations(self, X, k, exclude_mask=None):
        """The k relations of rel[0:R] of smallest distance for every pair (X[t, 0], ?, X[t, 2]) (the relation column
        is not read), with top_k's order, exclusion and padding; exclude_mask uint32 [n, ceil(R/32)] CUDA or None."""
        lib = _lib.load()
        R, d = self.relation_count, self.codes.shape[1]
        return self._top_k("rgcn_transe_relation_topk", X, k, exclude_mask, self._lead(True), (),
                           lambda m: lib.rgcn_transe_relation_topk_workspace_bytes(R, d, m, int(k)))


class EnsembleRanker(object):
    """Fused ranking under the weighted sum of two members' scores (R-GCN+; rgcn_ensemble_rank): member A scored by
    ranker_a with weight w, member B by ranker_b with 1 - w, combined in float64.  The members are DistMultRanker /
    ComplexRanker objects over the same V entities; their code widths may differ.  The ensemble keeps its own
    workspace, whose head holds both members' hi/lo splits, made once and reused by every later call."""

    def __init__(self, ranker_a, ranker_b, weight):
        for name, r in (("ranker_a", ranker_a), ("ranker_b", ranker_b)):
            if not isinstance(r, DistMultRanker):
                raise TypeError("%s must be a DistMultRanker or ComplexRanker, got %s" % (name, type(r).__name__))
        if ranker_a.codes.shape[0] != ranker_b.codes.shape[0]:
            raise ValueError("the members rank different entity sets (%d and %d entities)"
                             % (ranker_a.codes.shape[0], ranker_b.codes.shape[0]))
        if ranker_a.codes.device != ranker_b.codes.device:
            raise ValueError("the members live on different devices (%s and %s)"
                             % (ranker_a.codes.device, ranker_b.codes.device))
        weight = float(weight)
        if not 0.0 <= weight <= 1.0:   # also refuses NaN
            raise ValueError("the weight must be in [0, 1], got %r" % weight)
        self.a, self.b, self.weight = ranker_a, ranker_b, weight
        self._ws, self._ws_n, self._split_ready = None, -1, False
        # relation queries keep their own workspace, with both members' splits of rel[0:R] at its head
        self._rel_ws, self._rel_split_ready = None, False

    def rank(self, X, side, known_mask=None):
        """As DistMultRanker.rank, with c = w s_A + (1 - w) s_B in place of the single score.  X int32 [n,3] CUDA;
        side 0 = subjects corrupted, 1 = objects; known_mask uint32 [n, ceil(V/32)] CUDA (as int32) or None.
        Returns (raw_rank, filtered_rank or None) int32 CUDA tensors."""
        lib = _lib.load()
        a, b = self.a, self.b
        V, d_a = a.codes.shape
        d_b = b.codes.shape[1]
        a._check_rows(X, known_mask, "known_mask")
        n = X.shape[0]
        dev = a.codes.device
        if self._ws is None or n > self._ws_n:
            nb = lib.rgcn_ensemble_rank_workspace_bytes(V, d_a, d_b, n)
            if nb < 0:
                _lib.check(int(nb), "rgcn_ensemble_rank_workspace_bytes")
            self._ws, self._ws_n, self._split_ready = _workspace(nb, dev), n, False
        raw = torch.empty(n, dtype=torch.int32, device=dev)
        filt = torch.empty(n, dtype=torch.int32, device=dev) if known_mask is not None else None
        rc = lib.rgcn_ensemble_rank(a.DECODER, _ptr(a.codes), _ptr(a.rel), a.rel.shape[0], d_a,
                                    b.DECODER, _ptr(b.codes), _ptr(b.rel), b.rel.shape[0], d_b,
                                    V, self.weight, _ptr(X), n, int(side), _ptr(known_mask), int(self._split_ready),
                                    _ptr(raw), _ptr(filt), _ptr(self._ws), self._ws.numel(), _stream(dev))
        _lib.check(rc, "rgcn_ensemble_rank")
        self._split_ready = True
        return raw, filt

    def _members(self):
        """The leading arguments of every ensemble entry point: both members' decoder, codes, relation table,
        table rows and width."""
        a, b = self.a, self.b
        return (a.DECODER, _ptr(a.codes), _ptr(a.rel), a.rel.shape[0], a.codes.shape[1],
                b.DECODER, _ptr(b.codes), _ptr(b.rel), b.rel.shape[0], b.codes.shape[1])

    def _outputs(self, n, k):
        dev = self.a.codes.device
        return (torch.empty((n, k), dtype=torch.int32, device=dev), torch.empty((n, k), dtype=torch.float64, device=dev),
                torch.empty((n, k), dtype=torch.float64, device=dev))

    def top_k(self, X, side, k, exclude_mask=None):
        """The k entities of best combined score for every triple of X (int32 [n,3] CUDA; side 0 predicts subjects,
        1 objects; the predicted column is not read), in the order of u = w sigma(-E_A) + (1 - w) sigma(-E_B)
        ascending (double), the smaller id first on ties, never one whose bit is set in exclude_mask (uint32
        [n, ceil(V/32)] CUDA, as int32, or None).  Returns CUDA tensors (ids int32 [n,k], u float64 [n,k], scores
        float64 [n,k] = 1 - u); rows with fewer than k eligible entities end in (-1, +inf, 0).  Queries go to the
        library in chunks whose workspace beyond the splits stays under TOPK_CHUNK_BYTES; the entity splits are
        shared with rank."""
        lib = _lib.load()
        a = self.a
        V, d_a = a.codes.shape
        d_b = self.b.codes.shape[1]
        a._check_rows(X, exclude_mask, "exclude_mask")
        k, n = int(k), X.shape[0]
        chunk, nb = a._chunk_rows(n, lambda m: lib.rgcn_ensemble_topk_workspace_bytes(V, d_a, d_b, m, k),
                                  "rgcn_ensemble_topk_workspace_bytes")
        dev = a.codes.device
        if self._ws is None or self._ws.numel() < nb:
            self._ws, self._ws_n, self._split_ready = _workspace(nb, dev), -1, False
        ids, u, scores = self._outputs(n, k)
        for c0 in range(0, max(n, 1), chunk):
            c1 = min(n, c0 + chunk)
            rc = lib.rgcn_ensemble_topk(*self._members(), V, self.weight, _ptr(X[c0:c1]), c1 - c0, int(side), k,
                                        _ptr(None if exclude_mask is None else exclude_mask[c0:c1]),
                                        int(self._split_ready), _ptr(ids[c0:c1]), _ptr(u[c0:c1]),
                                        _ptr(scores[c0:c1]), _ptr(self._ws), self._ws.numel(), _stream(dev))
            _lib.check(rc, "rgcn_ensemble_topk")
            self._split_ready = True
        return ids, u, scores

    # ---- relation queries (h, ?, t) over the first R relations of both members ----
    @property
    def relation_count(self):
        """R, the relation candidates both members share; ValueError when they differ."""
        if self.a.relation_count != self.b.relation_count:
            raise ValueError("the members predict different relation sets (%d and %d relations)"
                             % (self.a.relation_count, self.b.relation_count))
        return self.a.relation_count

    def _relation_calls(self, X, mask, name, workspace_bytes):
        """As DistMultRanker._relation_calls, with the ensemble's own relation workspace (both members' splits of
        rel[0:R] at its head).  Relation queries need both members to have the same R candidates; entity ranking
        and top-k do not."""
        a = self.a
        a._check_rows(X, mask, name, self.relation_count, "R")
        n = X.shape[0]
        chunk, nb = a._chunk_rows(n, workspace_bytes, "relation workspace bytes")
        if self._rel_ws is None or self._rel_ws.numel() < nb:
            self._rel_ws, self._rel_split_ready = _workspace(nb, a.codes.device), False
        for c0 in range(0, max(n, 1), chunk):
            yield c0, min(n, c0 + chunk)
            self._rel_split_ready = True

    def rank_relations(self, X, known_mask=None):
        """Ranks of the relation X[t, 1] in [0, R) among the R relations for the pair (X[t, 0], X[t, 2]) under the
        combined score, by the rules of rank.  X int32 [n,3] CUDA; known_mask uint32 [n, ceil(R/32)] CUDA (as int32)
        or None.  Returns (raw_rank, filtered_rank or None) int32 CUDA tensors."""
        lib = _lib.load()
        R, V = self.relation_count, self.a.codes.shape[0]
        d_a, d_b = self.a.codes.shape[1], self.b.codes.shape[1]
        dev = self.a.codes.device
        n = X.shape[0]
        raw = torch.empty(n, dtype=torch.int32, device=dev)
        filt = torch.empty(n, dtype=torch.int32, device=dev) if known_mask is not None else None
        for c0, c1 in self._relation_calls(X, known_mask, "known_mask",
                                           lambda m: lib.rgcn_ensemble_relation_rank_workspace_bytes(R, d_a, d_b, m)):
            rc = lib.rgcn_ensemble_relation_rank(*self._members(), V, R, self.weight, _ptr(X[c0:c1]), c1 - c0,
                                                 _ptr(None if known_mask is None else known_mask[c0:c1]),
                                                 int(self._rel_split_ready), _ptr(raw[c0:c1]),
                                                 _ptr(None if filt is None else filt[c0:c1]), _ptr(self._rel_ws),
                                                 self._rel_ws.numel(), _stream(dev))
            _lib.check(rc, "rgcn_ensemble_relation_rank")
        return raw, filt

    def top_k_relations(self, X, k, exclude_mask=None):
        """The k relations of the first R of best combined score for every pair (X[t, 0], ?, X[t, 2]) (the relation
        column is not read), in top_k's order, never one whose bit is set in exclude_mask (uint32 [n, ceil(R/32)]
        CUDA, as int32, or None).  Returns CUDA tensors (ids int32 [n,k], u float64 [n,k], scores float64 [n,k]);
        rows with fewer than k eligible relations end in (-1, +inf, 0)."""
        lib = _lib.load()
        R, V, k = self.relation_count, self.a.codes.shape[0], int(k)
        d_a, d_b = self.a.codes.shape[1], self.b.codes.shape[1]
        dev = self.a.codes.device
        n = X.shape[0]
        ids, u, scores = self._outputs(n, k)
        for c0, c1 in self._relation_calls(
                X, exclude_mask, "exclude_mask",
                lambda m: lib.rgcn_ensemble_relation_topk_workspace_bytes(R, d_a, d_b, m, k)):
            rc = lib.rgcn_ensemble_relation_topk(*self._members(), V, R, self.weight, _ptr(X[c0:c1]), c1 - c0, k,
                                                 _ptr(None if exclude_mask is None else exclude_mask[c0:c1]),
                                                 int(self._rel_split_ready), _ptr(ids[c0:c1]), _ptr(u[c0:c1]),
                                                 _ptr(scores[c0:c1]), _ptr(self._rel_ws), self._rel_ws.numel(),
                                                 _stream(dev))
            _lib.check(rc, "rgcn_ensemble_relation_topk")
        return ids, u, scores


# ---- 1-N training (distmult_one_to_n / rgcn_complex_one_to_n, include/rgcn_b200.h) ----
ONE_TO_N_DECODERS = {"distmult": "distmult_one_to_n", "complex": "rgcn_complex_one_to_n",
                     "quate": "rgcn_quate_one_to_n", "hole": "rgcn_hole_one_to_n"}
# device bytes of the per-query buffers (energy gradients Gt [V, chunk], query rows and their gradients) of one
# internal pass; more queries than fit run in several passes of one call
ONE_TO_N_CHUNK_BYTES = 1 << 30


def one_to_n_queries(triples):
    """The de-duplicated 1-N queries of positive triples [m, 3]: (s, r, 1) asks for the objects of (s, r, ?) and
    (o, r, 0) for the subjects of (?, r, o).  int32 [n, 3] rows (anchor, relation, side), sorted by (side, relation,
    anchor): all subject queries first.  The rows are de-duplicated as the 1-D keys (side R' + r) V' + anchor
    (V', R' one past the largest ids): one sort of int64 keys, far faster than a de-duplication of rows."""
    tri = np.asarray(triples, dtype=np.int64).reshape(-1, 3)
    if len(tri) == 0:
        return np.zeros((0, 3), np.int32)
    V, R = int(max(tri[:, 0].max(), tri[:, 2].max())) + 1, int(tri[:, 1].max()) + 1
    keys = np.sort(np.concatenate([tri[:, 1] * V + tri[:, 2], (R + tri[:, 1]) * V + tri[:, 0]]))
    keys = keys[np.concatenate([[True], keys[1:] != keys[:-1]])]
    q = np.empty((len(keys), 3), np.int32)
    q[:, 0] = keys % V
    q[:, 1] = (keys // V) % R
    q[:, 2] = keys // (V * R)
    return q


def _check_queries(queries, V, R):
    q = np.ascontiguousarray(np.asarray(queries, dtype=np.int32).reshape(-1, 3))
    if len(q) and (q[:, 0].min() < 0 or q[:, 0].max() >= V or q[:, 1].min() < 0 or q[:, 1].max() >= R
                   or not np.isin(q[:, 2], (0, 1)).all()):
        raise ValueError("1-N queries need 0 <= anchor < %d, 0 <= relation < %d and side in {0, 1}" % (V, R))
    return q


class OneToNLabels(object):
    """The 1-N targets of a training split on the device: a CSR from the query key (2 relation + side) V + anchor to
    the entities that complete a training triple, built once; rows(queries) writes the [n, ceil(V/32)] label bits of a
    step with one library call (rgcn_one_to_n_labels)."""

    def __init__(self, triples, n_entities, n_relations, device):
        tri = np.asarray(triples, dtype=np.int64).reshape(-1, 3)
        V = self.V = int(n_entities)
        self.R = int(n_relations)
        if len(tri) and (tri[:, [0, 2]].min() < 0 or tri[:, [0, 2]].max() >= V or tri[:, 1].min() < 0
                         or tri[:, 1].max() >= self.R):
            raise ValueError("OneToNLabels: training triples need entity ids in [0, %d) and relation ids in [0, %d)"
                             % (V, self.R))
        s, r, o = tri[:, 0], tri[:, 1], tri[:, 2]
        # (query key, entity) pairs as one sorted, de-duplicated int64 key V + entity
        pairs = np.sort(np.concatenate([((2 * r + 1) * V + s) * V + o, ((2 * r) * V + o) * V + s]))
        pairs = pairs[np.concatenate([[True], pairs[1:] != pairs[:-1]])]
        qkey, ent = pairs // V, pairs % V
        starts = np.flatnonzero(np.concatenate([[True], qkey[1:] != qkey[:-1]]))
        dev = torch.device(device)
        self.keys = torch.as_tensor(qkey[starts].astype(np.int64), device=dev)
        self.offsets = torch.as_tensor(np.append(starts, len(pairs)).astype(np.int64), device=dev)
        self.entities = torch.as_tensor(ent.astype(np.int32), device=dev)
        self.device = dev

    def rows(self, queries):
        """uint32 label bits [n, ceil(V/32)] (as int32) of host queries (anchor, relation, side): bit e of an object
        query (s, r, 1) is set iff (s, r, e) is a training triple, of a subject query (o, r, 0) iff (e, r, o) is."""
        q = _check_queries(queries, self.V, self.R)
        bits = torch.empty(len(q), (self.V + 31) // 32, dtype=torch.int32, device=self.device)
        _call("rgcn_one_to_n_labels", "rgcn_one_to_n_labels_workspace_bytes", (len(q),),
              (_ptr(self.keys), _ptr(self.offsets), _ptr(self.entities), self.keys.numel(), self.V, self.R,
               _np_ptr(q), len(q), _ptr(bits)), self.device)
        return bits


class _OneToNFn(torch.autograd.Function):
    """Returns (loss, reg) of distmult_one_to_n / rgcn_complex_one_to_n / rgcn_quate_one_to_n / rgcn_hole_one_to_n.
    When codes or rel need a gradient, the forward also writes the gradient of the loss alone (g_scale = (1, 0)); the
    gradient is linear in the two upstream scalars, so the backward is rgcn_one_to_n_finish: one scaling pass and the
    L2 term, no GEMM."""

    @staticmethod
    def forward(ctx, codes, rel, labels, queries, smoothing, entry, R, chunk, grads):
        V, d = codes.shape
        dev = codes.device
        loss = torch.empty(2, dtype=torch.float32, device=dev)
        dcodes = torch.empty_like(codes) if grads else None
        drel = torch.empty_like(rel) if grads else None
        g_loss_only = torch.tensor([1.0, 0.0], dtype=torch.float32, device=dev) if grads else None
        _call(entry, "rgcn_one_to_n_workspace_bytes", (V, d, len(queries), chunk),
              (_ptr(codes), _ptr(rel), V, rel.shape[0], R, d, _np_ptr(queries), len(queries), _ptr(labels),
               smoothing, _ptr(g_loss_only), _ptr(loss), _ptr(dcodes), _ptr(drel), chunk), dev)
        ctx.args = (queries, R)
        if grads:
            ctx.save_for_backward(codes, rel, dcodes, drel)
        return loss[0], loss[1]

    @staticmethod
    def backward(ctx, g_loss, g_reg):
        codes, rel, dcodes_loss, drel_loss = ctx.saved_tensors
        queries, R = ctx.args
        V, d = codes.shape
        dev = codes.device
        gs = torch.zeros(2, dtype=torch.float32, device=dev)
        if g_loss is not None:
            gs[0] = g_loss
        if g_reg is not None:
            gs[1] = g_reg
        dcodes, drel = torch.empty_like(codes), torch.empty_like(rel)
        _call("rgcn_one_to_n_finish", "rgcn_one_to_n_finish_workspace_bytes", (len(queries),),
              (_ptr(codes), _ptr(rel), V, rel.shape[0], R, d, _np_ptr(queries), len(queries), _ptr(gs),
               _ptr(dcodes_loss), _ptr(drel_loss), _ptr(dcodes), _ptr(drel)), dev)
        return dcodes, drel, None, None, None, None, None, None, None


def one_to_n_loss(codes, rel, queries, labels, smoothing, decoder, relation_count=None):
    """1-N loss of host queries (anchor, relation, side) int32 [n, 3] against every entity, with the label bits of
    OneToNLabels.rows and label smoothing eps in [0, 1): returns (loss, reg), loss = the mean over the n V scores of the
    sigmoid cross-entropy against y' = (1 - eps) y + eps / V, reg = (|codes[anchor]|^2 + |rel[r]|^2) / (n d) summed
    over the queries (the decoders' un-scaled L2 term).  decoder is "distmult", "complex", "quate" or "hole" (on tables
    in the HolE basis); the relation ids must be below relation_count (default: all rows of rel).  Differentiable in
    codes and rel."""
    if decoder not in ONE_TO_N_DECODERS:
        raise ValueError("one_to_n_loss: decoder must be one of %s, got %r" % (sorted(ONE_TO_N_DECODERS), decoder))
    _check_cuda_f32("codes", codes)
    _check_cuda_f32("relation table", rel)
    V, d = codes.shape
    R = rel.shape[0] if relation_count is None else int(relation_count)
    q = _check_queries(queries, V, R)
    words = (V + 31) // 32
    if not (labels.is_cuda and labels.dtype == torch.int32 and labels.is_contiguous()
            and tuple(labels.shape) == (len(q), words)):
        raise _lib.RgcnError("labels must be a contiguous CUDA int32 [n, ceil(V/32)] tensor (bit rows)")
    if not 0.0 <= float(smoothing) < 1.0:
        raise ValueError("one_to_n_loss: label smoothing must be in [0, 1), got %r" % (smoothing,))
    chunk = max(1, min(len(q), ONE_TO_N_CHUNK_BYTES // ((V + 4 * d) * 4)))
    # inside Function.forward the grad mode is off and needs_input_grad ignores torch.no_grad(): decide here
    grads = torch.is_grad_enabled() and (codes.requires_grad or rel.requires_grad)
    return _OneToNFn.apply(codes, rel, labels, q, float(smoothing), ONE_TO_N_DECODERS[decoder], R, chunk, grads)


# ---- ConvE (rgcn_conve_*, include/rgcn_b200.h): the query network in front of the 1-N, rank and top-k paths ----
class ConvEWeights(tuple):
    """(rel_inv [R, d], filters [C, 3, 3], conv_bias [C], W_fc [F, d], b_fc [d]) of a ConvE decoder with image height
    h (d = h w): the reciprocal relation rows and the network weights, CUDA float32, contiguous."""

    def __new__(cls, rel_inv, filters, conv_bias, W_fc, b_fc, h):
        self = tuple.__new__(cls, (rel_inv, filters, conv_bias, W_fc, b_fc))
        self.h = int(h)
        return self

    @property
    def C(self):
        return self[1].shape[0]

    def check(self, d):
        """Checks the shapes against the code width d; returns F."""
        h, C = self.h, self[1].shape[0] if self[1].dim() else 0
        if h < 2 or d % h or d // h < 3 or C < 1 or d % 4:
            raise ValueError("ConvE needs d %% 4 == 0, d = h w with h >= 2, w >= 3 and C >= 1 filters (d = %d, h = %d, "
                             "C = %d)" % (d, h, C))
        F = C * (2 * h - 2) * (d // h - 2)
        for name, t, shape in (("rel_inv", self[0], (self[0].shape[0], d)), ("filters", self[1], (C, 3, 3)),
                               ("conv_bias", self[2], (C,)), ("W_fc", self[3], (F, d)), ("b_fc", self[4], (d,))):
            _check_cuda_f32(name, t, shape)
        return F


def _conve_net(weights, masks=(None, None, None), keeps=(1.0, 1.0, 1.0)):
    rel_inv, filters, conv_bias, W_fc, b_fc = weights
    ptrs = [_ptr(t).value for t in (rel_inv, filters, conv_bias, W_fc, b_fc) + tuple(masks)]
    return _lib.ConvENet(weights.h, filters.shape[0], *ptrs, *[float(k) for k in keeps])


def _conve_grads(tensors):
    return _lib.ConvEGrads(*[_ptr(t).value for t in tensors])


class _ConvEOneToNFn(torch.autograd.Function):
    """Returns (loss, reg) of rgcn_conve_one_to_n; the gradients of all seven tensors come from the forward with
    g_scale = (1, 0) and are finished by rgcn_conve_one_to_n_finish, as _OneToNFn does."""

    @staticmethod
    def forward(ctx, codes, rel, rel_inv, filters, conv_bias, W_fc, b_fc, labels, queries, smoothing, h, masks, keeps,
                R, chunk, grads):
        V, d = codes.shape
        dev = codes.device
        weights = ConvEWeights(rel_inv, filters, conv_bias, W_fc, b_fc, h)
        net = _conve_net(weights, masks, keeps)
        loss = torch.empty(2, dtype=torch.float32, device=dev)
        dcodes = torch.empty_like(codes) if grads else None
        drel = torch.empty_like(rel) if grads else None
        dnet = [torch.empty_like(t) for t in weights] if grads else None
        g_loss_only = torch.tensor([1.0, 0.0], dtype=torch.float32, device=dev) if grads else None
        _call("rgcn_conve_one_to_n", "rgcn_conve_one_to_n_workspace_bytes",
              (V, R, d, h, weights.C, len(queries), chunk),
              (_ptr(codes), _ptr(rel), V, rel.shape[0], R, d, ctypes.byref(net), _np_ptr(queries), len(queries),
               _ptr(labels), smoothing, _ptr(g_loss_only), _ptr(loss), _ptr(dcodes), _ptr(drel),
               ctypes.byref(_conve_grads(dnet)) if grads else None, chunk), dev)
        ctx.args = (queries, R, h, keeps)
        if grads:
            ctx.save_for_backward(codes, rel, *weights, dcodes, drel, *dnet)
        return loss[0], loss[1]

    @staticmethod
    def backward(ctx, g_loss, g_reg):
        saved = ctx.saved_tensors
        codes, rel = saved[0], saved[1]
        weights = ConvEWeights(*saved[2:7], h=ctx.args[2])
        dcodes_loss, drel_loss, dnet_loss = saved[7], saved[8], saved[9:14]
        queries, R, h, keeps = ctx.args
        V, d = codes.shape
        dev = codes.device
        gs = torch.zeros(2, dtype=torch.float32, device=dev)
        if g_loss is not None:
            gs[0] = g_loss
        if g_reg is not None:
            gs[1] = g_reg
        dcodes, drel = torch.empty_like(codes), torch.empty_like(rel)
        dnet = [torch.empty_like(t) for t in weights]
        net = _conve_net(weights)
        _call("rgcn_conve_one_to_n_finish", "rgcn_conve_one_to_n_finish_workspace_bytes", (len(queries),),
              (_ptr(codes), _ptr(rel), V, rel.shape[0], R, d, ctypes.byref(net), _np_ptr(queries), len(queries),
               _ptr(gs), _ptr(dcodes_loss), _ptr(drel_loss), ctypes.byref(_conve_grads(dnet_loss)), _ptr(dcodes),
               _ptr(drel), ctypes.byref(_conve_grads(dnet))), dev)
        return (dcodes, drel) + tuple(dnet) + (None,) * 9


def _check_conve_masks(masks, n, d, C):
    masks = tuple(masks) if masks is not None else (None, None, None)
    for name, m, width in zip(("input_mask", "feature_mask", "hidden_mask"), masks, (2 * d, C, d)):
        if m is not None and not (m.is_cuda and m.dtype == torch.uint8 and m.is_contiguous()
                                  and tuple(m.shape) == (n, width)):
            raise _lib.RgcnError("%s must be a contiguous CUDA uint8 [%d, %d] keep-mask" % (name, n, width))
    return masks


def conve_one_to_n_loss(codes, rel, weights, queries, labels, smoothing, masks=None, keeps=(1.0, 1.0, 1.0),
                        relation_count=None):
    """1-N loss of the ConvE decoder: ops.one_to_n_loss with the query rows of the ConvE network (weights a
    ConvEWeights), (anchor, r, 1) reading rel[r] and (anchor, r, 0) the reciprocal row rel_inv[r].  masks: None or the
    (input [n, 2d], feature [n, C], hidden [n, d]) uint8 keep-masks of the queries, each None for no dropout, scaled by
    1 / keeps.  Returns (loss, reg), reg the L2 term of the anchor row and the relation or reciprocal row.
    Differentiable in codes, rel and the five tensors of weights."""
    _check_cuda_f32("codes", codes)
    _check_cuda_f32("relation table", rel)
    V, d = codes.shape
    F = weights.check(d)
    R = rel.shape[0] if relation_count is None else int(relation_count)
    if weights[0].shape[0] != R:
        raise _lib.RgcnError("rel_inv must have one row per relation (%d)" % R)
    q = _check_queries(queries, V, R)
    words = (V + 31) // 32
    if not (labels.is_cuda and labels.dtype == torch.int32 and labels.is_contiguous()
            and tuple(labels.shape) == (len(q), words)):
        raise _lib.RgcnError("labels must be a contiguous CUDA int32 [n, ceil(V/32)] tensor (bit rows)")
    if not 0.0 <= float(smoothing) < 1.0:
        raise ValueError("conve_one_to_n_loss: label smoothing must be in [0, 1), got %r" % (smoothing,))
    masks = _check_conve_masks(masks, len(q), d, weights.C)
    Fp = (F + 3) // 4 * 4
    chunk = max(1, min(len(q), ONE_TO_N_CHUNK_BYTES // ((V + 6 * d + 3 * Fp) * 4)))
    tensors = (codes, rel) + tuple(weights)
    grads = torch.is_grad_enabled() and any(t.requires_grad for t in tensors)
    return _ConvEOneToNFn.apply(codes, rel, *weights, labels, q, float(smoothing), weights.h, masks,
                                tuple(float(k) for k in keeps), R, chunk, grads)


def conve_query_rows(codes, rel, weights, X, side, relation_count=None):
    """Test-mode ConvE query rows [n, d] of the triples X (int32 [n, 3] CUDA): side 1 f(codes[s], rel[r]), side 0
    f(codes[o], rel_inv[r]) (rgcn_conve_query_rows)."""
    _check_cuda_f32("codes", codes)
    _check_cuda_f32("relation table", rel)
    V, d = codes.shape
    weights.check(d)
    R = rel.shape[0] if relation_count is None else int(relation_count)
    if not (X.is_cuda and X.dtype == torch.int32 and X.is_contiguous() and X.dim() == 2 and X.shape[1] == 3):
        raise _lib.RgcnError("X must be a contiguous CUDA int32 [n,3] tensor")
    n = X.shape[0]
    Q = torch.empty((n, d), dtype=torch.float32, device=codes.device)
    net = _conve_net(weights)
    _call("rgcn_conve_query_rows", "rgcn_conve_query_rows_workspace_bytes", (d, weights.h, weights.C, n),
          (_ptr(codes), _ptr(rel), V, rel.shape[0], R, d, ctypes.byref(net), _ptr(X), n, int(side), _ptr(Q)),
          codes.device)
    return Q


class ConvERanker(object):
    """Fused all-entity ranking and top-k of the ConvE decoder (rgcn_conve_rank / rgcn_conve_topk): the interface and
    split reuse of DistMultRanker, the query rows from the ConvE network.  ConvE has no relation prediction (its
    energy is not linear in the relation row) and is no member of the fused ensemble (EnsembleRanker takes
    DistMultRanker objects only)."""
    TOPK_CHUNK_BYTES = DistMultRanker.TOPK_CHUNK_BYTES

    def __init__(self, codes, rel, weights, relation_count=None):
        _check_cuda_f32("codes", codes)
        _check_cuda_f32("relation table", rel)
        weights.check(codes.shape[1])
        self.codes, self.rel, self.weights = codes, rel, weights
        self.relation_count = rel.shape[0] if relation_count is None else int(relation_count)
        self._net = _conve_net(weights)
        self._ws, self._ws_n, self._split_ready = None, -1, False

    _check_rows = DistMultRanker._check_rows
    _chunk_rows = DistMultRanker._chunk_rows

    def top_k(self, X, side, k, exclude_mask=None):
        """As DistMultRanker.top_k, over the ConvE query rows."""
        lib = _lib.load()
        V, d = self.codes.shape
        h, C, R = self.weights.h, self.weights.C, self.relation_count
        self._check_rows(X, exclude_mask, "exclude_mask")
        k, n = int(k), X.shape[0]
        chunk, nb = self._chunk_rows(n, lambda m: lib.rgcn_conve_topk_workspace_bytes(V, d, h, C, m, k),
                                     "rgcn_conve_topk_workspace_bytes")
        dev = self.codes.device
        if self._ws is None or self._ws.numel() < nb:
            self._ws, self._ws_n, self._split_ready = _workspace(nb, dev), -1, False
        ids = torch.empty((n, k), dtype=torch.int32, device=dev)
        energies = torch.empty((n, k), dtype=torch.float32, device=dev)
        for c0 in range(0, max(n, 1), chunk):
            c1 = min(n, c0 + chunk)
            rc = lib.rgcn_conve_topk(_ptr(self.codes), _ptr(self.rel), V, self.rel.shape[0], R, d,
                                     ctypes.byref(self._net), _ptr(X[c0:c1]), c1 - c0, int(side), k,
                                     _ptr(None if exclude_mask is None else exclude_mask[c0:c1]),
                                     int(self._split_ready), _ptr(ids[c0:c1]), _ptr(energies[c0:c1]), _ptr(self._ws),
                                     self._ws.numel(), _stream(dev))
            _lib.check(rc, "rgcn_conve_topk")
            self._split_ready = True
        return ids, energies

    def rank(self, X, side, known_mask=None):
        """As DistMultRanker.rank, over the ConvE query rows."""
        lib = _lib.load()
        V, d = self.codes.shape
        h, C, R = self.weights.h, self.weights.C, self.relation_count
        self._check_rows(X, known_mask, "known_mask")
        n = X.shape[0]
        dev = self.codes.device
        if self._ws is None or n > self._ws_n:
            nb = lib.rgcn_conve_rank_workspace_bytes(V, d, h, C, n)
            if nb < 0:
                _lib.check(int(nb), "rgcn_conve_rank_workspace_bytes")
            self._ws, self._ws_n, self._split_ready = _workspace(nb, dev), n, False
        raw = torch.empty(n, dtype=torch.int32, device=dev)
        filt = torch.empty(n, dtype=torch.int32, device=dev) if known_mask is not None else None
        rc = lib.rgcn_conve_rank(_ptr(self.codes), _ptr(self.rel), V, self.rel.shape[0], R, d, ctypes.byref(self._net),
                                 _ptr(X), n, int(side), _ptr(known_mask), int(self._split_ready), _ptr(raw), _ptr(filt),
                                 _ptr(self._ws), self._ws.numel(), _stream(dev))
        _lib.check(rc, "rgcn_conve_rank")
        self._split_ready = True
        return raw, filt

    def rank_relations(self, X, known_mask=None):
        raise NotImplementedError("the ConvE decoder has no relation prediction")

    def top_k_relations(self, X, k, exclude_mask=None):
        raise NotImplementedError("the ConvE decoder has no relation prediction")
