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
         "none": _lib.RGCN_NORM_NONE}


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


def _triple_forward(ctx, entry, codes, rel, X, Y):
    """Forward of a triple scorer entry point with the distmult_forward argument list."""
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
    rc = getattr(lib, entry)(_ptr(codes), _ptr(rel), V, rel.shape[0], d, _ptr(X), N, _ptr(Y),
                             _ptr(energies), _ptr(loss2), _stream(dev))
    _lib.check(rc, entry)
    ctx.has_y = Y is not None
    ctx.rel_param = rel
    ctx.save_for_backward(codes, rel, X, Y if Y is not None else torch.empty(0, device=dev),
                          energies)
    return energies, loss2[0], loss2[1]


def _triple_backward(ctx, entry, g_energy, g_loss, g_reg):
    """Backward of a triple scorer entry point with the distmult_backward_slices argument list."""
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
                             _ptr(Y), _ptr(energies), 1.0, 1.0, _ptr(gs), _ptr(ge),
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
                                           lambda m: lib.rgcn_relation_rank_workspace_bytes(R, d, m)):
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
                                           lambda m: lib.rgcn_relation_topk_workspace_bytes(R, d, m, k)):
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
