"""1-D node sharding of the R-GCN layer across GPUs (SURVEY.md 8e), one process per GPU.

Rank p owns the contiguous node range [V*p/P, V*(p+1)/P): its rows of H / out / dH and every MESSAGE
whose destination it owns.  Sources are addressed in an extended local row space
[local rows | halo rows]; the halo rows (unique remote sources) arrive once per layer forward -- pushed
by their owners into this rank's peer-mapped halo buffer (PeerHalo), or by ONE all-to-all-v (NCCL
transport) -- and their gradients return the same way per layer backward (then a local row add).  Weights are replicated; their gradients are summed with one all-reduce.  The
per-message normalisation uses GLOBAL degrees, so sharded results equal the single-GPU ones.

The reference has no distributed code at all (single tf.Session, train.py:278); this module is the
multi-GPU design for the hot path only.
"""
import math
import os
import warnings

import numpy as np
import torch
import torch.distributed as dist

from . import ops


def node_bounds(n_nodes, world):
    return [(n_nodes * p) // world for p in range(world + 1)]


def owner_of(nodes, bounds):
    return np.searchsorted(np.asarray(bounds[1:]), nodes, side="right").astype(np.int32)


def global_messages(triples, n_nodes, n_relations, norm_mode="canonical", norm_f=None, norm_b=None):
    """The 2E messages with globally computed norms (same rules as rgcn_graph_create)."""
    t = np.asarray(triples, dtype=np.int32).reshape(-1, 3)
    s, r, o = t[:, 0], t[:, 1], t[:, 2]
    dst = np.concatenate([o, s]).astype(np.int32)
    src = np.concatenate([s, o]).astype(np.int32)
    relw = np.concatenate([r, r + n_relations]).astype(np.int32)
    if norm_mode == "canonical":
        cf = np.bincount(o, minlength=n_nodes).astype(np.float32)
        cb = np.bincount(s, minlength=n_nodes).astype(np.float32)
        norm = np.concatenate([np.float32(1) / cf[o], np.float32(1) / cb[s]]).astype(np.float32)
    elif norm_mode == "explicit":
        norm = np.concatenate([norm_f, norm_b]).astype(np.float32)
    else:
        norm = np.ones(dst.shape[0], np.float32)
    return dst, src, relw, norm


class ShardPlan(object):
    """Pure host-side partition description of one rank (testable without any GPU)."""

    def __init__(self, triples, n_nodes, n_relations, rank, world, norm_mode="canonical", norm_f=None,
                 norm_b=None):
        self.rank, self.world = rank, world
        self.n_nodes, self.n_relations = n_nodes, n_relations
        self.bounds = node_bounds(n_nodes, world)
        lo, hi = self.bounds[rank], self.bounds[rank + 1]
        self.lo, self.hi = lo, hi
        self.n_local = hi - lo
        dst, src, relw, norm = global_messages(triples, n_nodes, n_relations, norm_mode, norm_f, norm_b)
        odst = owner_of(dst, self.bounds)
        osrc = owner_of(src, self.bounds)
        mine = odst == rank
        src_g = src[mine]
        remote = osrc[mine] != rank
        # halo rows: unique remote sources, ascending global id (hence grouped by owner)
        self.halo_nodes = np.unique(src_g[remote]).astype(np.int32)
        self.n_halo = int(self.halo_nodes.shape[0])
        src_l = np.where(remote, self.n_local + np.searchsorted(self.halo_nodes, src_g), src_g - lo)
        self.msg_dst = (dst[mine] - lo).astype(np.int32)
        self.msg_src = src_l.astype(np.int32)
        self.msg_relw = relw[mine].astype(np.int32)
        self.msg_norm = norm[mine].astype(np.float32)
        self.msg_global_id = np.nonzero(mine)[0]
        halo_owner = owner_of(self.halo_nodes, self.bounds)
        self.recv_counts = np.bincount(halo_owner, minlength=world).astype(np.int64)
        # rows every peer needs from me = unique sources I own of messages whose destination it owns
        need = (osrc == rank) & (odst != rank)
        pairs = np.unique(np.stack([odst[need].astype(np.int64), src[need].astype(np.int64)], 1), axis=0) \
            if need.any() else np.zeros((0, 2), np.int64)
        self.send_counts = np.bincount(pairs[:, 0], minlength=world).astype(np.int64)
        self.send_rows = (pairs[:, 1] - lo).astype(np.int64)  # grouped by peer, ascending id inside


class ShardPlanDevice(object):
    """The same partition computed with torch ops ON THE DEVICE that holds the edge list (a CUDA tensor of triples):
    no per-rank pass of numpy over the global 2E-message list, so a 100 M-edge graph is planned in well under a
    second per rank and never visits the host.  Attributes mirror ShardPlan; the per-message / per-row arrays are
    device tensors (int32 / float32 / int64 for send_rows), the per-peer counts small host arrays.  Element for
    element identical to ShardPlan (tests/test_gpu_parallel.py compares them)."""

    def __init__(self, triples, n_nodes, n_relations, rank, world, norm_mode="canonical", norm_f=None, norm_b=None,
                 keep_global_ids=False):
        t = triples
        if not (isinstance(t, torch.Tensor) and t.dtype == torch.int32 and t.dim() == 2 and t.shape[1] == 3):
            raise ValueError("ShardPlanDevice: triples must be an int32 [E,3] tensor")
        dev = t.device
        self.rank, self.world = rank, world
        self.n_nodes, self.n_relations = n_nodes, n_relations
        self.bounds = node_bounds(n_nodes, world)
        lo, hi = self.bounds[rank], self.bounds[rank + 1]
        self.lo, self.hi, self.n_local = lo, hi, hi - lo
        E = t.shape[0]
        s, r, o = t[:, 0], t[:, 1], t[:, 2]
        if norm_mode == "canonical":
            cf = torch.bincount(o.long(), minlength=n_nodes).to(torch.float32)
            cb = torch.bincount(s.long(), minlength=n_nodes).to(torch.float32)
            one = torch.ones((), dtype=torch.float32, device=dev)
            inv_f, inv_b = one / cf, one / cb      # fp32 division, as in ShardPlan / rgcn_graph_create
        inner = torch.as_tensor(self.bounds[1:], dtype=torch.int32, device=dev)

        def owner(nodes):
            return torch.bucketize(nodes.contiguous(), inner, out_int32=True, right=True)

        parts = {k: [] for k in ("dst", "src", "relw", "norm", "gid")}
        need_keys = []
        # forward messages (dst = o, src = s, weight id r), then backward (dst = s, src = o, weight id r + R):
        # the global message order of ShardPlan, handled per direction to keep the temporaries at E elements
        for direction, (dn, sn) in enumerate(((o, s), (s, o))):
            od, os_ = owner(dn), owner(sn)
            mine = (od == rank).nonzero(as_tuple=True)[0]
            parts["dst"].append((dn[mine] - lo).to(torch.int32))
            parts["src"].append(sn[mine])
            parts["relw"].append((r[mine] + direction * n_relations).to(torch.int32))
            if norm_mode == "canonical":
                parts["norm"].append((inv_f if direction == 0 else inv_b)[dn[mine].long()])
            elif norm_mode == "explicit":
                parts["norm"].append((norm_f if direction == 0 else norm_b)[mine].to(torch.float32))
            else:
                parts["norm"].append(torch.ones(mine.shape[0], dtype=torch.float32, device=dev))
            if keep_global_ids:
                parts["gid"].append(mine + direction * E)
            need = ((os_ == rank) & (od != rank)).nonzero(as_tuple=True)[0]
            need_keys.append(od[need].long() * n_nodes + sn[need].long())
            del od, os_, mine, need
        self.msg_dst = torch.cat(parts["dst"])
        src_g = torch.cat(parts["src"])
        self.msg_relw = torch.cat(parts["relw"])
        self.msg_norm = torch.cat(parts["norm"])
        self.msg_global_id = torch.cat(parts["gid"]) if keep_global_ids else None
        del parts
        remote = (src_g < lo) | (src_g >= hi)
        self.halo_nodes = torch.unique(src_g[remote])          # ascending global id, hence grouped by owner
        self.n_halo = int(self.halo_nodes.shape[0])
        pos = torch.searchsorted(self.halo_nodes, src_g, out_int32=True) if self.n_halo else torch.zeros_like(src_g)
        self.msg_src = torch.where(remote, pos + self.n_local, src_g - lo).to(torch.int32)
        del src_g, remote, pos
        self.recv_counts = torch.bincount(owner(self.halo_nodes).long(), minlength=world).cpu().numpy().astype(np.int64)
        keys = torch.unique(torch.cat(need_keys))               # (peer, source) pairs, sorted by peer then id
        del need_keys
        self.send_counts = torch.bincount(torch.div(keys, n_nodes, rounding_mode="floor"),
                                          minlength=world).cpu().numpy().astype(np.int64)
        self.send_rows = (keys % n_nodes) - lo                  # int64, grouped by peer, ascending id inside


def all_ranks_agree(ok, group, device):
    """True on every rank iff `ok` is true on every rank (one MIN all-reduce): ranks must take the same branch before
    any collective setup step, or the ones that went ahead wait forever for the one that did not."""
    flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=device)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
    return bool(int(flag.item()) == 1)


class PeerHalo(object):
    """Peer-mapped (CUDA symmetric memory) buffers for the halo exchange of ONE layer call in flight.

    Every rank owns `halo` [max n_halo, d] -- the rows its aggregation kernels gather from -- and `back` [max rows
    sent, d] -- the gradients of the rows it sent -- allocated symmetrically and mapped into every peer.  The forward
    exchange is then rgcn_rows_gather writing each peer's rows from H straight into that peer's `halo` over NVLink
    (no packed send buffer, no all-to-all), the backward return is one peer-to-peer copy per owner into its `back`
    (the halo gradients are already grouped by owner), and three stream-ordered cross-GPU barriers per layer step
    replace the collectives: buffers free -> rows landed -> gradients landed."""

    def __init__(self, sg, d):
        import torch.distributed._symmetric_memory as symm
        p = sg.plan
        dev = sg.device
        group = sg.group if sg.group is not None else dist.group.WORLD
        me, P = p.rank, p.world
        mine = torch.tensor([p.n_halo, int(np.sum(p.send_counts))] + [int(x) for x in sg.halo_off[:P]] +
                            [int(x) for x in sg.send_off[:P]], dtype=torch.int64, device=dev)
        table = [torch.empty_like(mine) for _ in range(P)]
        dist.all_gather(table, mine, group=group)
        table = torch.stack(table).cpu().numpy()
        self.halo_rows = max(int(table[:, 0].max()), 1)
        self.back_rows = max(int(table[:, 1].max()), 1)
        # where MY rows start inside peer q's halo buffer / where my gradients for q's rows start in q's back buffer
        self.peer_halo_off = [int(table[q, 2 + me]) for q in range(P)]
        self.peer_back_off = [int(table[q, 2 + P + me]) for q in range(P)]
        self.d = int(d)
        with warnings.catch_warnings():   # needed by torch <= 2.8, a deprecated no-op afterwards
            warnings.simplefilter("ignore")
            try:
                symm.enable_symm_mem_for_group(group.group_name)
            except Exception:
                pass
        # The symmetric allocation bypasses torch's caching allocator: hand cached blocks back first, then let every
        # rank check that the buffers fit (with 2 GB to spare) and AGREE on it -- a rank that ran out of memory alone
        # would leave its peers waiting in the rendezvous.
        need = (self.halo_rows + self.back_rows) * self.d * 4
        torch.cuda.empty_cache()
        free = torch.cuda.mem_get_info(dev)[0]
        if not all_ranks_agree(free >= need + (2 << 30), group, dev):
            raise RuntimeError("not enough free device memory on some rank for %.1f GB of peer-mapped halo buffers"
                               % (need / 1e9))
        self.buf = symm.empty((self.halo_rows + self.back_rows, self.d), dtype=torch.float32, device=dev)
        self.hdl = symm.rendezvous(self.buf, group)
        self.halo = self.buf[:self.halo_rows]
        self.back = self.buf[self.halo_rows:]
        self.busy = False

    def peer_halo_ptr(self, q):
        return int(self.hdl.buffer_ptrs[q]) + self.peer_halo_off[q] * self.d * 4

    def peer_back_view(self, q, n):
        return self.hdl.get_buffer(q, (n, self.d), torch.float32, (self.halo_rows + self.peer_back_off[q]) * self.d)

    def barrier(self):
        self.hdl.barrier(channel=0)


def _unpack_add(dH, sg, back):
    """dH[send_rows] += back.  `back` is grouped by peer and a peer's rows are unique, so on the GPU each peer segment is
    one non-atomic row-add kernel (rgcn_rows_add); elsewhere (CPU tests) torch's index_add_."""
    if dH.is_cuda and back.dtype == torch.float32:
        for q in range(len(sg.send_off) - 1):
            a, b = sg.send_off[q], sg.send_off[q + 1]
            if b > a:
                ops.rows_add_(dH, sg.send_rows[a:b], back[a:b])
    else:
        dH.index_add_(0, sg.send_rows, back)
    return dH


class _HaloExchange(torch.autograd.Function):
    """H_local [n_local,d] -> H_ext [n_local+n_halo,d]; backward returns halo gradients to their owners."""

    @staticmethod
    def forward(ctx, H_local, plan, send_rows, group):
        d = H_local.shape[1]
        H_ext = torch.empty(plan.n_local + plan.n_halo, d, dtype=H_local.dtype, device=H_local.device)
        H_ext[:plan.n_local].copy_(H_local)
        send = H_local.index_select(0, send_rows)
        dist.all_to_all_single(H_ext[plan.n_local:], send, output_split_sizes=plan.recv_counts.tolist(),
                               input_split_sizes=plan.send_counts.tolist(), group=group)
        ctx.plan, ctx.group = plan, group
        ctx.save_for_backward(send_rows)
        return H_ext

    @staticmethod
    def backward(ctx, dH_ext):
        plan = ctx.plan
        (send_rows,) = ctx.saved_tensors
        dH_ext = dH_ext.contiguous()
        back = torch.empty(int(plan.send_counts.sum()), dH_ext.shape[1], dtype=dH_ext.dtype,
                           device=dH_ext.device)
        dist.all_to_all_single(back, dH_ext[plan.n_local:].contiguous(),
                               output_split_sizes=plan.send_counts.tolist(),
                               input_split_sizes=plan.recv_counts.tolist(), group=ctx.group)
        dH = dH_ext[:plan.n_local].clone()
        dH.index_add_(0, send_rows, back)
        return dH, None, None, None


class _OverlappedBlockLayer(torch.autograd.Function):
    """Sharded block layer with the halo exchange hidden behind the local work.

    forward : start the halo exchange || self-loop GEMM + LOCAL-source messages (rgcn_block_forward on the local
              graph, ReLU deferred) -> wait -> HALO-source messages (rgcn_block_aggregate) -> ReLU
    backward: G = dOut * relu'(out) -> halo-source backward first (rgcn_block_aggregate_backward) -> start the
              gradient return || local backward (rgcn_block_backward) -> wait -> add the returned rows.
    Exchange = peer transport (PeerHalo: rgcn_rows_gather pushes my rows into the peers' mapped halo buffers, the
    gradients return by one peer-to-peer copy per owner, stream-ordered cross-GPU barriers) or, when that is not
    available / not wanted, NCCL all-to-all-v of packed rows in both directions."""

    @staticmethod
    def forward(ctx, H_local, Wf, Wb, Ws, sg, n_blocks, drop_mask, keep, relu):
        p = sg.plan
        d = H_local.shape[1]
        dev = H_local.device
        H_local = H_local.contiguous()
        slot = sg.peer_slot(d) if H_local.dtype == torch.float32 else None
        if slot is not None:   # push my rows straight into the peers' halo buffers (rgcn_rows_gather over NVLink)
            main, side = torch.cuda.current_stream(dev), sg.side_stream
            side.wait_stream(main)
            with torch.cuda.stream(side):
                slot.barrier()                               # every rank is done with the buffers' previous contents
                for k in range(1, p.world):                  # ring order: every receiver hears from one sender at a time
                    q = (p.rank + k) % p.world
                    a, b = sg.send_off[q], sg.send_off[q + 1]
                    if b > a:
                        ops.rows_gather_to(slot.peer_halo_ptr(q), H_local, sg.send_rows[a:b], sg.push_ctas)
                slot.barrier()                               # every peer's rows have landed in my halo buffer
            H_halo = slot.halo[:p.n_halo]
            slot.busy = any(ctx.needs_input_grad)             # held until backward returns
            work = None
        else:
            send = H_local.index_select(0, sg.send_rows)
            H_halo = torch.empty(p.n_halo, d, dtype=H_local.dtype, device=dev)
            work = dist.all_to_all_single(H_halo, send, output_split_sizes=p.recv_counts.tolist(),
                                          input_split_sizes=p.send_counts.tolist(), group=sg.group, async_op=True)
        with torch.no_grad():
            out = ops._BlockLayerFn.apply(H_local, Wf, Wb, Ws, sg.graph_local, n_blocks, drop_mask, keep, False)
        if work is not None:
            work.wait()
        else:
            torch.cuda.current_stream(dev).wait_stream(sg.side_stream)
        if p.n_halo > 0:  # a rank whose messages all have local sources has no halo graph work at all
            ops.block_aggregate_(out, H_halo, Wf, Wb, sg.graph_halo, n_blocks)
        if relu:
            out.relu_()
        ctx.sg, ctx.n_blocks, ctx.keep, ctx.relu, ctx.mask = sg, n_blocks, keep, relu, drop_mask
        ctx.slot = slot
        ctx.save_for_backward(H_local, Wf, Wb, Ws, H_halo, out)
        return out

    @staticmethod
    def backward(ctx, dOut):
        H_local, Wf, Wb, Ws, H_halo, out = ctx.saved_tensors
        sg, B = ctx.sg, ctx.n_blocks
        p = sg.plan
        slot = ctx.slot
        if ctx.relu and dOut.is_cuda and dOut.dtype == torch.float32 and dOut.numel() % 4 == 0:
            G = ops.relu_backward(dOut, out)       # one pass (torch: compare + multiply, 35 GB instead of 30)
        else:
            G = ((dOut * (out > 0)) if ctx.relu else dOut).contiguous()
        if p.n_halo > 0:
            dHalo, dWf, dWb = ops.block_aggregate_backward(H_halo, Wf, Wb, G, sg.graph_halo, B)
        else:  # empty halo: nothing to send back, no halo contribution to the block weight gradients
            dHalo = torch.empty(0, G.shape[1], dtype=G.dtype, device=G.device)
            dWf, dWb = torch.zeros_like(Wf), torch.zeros_like(Wb)
        if slot is not None:   # the halo gradients are grouped by owner: one peer-to-peer copy per owner, into its `back`
            main, side = torch.cuda.current_stream(G.device), sg.side_stream
            side.wait_stream(main)
            dHalo.record_stream(side)
            with torch.cuda.stream(side):
                for k in range(1, p.world):
                    q = (p.rank - k) % p.world
                    a, b = sg.halo_off[q], sg.halo_off[q + 1]
                    if b > a:
                        slot.peer_back_view(q, b - a).copy_(dHalo[a:b])
                slot.barrier()                               # every peer's gradients for my rows have landed
            back = slot.back[:int(np.sum(p.send_counts))]
            work = None
        else:
            back = torch.empty(int(p.send_counts.sum()), G.shape[1], dtype=G.dtype, device=G.device)
            work = dist.all_to_all_single(back, dHalo, output_split_sizes=p.send_counts.tolist(),
                                          input_split_sizes=p.recv_counts.tolist(), group=sg.group, async_op=True)
        d = H_local.shape[1]
        dH = torch.empty_like(H_local)
        dWf_l, dWb_l, dWs = torch.empty_like(Wf), torch.empty_like(Wb), torch.empty_like(Ws)
        h = sg.graph_local.handle
        ops._call("rgcn_block_backward", "rgcn_block_workspace_bytes", (h, d, B, 1),
                  (h, d, B, ops._ptr(H_local), ops._ptr(Wf), ops._ptr(Wb), ops._ptr(Ws), ops._ptr(ctx.mask),
                   float(ctx.keep), 0, ops._ptr(out), ops._ptr(G), ops._ptr(dH), ops._ptr(dWf_l), ops._ptr(dWb_l),
                   ops._ptr(dWs)), G.device)
        dWf += dWf_l
        dWb += dWb_l
        if work is not None:
            work.wait()
        else:
            torch.cuda.current_stream(G.device).wait_stream(sg.side_stream)
        _unpack_add(dH, sg, back)
        if slot is not None:
            slot.busy = False   # the next forward's first barrier orders every rank after this unpack
        return dH, dWf, dWb, dWs, None, None, None, None, None


def _post(ops_list):
    return dist.batch_isend_irecv(ops_list) if ops_list else []


def ring_post_forward(sg, send_all, H_halo):
    """Post the P-1 ring steps of the halo exchange (step k: send my rows to rank me+k, receive the rows
    of rank me-k).  Returns one list of Work handles per step; step k's rows are usable after waiting
    on works[k-1], so the consumer can process peer me-1's rows while peer me-2's are still in flight."""
    p = sg.plan
    me, P = p.rank, p.world
    works = []
    for k in range(1, P):
        st, rf = (me + k) % P, (me - k) % P
        ops_k = []
        if p.send_counts[st]:
            ops_k.append(dist.P2POp(dist.isend, send_all[sg.send_off[st]:sg.send_off[st + 1]], st, sg.group))
        if p.recv_counts[rf]:
            ops_k.append(dist.P2POp(dist.irecv, H_halo[sg.halo_off[rf]:sg.halo_off[rf + 1]], rf, sg.group))
        works.append(_post(ops_k))
    return works


def ring_post_backward_step(sg, k, dX_from_rf, back):
    """Backward ring step k: return the gradient of the rows received from rank me-k to their owner and
    receive, from rank me+k, the gradient of the rows sent to it."""
    p = sg.plan
    me, P = p.rank, p.world
    st, rf = (me + k) % P, (me - k) % P
    ops_k = []
    if p.recv_counts[rf]:
        ops_k.append(dist.P2POp(dist.isend, dX_from_rf, rf, sg.group))
    if p.send_counts[st]:
        ops_k.append(dist.P2POp(dist.irecv, back[sg.send_off[st]:sg.send_off[st + 1]], st, sg.group))
    return _post(ops_k)


class _PipelinedBlockLayer(torch.autograd.Function):
    """Sharded block layer with a PIPELINED ring halo exchange: the rows of every peer are a separate
    transfer and a separate message sub-graph, so peer q's messages are aggregated while peer q+1's rows
    are still crossing NVLink (forward), and every peer's halo gradients leave as soon as they are
    computed while the next peer's are being computed (backward)."""

    @staticmethod
    def forward(ctx, H_local, Wf, Wb, Ws, sg, n_blocks, drop_mask, keep, relu):
        p = sg.plan
        me, P = p.rank, p.world
        d = H_local.shape[1]
        H_local = H_local.contiguous()
        send_all = H_local.index_select(0, sg.send_rows)
        H_halo = torch.empty(p.n_halo, d, dtype=H_local.dtype, device=H_local.device)
        works = ring_post_forward(sg, send_all, H_halo)
        with torch.no_grad():
            out = ops._BlockLayerFn.apply(H_local, Wf, Wb, Ws, sg.graph_local, n_blocks, drop_mask, keep, False)
        for k in range(1, P):
            for w in works[k - 1]:
                w.wait()
            rf = (me - k) % P
            if p.recv_counts[rf]:
                ops.block_aggregate_(out, H_halo[sg.halo_off[rf]:sg.halo_off[rf + 1]], Wf, Wb,
                                     sg.graph_halo_peer[rf], n_blocks)
        if relu:
            out.relu_()
        ctx.sg, ctx.n_blocks, ctx.keep, ctx.relu, ctx.mask = sg, n_blocks, keep, relu, drop_mask
        ctx.keep_alive = send_all
        ctx.save_for_backward(H_local, Wf, Wb, Ws, H_halo, out)
        return out

    @staticmethod
    def backward(ctx, dOut):
        H_local, Wf, Wb, Ws, H_halo, out = ctx.saved_tensors
        sg, B = ctx.sg, ctx.n_blocks
        p = sg.plan
        me, P = p.rank, p.world
        G = ((dOut * (out > 0)) if ctx.relu else dOut).contiguous()
        d = G.shape[1]
        back = torch.empty(int(p.send_counts.sum()), d, dtype=G.dtype, device=G.device)
        works, alive = [], []
        dWf = dWb = None
        for k in range(1, P):
            rf = (me - k) % P
            dX = None
            if p.recv_counts[rf]:
                dX, dWf, dWb = ops.block_aggregate_backward(H_halo[sg.halo_off[rf]:sg.halo_off[rf + 1]], Wf, Wb, G,
                                                            sg.graph_halo_peer[rf], B, dWf, dWb)
                alive.append(dX)
            works.append(ring_post_backward_step(sg, k, dX, back))
        dH = torch.empty_like(H_local)
        dWf_l, dWb_l, dWs = torch.empty_like(Wf), torch.empty_like(Wb), torch.empty_like(Ws)
        h = sg.graph_local.handle
        ops._call("rgcn_block_backward", "rgcn_block_workspace_bytes", (h, d, B, 1),
                  (h, d, B, ops._ptr(H_local), ops._ptr(Wf), ops._ptr(Wb), ops._ptr(Ws), ops._ptr(ctx.mask),
                   float(ctx.keep), 0, ops._ptr(out), ops._ptr(G), ops._ptr(dH), ops._ptr(dWf_l), ops._ptr(dWb_l),
                   ops._ptr(dWs)), G.device)
        if dWf is not None:
            dWf_l += dWf
            dWb_l += dWb
        for wk in works:
            for w in wk:
                w.wait()
        _unpack_add(dH, sg, back)
        return dH, dWf_l, dWb_l, dWs, None, None, None, None, None


class ShardedGraph(object):
    def __init__(self, triples, n_nodes, n_relations, rank, world, device, norm_mode="canonical",
                 norm_f=None, norm_b=None, group=None, overlap=True, pipelined=None, transport=None):
        """transport (overlapped block layers on CUDA, world > 1): "peer" = halo rows pushed into peer-mapped buffers by
        rgcn_rows_gather (PeerHalo), "nccl" = packed rows + all-to-all; None = $RGCN_HALO_TRANSPORT, else "peer" with
        "nccl" taking over (one warning) when symmetric memory cannot be set up on this system."""
        self.device = torch.device(device)
        self.transport = transport or os.environ.get("RGCN_HALO_TRANSPORT") or "auto"
        if self.transport not in ("auto", "peer", "nccl"):
            raise ValueError("transport must be 'peer', 'nccl' or None")
        self._peer_slots, self._peer_failed = [], False
        self.side_stream = None
        self.push_ctas = int(os.environ.get("RGCN_PUSH_CTAS", "64"))
        on_device = isinstance(triples, torch.Tensor) and triples.is_cuda
        if on_device:   # edge list already on the GPU: plan + graph preparation never leave it
            self.plan = ShardPlanDevice(triples, n_nodes, n_relations, rank, world, norm_mode, norm_f, norm_b)
        else:
            self.plan = ShardPlan(triples, n_nodes, n_relations, rank, world, norm_mode, norm_f, norm_b)
        self.group = group
        p = self.plan
        self.n_local, self.n_halo = p.n_local, p.n_halo
        index = None
        if self.device.type == "cuda":
            index = self.device.index if self.device.index is not None else torch.cuda.current_device()

        def make_graph(dst, src, relw, norm, v_dst, v_src):
            if on_device:
                return ops.Graph.from_device_messages(dst.contiguous(), src.contiguous(), relw.contiguous(),
                                                      norm.contiguous(), v_dst, v_src, 2 * n_relations)
            return ops.Graph.from_messages(dst, src, relw, norm, v_dst, v_src, 2 * n_relations, device=index)

        self.graph = None
        if not (overlap and world > 1) or not on_device:   # the un-split graph (basis layers, non-overlapped path)
            self.graph = make_graph(p.msg_dst, p.msg_src, p.msg_relw, p.msg_norm, p.n_local, p.n_local + p.n_halo)
        self.send_rows = torch.as_tensor(p.send_rows, device=self.device)
        self.send_off = np.concatenate([[0], np.cumsum(p.send_counts)]).astype(np.int64).tolist()
        self.halo_off = np.concatenate([[0], np.cumsum(p.recv_counts)]).astype(np.int64).tolist()
        # split by source locality so the halo exchange can overlap the local-source work
        self.overlap = overlap and world > 1
        # per-peer ring pipeline: opt-in.  P-1 small sub-graph launches and NCCL groups per direction can cost
        # more than the exposed transfer they hide, so the single overlapped all-to-all is the default.
        self.pipelined = self.overlap and bool(pipelined)
        if self.overlap:
            loc = p.msg_src < p.n_local
            self.graph_local = make_graph(p.msg_dst[loc], p.msg_src[loc], p.msg_relw[loc], p.msg_norm[loc],
                                          p.n_local, p.n_local)
            rem = ~loc
            self.graph_halo = make_graph(p.msg_dst[rem], p.msg_src[rem] - p.n_local, p.msg_relw[rem],
                                         p.msg_norm[rem], p.n_local, max(p.n_halo, 0))
            self.graph_halo_peer = {}
            if self.pipelined:
                hsrc = p.msg_src - p.n_local  # halo-row index of every remote-source message
                for q in range(world):
                    lo_q, hi_q = self.halo_off[q], self.halo_off[q + 1]
                    if q == rank or hi_q == lo_q:
                        continue
                    sel = rem & (hsrc >= lo_q) & (hsrc < hi_q)
                    self.graph_halo_peer[q] = make_graph(p.msg_dst[sel], hsrc[sel] - lo_q, p.msg_relw[sel],
                                                         p.msg_norm[sel], p.n_local, hi_q - lo_q)
            if on_device:   # the plan's per-message arrays are no longer needed: free the device memory
                p.msg_dst = p.msg_src = p.msg_relw = p.msg_norm = None

    def peer_slot(self, d):
        """A free PeerHalo of width d (created collectively on first use: every rank runs the same layer sequence), or
        None when the NCCL transport is in force."""
        if self.transport == "nccl" or self._peer_failed or self.device.type != "cuda" or self.plan.world < 2:
            return None
        for slot in self._peer_slots:
            if slot.d == d and not slot.busy:
                return slot
        if len(self._peer_slots) >= 4:   # forwards whose backward never ran hold their slots: do not grow without bound
            return None
        try:
            slot = PeerHalo(self, d)
        except Exception as e:   # symmetric memory unavailable (no P2P mapping between these GPUs, old driver, ...)
            if self.transport == "peer":
                raise
            warnings.warn("peer-mapped halo buffers unavailable (%s: %s); using the NCCL all-to-all transport"
                          % (type(e).__name__, e))
            self._peer_failed = True
            return None
        if self.side_stream is None:
            self.side_stream = torch.cuda.Stream(device=self.device)
        self._peer_slots.append(slot)
        return slot

    def halo_transport(self):
        """Transport the overlapped block layer used so far: "peer", "nccl", or None before the first call."""
        if self._peer_slots:
            return "peer"
        return "nccl" if (self._peer_failed or self.transport == "nccl") else None

    def halo_exchange(self, H_local):
        return _HaloExchange.apply(H_local, self.plan, self.send_rows, self.group)

    def block_layer(self, H_local, W_forward, W_backward, W_self, n_blocks, drop_mask=None, keep=1.0,
                    relu=True):
        if self.pipelined and self.device.type == "cuda":
            return _PipelinedBlockLayer.apply(H_local, W_forward, W_backward, W_self, self, int(n_blocks),
                                              drop_mask, keep, relu)
        if self.overlap and self.device.type == "cuda":
            return _OverlappedBlockLayer.apply(H_local, W_forward, W_backward, W_self, self, int(n_blocks),
                                               drop_mask, keep, relu)
        return ops.block_layer(self.halo_exchange(H_local), W_forward, W_backward, W_self, self.graph,
                               n_blocks, drop_mask, keep, relu)

    def basis_layer(self, H_local, W_forward, W_backward, C_forward, C_backward, W_self, drop_mask=None,
                    keep=1.0, relu=True):
        if self.graph is None:
            raise ValueError("this ShardedGraph was planned on the device for the overlapped block path only "
                             "(pass overlap=False to also build the un-split graph the basis layer walks)")
        return ops.basis_layer(self.halo_exchange(H_local), W_forward, W_backward, C_forward, C_backward,
                               W_self, self.graph, drop_mask, keep, relu)

    def allreduce_weight_grads(self, weights):
        """One all-reduce(sum) over the replicated weights' gradients (flattened into one bucket)."""
        grads = [w.grad for w in weights if w.grad is not None]
        if not grads:
            return
        flat = torch.cat([g.reshape(-1) for g in grads])
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=self.group)
        off = 0
        for g in grads:
            n = g.numel()
            g.copy_(flat[off:off + n].view_as(g))
            off += n



# ------------------------------------------------------------------------------------------------------------
# Feature-sharded message passing (block-diagonal layers only; EXPERIMENTAL, opt-in -- DESIGN.md section 7)
# ------------------------------------------------------------------------------------------------------------
def block_bounds(n_blocks, block_size, world):
    """Contiguous block ranges per rank.  Blocks are dealt in groups of 4/gcd(s,4) so that every rank's column
    count is a multiple of 4 floats (the kernels move rows as float4 quads)."""
    g = 4 // math.gcd(int(block_size), 4)
    if n_blocks % g != 0:
        raise ValueError("feature sharding needs NumberOfBasisFunctions to be a multiple of %d for block size %d"
                         % (g, block_size))
    groups = n_blocks // g
    if groups < world:
        raise ValueError("feature sharding: only %d column groups for %d ranks" % (groups, world))
    return [((groups * p) // world) * g for p in range(world + 1)]


class _FeatureShardedBlockLayer(torch.autograd.Function):
    """Block layer with the MESSAGE part computed feature-parallel and the self loop node-parallel.

    Block-diagonal weights never mix features of different blocks, so a rank that holds the columns of its own
    blocks for ALL nodes can aggregate every message of the graph without any neighbour exchange:

      forward : all-to-all transpose H_local [n_local, d] -> Hf [V, d_q]   ||  S = dropout(H_local @ W_self)
                Af = rgcn_block_aggregate(Hf, W[:, blocks_q])  on the FULL graph           [V, d_q]
                all-to-all transpose back -> columns of out;  out = act(S + messages)
      backward: G = dOut * act'  ->  transpose  ||  self-loop gradients (two local GEMMs)
                rgcn_block_aggregate_backward -> dHf, dW[:, blocks_q]  ->  transpose back, dH += .

    Traffic per GPU and direction: 2 transposes of V*d*4/N bytes, independent of the graph's locality."""

    @staticmethod
    def forward(ctx, H_local, Wf, Wb, Ws, fs, drop_mask, keep, relu):
        H_local = H_local.contiguous()
        work, Hf = fs.to_feature_async(H_local)
        S = H_local @ Ws
        if drop_mask is not None:
            S = S * drop_mask.to(S.dtype) / keep
        work.wait()
        b0, b1 = fs.blocks
        Wf_q, Wb_q = Wf[:, b0:b1].contiguous(), Wb[:, b0:b1].contiguous()
        Af = torch.zeros(fs.n_nodes, fs.d_local, dtype=H_local.dtype, device=H_local.device)
        ops.block_aggregate_(Af, Hf, Wf_q, Wb_q, fs.graph, b1 - b0)
        out = fs.to_node_add(Af, S)
        if relu:
            out = torch.relu_(out)
        ctx.fs, ctx.keep, ctx.relu = fs, keep, relu
        ctx.save_for_backward(H_local, Wf_q, Wb_q, Ws, Hf, out, drop_mask if drop_mask is not None
                              else torch.empty(0, device=H_local.device))
        ctx.full_shapes = (Wf.shape, Wb.shape)
        return out

    @staticmethod
    def backward(ctx, dOut):
        H_local, Wf_q, Wb_q, Ws, Hf, out, mask = ctx.saved_tensors
        fs = ctx.fs
        G = (dOut * (out > 0)) if ctx.relu else dOut
        G = G.contiguous()
        work, Gf = fs.to_feature_async(G)
        Gs = G if mask.numel() == 0 else G * mask.to(G.dtype) / ctx.keep
        dWs = H_local.t() @ Gs
        dH = Gs @ Ws.t()
        work.wait()
        b0, b1 = fs.blocks
        dHf, dWf_q, dWb_q = ops.block_aggregate_backward(Hf, Wf_q, Wb_q, Gf, fs.graph, b1 - b0)
        dH = fs.to_node_add(dHf, dH)
        # the other ranks' blocks get zeros here; allreduce_weight_grads (sum) assembles the full tables
        dWf = torch.zeros(ctx.full_shapes[0], dtype=dWf_q.dtype, device=dWf_q.device)
        dWb = torch.zeros(ctx.full_shapes[1], dtype=dWb_q.dtype, device=dWb_q.device)
        dWf[:, b0:b1] = dWf_q
        dWb[:, b0:b1] = dWb_q
        return dH, dWf, dWb, dWs, None, None, None, None


class FeatureShardedGraph(object):
    """Replicated graph structure, features sharded by BLOCK for the message part, by node for everything else
    (inputs, outputs and the self loop stay in the 1-D node shard's layout, so it is a drop-in for ShardedGraph
    in block layers).  See _FeatureShardedBlockLayer."""

    def __init__(self, triples, n_nodes, n_relations, rank, world, device, n_blocks, block_size,
                 norm_mode="canonical", norm_f=None, norm_b=None, group=None):
        self.rank, self.world, self.group = int(rank), int(world), group
        self.device = torch.device(device)
        self.n_nodes = int(n_nodes)
        self.node_bounds = node_bounds(n_nodes, world)
        self.lo, self.hi = self.node_bounds[rank], self.node_bounds[rank + 1]
        self.n_local, self.n_halo, self.overlap, self.pipelined = self.hi - self.lo, 0, False, False
        self.block_size = int(block_size)
        self.block_bounds = block_bounds(n_blocks, block_size, world)
        self.blocks = (self.block_bounds[rank], self.block_bounds[rank + 1])
        self.col_bounds = [b * self.block_size for b in self.block_bounds]
        self.d = self.col_bounds[-1]
        self.d_local = self.col_bounds[rank + 1] - self.col_bounds[rank]
        index = None
        if self.device.type == "cuda":
            index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.graph = ops.Graph(triples, n_nodes, n_relations, norm_mode=norm_mode, norm_f=norm_f, norm_b=norm_b,
                               device=index)
        rows = [self.node_bounds[p + 1] - self.node_bounds[p] for p in range(world)]
        cols = [self.col_bounds[q + 1] - self.col_bounds[q] for q in range(world)]
        # node -> feature: I send my rows' columns of rank q to q; I receive every rank's rows of MY columns
        self._nf_send = [self.n_local * c for c in cols]
        self._nf_recv = [r * self.d_local for r in rows]
        self._cols = cols

    # [n_local, d] -> [V, d_local]
    def to_feature_async(self, X_local):
        send = torch.cat([X_local[:, self.col_bounds[q]:self.col_bounds[q + 1]].reshape(-1)
                          for q in range(self.world)])
        recv = torch.empty(self.n_nodes * self.d_local, dtype=X_local.dtype, device=X_local.device)
        work = dist.all_to_all_single(recv, send, output_split_sizes=self._nf_recv,
                                      input_split_sizes=self._nf_send, group=self.group, async_op=True)
        return work, recv.view(self.n_nodes, self.d_local)

    # [V, d_local] -> added into the columns of a [n_local, d] base (the adjoint of to_feature)
    def to_node_add(self, Xf, base):
        recv = torch.empty(self.n_local * self.d, dtype=Xf.dtype, device=Xf.device)
        dist.all_to_all_single(recv, Xf.contiguous().view(-1), output_split_sizes=self._nf_send,
                               input_split_sizes=self._nf_recv, group=self.group)
        out = base if base.is_contiguous() else base.contiguous()
        off = 0
        for q in range(self.world):
            n = self.n_local * self._cols[q]
            out[:, self.col_bounds[q]:self.col_bounds[q + 1]] += recv[off:off + n].view(self.n_local, self._cols[q])
            off += n
        return out

    def block_layer(self, H_local, W_forward, W_backward, W_self, n_blocks, drop_mask=None, keep=1.0,
                    relu=True):
        if int(n_blocks) != self.block_bounds[-1] or W_forward.shape[2] != self.block_size:
            raise ValueError("FeatureShardedGraph was planned for %d blocks of size %d"
                             % (self.block_bounds[-1], self.block_size))
        return _FeatureShardedBlockLayer.apply(H_local, W_forward, W_backward, W_self, self, drop_mask, keep, relu)

    def basis_layer(self, *args, **kwargs):
        raise NotImplementedError("basis weights are dense in the feature dimension: use the node shard")

    allreduce_weight_grads = ShardedGraph.allreduce_weight_grads
