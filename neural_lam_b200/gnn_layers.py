"""InteractionNet / PropagationNet / SplitMLPs with the reference's Python interface
(reference neural_lam/gnn_layers.py: InteractionNet :14-189, PropagationNet :192-249,
GNN_TYPES / get_gnn_class :252-271, SplitMLPs :274-324), backed by libnlam_b200.so.

Drop-in surface kept (SURVEY.md section 8b): constructor and ``forward`` signatures, return
type depending on ``update_edges``, 2-D ``(N,H)`` or 3-D ``(B,N,H)`` inputs (stride-0 batch
expansions are consumed without materialising), attributes ``edge_index`` (senders offset by
``num_rec``, non-persistent buffer), ``num_rec``, ``aggr``, ``update_edges``, ``edge_mlp``,
``aggr_mlp``, ``propagate(edge_index, x=, edge_attr=) -> (aggr, messages)``, state_dict
keys/shapes, full autograd.  CPU tensors raise (no CPU fallback).
"""
import torch
from torch import nn

from . import _lib, backward, ops
from .networks import _aten_forward, make_mlp

_DEFAULT_MATH = "auto"
_MATH_FLAGS = {"auto": 0, "tf32": _lib.MATH_TF32, "fp32": _lib.MATH_FP32}


def set_default_math(mode):
    """``"auto"`` (wgmma TF32 kernels where the shape is supported, exact fp32 kernels
    otherwise), ``"tf32"`` (require the tensor-core kernels) or ``"fp32"`` (exact FFMA)."""
    global _DEFAULT_MATH
    if mode not in _MATH_FLAGS:
        raise ValueError(f"unknown math mode {mode!r}")
    _DEFAULT_MATH = mode


def get_default_math():
    return _DEFAULT_MATH


class SplitMLPs(nn.Module):
    """Feeds chunks of the input (split along dim -2 by ``chunk_sizes``) through separate
    MLPs and concatenates the results (reference gnn_layers.py:274-324)."""

    def __init__(self, mlps, chunk_sizes):
        super().__init__()
        assert len(mlps) == len(chunk_sizes), "Number of MLPs must match the number of chunks"
        self.mlps = nn.ModuleList(mlps)
        self.chunk_sizes = chunk_sizes

    def forward(self, x):
        parts = torch.split(x, self.chunk_sizes, dim=-2)
        return torch.cat([m(c) for m, c in zip(self.mlps, parts)], dim=-2)


def _mlp_chunks(mod, n_rows):
    """[(make_mlp Sequential, row0, row1)] for a plain MLP or a SplitMLPs."""
    if isinstance(mod, SplitMLPs):
        out, r = [], 0
        for m, n in zip(mod.mlps, mod.chunk_sizes):
            out.append((m, r, r + n))
            r += n
        if r != n_rows:
            raise ValueError(f"chunk sizes sum to {r}, expected {n_rows}")
        return out
    return [(mod, 0, n_rows)]


def _aten_apply(mod, names, params, prefix, x):
    """Differentiable evaluation of edge_mlp/aggr_mlp (plain or SplitMLPs) with explicit params."""
    table = {n[len(prefix):]: p for n, p in zip(names, params) if n.startswith(prefix)}
    if isinstance(mod, SplitMLPs):
        parts = torch.split(x, mod.chunk_sizes, dim=-2)
        outs = []
        for k, (m, c) in enumerate(zip(mod.mlps, parts)):
            sub = {n[len(f"mlps.{k}."):]: p for n, p in table.items() if n.startswith(f"mlps.{k}.")}
            outs.append(_aten_forward(m, sub, c))
        return torch.cat(outs, dim=-2)
    return _aten_forward(mod, table, x)


class InteractionNet(nn.Module):
    """Interaction network (Battaglia et al. 2016) message-passing layer:
    ``m_e = edge_mlp([e, x_sender, x_receiver])``; ``aggr_r = sum|mean_{e->r} m_e``;
    ``rec' = rec + aggr_mlp([rec, aggr])``; ``e' = e + m`` — computed by fused sm_90a kernels.
    """

    propagation = False
    # node-partitioned rollout (dist.partition_model): callable mapping this rank's OWN sender rows (B, n_own, H) to
    # the extended rows [own | halo] the layer's local edge_index refers to
    _halo = None

    def __init__(self, edge_index, input_dim, update_edges=True, hidden_layers=1, hidden_dim=None,
                 edge_chunk_sizes=None, aggr_chunk_sizes=None, aggr="sum", math=None):
        if aggr not in ("sum", "mean"):
            raise ValueError(f"Unknown aggregation method: {aggr}")
        super().__init__()
        self.aggr = aggr
        if hidden_dim is None:
            hidden_dim = input_dim
        if hidden_dim != input_dim:
            raise ValueError("neural_lam_b200.InteractionNet: hidden_dim must equal input_dim "
                             "(the residual connections require it; every reference call site uses it)")
        self.input_dim = input_dim
        self.hidden_layers = hidden_layers
        self.math = math

        ei = edge_index.detach().to(torch.int64)
        if ei.dim() != 2 or ei.shape[0] != 2 or ei.shape[1] < 1:
            raise ValueError(f"edge_index must have shape (2, E>=1), got {tuple(ei.shape)}")
        self.num_rec = int(ei[1].max()) + 1
        # reference convention: receivers [0,num_rec), senders offset by num_rec (gnn_layers.py:73-86)
        self.register_buffer("edge_index", torch.stack((ei[0] + self.num_rec, ei[1]), dim=0), persistent=False)

        # int32 index tables (original edge order) used by the composed / backward paths
        cpu = ei.cpu()
        snd, rcv = cpu[0], cpu[1]
        E = cpu.shape[1]
        perm = torch.sort(rcv, stable=True).indices
        inv_perm = torch.empty_like(perm)
        inv_perm[perm] = torch.arange(E)
        rowptr = torch.zeros(self.num_rec + 1, dtype=torch.int64)
        rowptr[1:] = torch.cumsum(torch.bincount(rcv, minlength=self.num_rec), 0)
        self.num_send_min = int(snd.max()) + 1
        sorder = torch.sort(snd, stable=True).indices
        sptr = torch.zeros(self.num_send_min + 1, dtype=torch.int64)
        sptr[1:] = torch.cumsum(torch.bincount(snd, minlength=self.num_send_min), 0)
        dev = edge_index.device
        for name, t in (("_src32", snd), ("_dst32", rcv), ("_perm32", perm), ("_inv_perm32", inv_perm),
                        ("_rowptr32", rowptr), ("_sorder32", sorder), ("_sptr32", sptr)):
            self.register_buffer(name, t.to(torch.int32).contiguous().to(dev), persistent=False)
        self._is_sorted = bool(torch.equal(perm, torch.arange(E)))
        self.max_in_degree = int((rowptr[1:] - rowptr[:-1]).max())
        self._graphs = {}

        edge_recipe = [3 * input_dim] + [hidden_dim] * (hidden_layers + 1)
        aggr_recipe = [2 * input_dim] + [hidden_dim] * (hidden_layers + 1)
        if edge_chunk_sizes is None:
            self.edge_mlp = make_mlp(edge_recipe)
        else:
            self.edge_mlp = SplitMLPs([make_mlp(edge_recipe) for _ in edge_chunk_sizes], edge_chunk_sizes)
        if aggr_chunk_sizes is None:
            self.aggr_mlp = make_mlp(aggr_recipe)
        else:
            self.aggr_mlp = SplitMLPs([make_mlp(aggr_recipe) for _ in aggr_chunk_sizes], aggr_chunk_sizes)
        self.update_edges = update_edges

    # graph handles (ctypes pointers into the library) are per-process device resources: copies and pickles of
    # the module drop them and rebuild lazily (copy.deepcopy for EMA / SWA, torch.save of whole modules)
    def __getstate__(self):
        state = self.__dict__.copy()
        state["_graphs"] = {}
        return state

    def __deepcopy__(self, memo):
        import copy

        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            new.__dict__[k] = {} if k == "_graphs" else copy.deepcopy(v, memo)
        return new

    # ------------------------------------------------------------------ helpers
    @property
    def num_edges(self):
        return self.edge_index.shape[1]

    def _flags(self):
        mode = self.math or _DEFAULT_MATH
        f = _MATH_FLAGS[mode]
        if self.aggr == "mean":
            f |= _lib.AGGR_MEAN
        if self.propagation:
            f |= _lib.PROPAGATION
        return f

    def _math_only_flags(self):
        return _MATH_FLAGS[self.math or _DEFAULT_MATH]

    def _graph(self, device):
        key = device.index if device.index is not None else torch.cuda.current_device()
        g = self._graphs.get(key)
        if g is None:
            ei = self.edge_index.detach().cpu()
            g = ops.Graph(torch.stack((ei[0] - self.num_rec, ei[1])), torch.device("cuda", key), self.num_rec)
            self._graphs[key] = g
        return g

    def _check_inputs(self, send_rep, rec_rep, edge_rep):
        for name, t in (("send_rep", send_rep), ("rec_rep", rec_rep), ("edge_rep", edge_rep)):
            if not isinstance(t, torch.Tensor):
                raise TypeError(f"{name} must be a tensor")
            if not t.is_cuda:
                raise RuntimeError(
                    f"neural_lam_b200.{type(self).__name__}: {name} is on {t.device}; this layer runs on "
                    "CUDA tensors only — there is no CPU fallback")
            if t.dtype != torch.float32:
                raise TypeError(f"{name}: float32 expected, got {t.dtype}")
            if t.dim() not in (2, 3) or t.shape[-1] != self.input_dim:
                raise ValueError(f"{name}: expected (..., N, {self.input_dim}), got {tuple(t.shape)}")
        if rec_rep.shape[-2] != self.num_rec:
            raise ValueError(f"rec_rep has {rec_rep.shape[-2]} rows, layer has num_rec={self.num_rec}")
        if send_rep.shape[-2] < self.num_send_min:
            raise ValueError(f"send_rep has {send_rep.shape[-2]} rows but edge_index references sender "
                             f"{self.num_send_min - 1}")
        if edge_rep.shape[-2] != self.num_edges:
            raise ValueError(f"edge_rep has {edge_rep.shape[-2]} rows, layer has {self.num_edges} edges")
        if self._src32.device != rec_rep.device:
            raise RuntimeError("module buffers and inputs are on different devices; call .to(device)")

    def _param_list(self):
        named = list(self.named_parameters())
        return [n for n, _ in named], [p for _, p in named]

    # ------------------------------------------------------ kernel paths (no autograd)
    def _fusable(self):
        return not isinstance(self.edge_mlp, SplitMLPs) and not isinstance(self.aggr_mlp, SplitMLPs)

    def _kernel_messages(self, send, rec, edge):
        """Messages in ORIGINAL edge order + aggregate, composed from the row-MLP and
        segment-sum kernels (used for SplitMLPs layers and ``propagate``)."""
        fl = self._math_only_flags()  # SplitMLPs chunks: gather-pack + the generic wgmma Linear kernel (or exact fp32)
        idx = [None, self._src32, self._dst32]
        outs = []
        for m, r0, r1 in _mlp_chunks(self.edge_mlp, self.num_edges):
            outs.append(ops.rowmlp(m, [edge, send, rec], res=send if self.propagation else None,
                                   res_idx=self._src32 if self.propagation else None, flags=fl,
                                   idx=idx, row_range=(r0, r1)))
        msg = outs[0] if len(outs) == 1 else torch.cat(outs, dim=-2)
        mean = self.aggr == "mean" or self.propagation
        aggr = ops.segment_sum(msg, self._rowptr32, self._perm32, mean=mean)
        return aggr, msg

    def _kernel_node_update(self, rec, aggr):
        fl = self._math_only_flags()
        base = aggr if self.propagation else rec
        outs = []
        for m, r0, r1 in _mlp_chunks(self.aggr_mlp, self.num_rec):
            outs.append(ops.rowmlp(m, [rec, aggr], res=base, flags=fl, row_range=(r0, r1)))
        return outs[0] if len(outs) == 1 else torch.cat(outs, dim=-2)

    def _kernel_forward(self, send, rec, edge):
        """(rec_out, edge_out) via libnlam_b200 for 3-D inputs of equal batch size."""
        if self._fusable():
            g = self._graph(rec.device)
            e_csr = edge if self._is_sorted else ops.gather_rows(edge, self._perm32)
            rec_out, edge_out, _ = ops.inet_fwd(g, self.edge_mlp, self.aggr_mlp, send, rec, e_csr,
                                                self.update_edges, self._flags())
            if edge_out is not None and not self._is_sorted:
                edge_out = ops.gather_rows(edge_out, self._inv_perm32)
        else:
            aggr, msg = self._kernel_messages(send, rec, edge)
            rec_out = self._kernel_node_update(rec, aggr)
            edge_out = (edge + msg) if self.update_edges else None
        return rec_out, edge_out

    # ------------------------------------------------------ differentiable restatement
    def _torch_messages(self, names, params, send, rec, edge):
        """Same math as the kernels as a differentiable graph (3-D inputs, equal batch)."""
        x_j = ops.GatherRowsFn.apply(send, self._src32, self._sptr32, self._sorder32)
        x_i = ops.GatherRowsFn.apply(rec, self._dst32, self._rowptr32, self._perm32)
        msg = _aten_apply(self.edge_mlp, names, params, "edge_mlp.", torch.cat((edge, x_j, x_i), dim=-1))
        if self.propagation:
            msg = x_j + msg
        mean = self.aggr == "mean" or self.propagation
        aggr = ops.SegmentSumFn.apply(msg.contiguous(), self._rowptr32, self._perm32, self._dst32, mean)
        return aggr, msg

    def _torch_forward(self, names, params, send, rec, edge):
        aggr, msg = self._torch_messages(names, params, send, rec, edge)
        diff = _aten_apply(self.aggr_mlp, names, params, "aggr_mlp.", torch.cat((rec, aggr), dim=-1))
        rec_out = (aggr if self.propagation else rec) + diff
        if self.update_edges:
            return rec_out, edge + msg
        return (rec_out,)

    @staticmethod
    def _batchify(*tensors):
        """Lift (N,H) inputs to (1,N,H) and expand (stride 0) to a common batch size."""
        three_d = any(t.dim() == 3 for t in tensors)
        ts = [t if t.dim() == 3 else t.unsqueeze(0) for t in tensors]
        B = max(t.shape[0] for t in ts)
        for t in ts:
            if t.shape[0] not in (1, B):
                raise ValueError("inconsistent batch sizes")
        ts = [t if t.shape[0] == B else t.expand(B, -1, -1) for t in ts]
        return three_d, ts

    # ------------------------------------------------------------------ public API
    def forward(self, send_rep, rec_rep, edge_rep):
        """Update receiver (and optionally edge) representations.

        send_rep ``(…, num_send, H)``, rec_rep ``(…, num_rec, H)``, edge_rep ``(…, E, H)`` ->
        rec_rep' or ``(rec_rep', edge_rep')`` when ``update_edges``."""
        if self._halo is not None:  # node-partitioned rollout: own sender rows -> [own | halo]
            send_rep = self._halo(send_rep if send_rep.dim() == 3 else send_rep.unsqueeze(0))
            if rec_rep.dim() == 2:
                send_rep = send_rep[0]
        self._check_inputs(send_rep, rec_rep, edge_rep)
        names, params = self._param_list()
        three_d, (s3, r3, e3) = self._batchify(send_rep, rec_rep, edge_rep)

        def kernel_fn(s, r, e, *_p):
            ro, eo = self._kernel_forward(s, r, e)
            return (ro, eo) if self.update_edges else (ro,)

        def torch_fn(s, r, e, *p):
            return self._torch_forward(names, p, s, r, e)

        bwd_fn = None
        if _MATH_FLAGS[self.math or _DEFAULT_MATH] != _lib.MATH_FP32 and backward.inet_supported(self, s3, r3, e3):
            # TF32 modes: the backward runs on the library's kernels too (backward.py); "fp32" keeps the exact ATen recompute
            def bwd_fn(saved, gouts, needs=None):
                s, r, e = saved[:3]
                g = self._graph(r.device)
                e_csr = e if self._is_sorted else ops.gather_rows(e, self._perm32)
                g_rec = gouts[0] if gouts[0] is not None else torch.zeros_like(r)
                g_eo = gouts[1] if (self.update_edges and len(gouts) > 1 and gouts[1] is not None) else None
                if g_eo is not None and not self._is_sorted:
                    g_eo = ops.gather_rows(g_eo.contiguous(), self._perm32)
                g_s, g_r, g_e, pg = backward.inet_backward(self, g, s, r, e_csr, g_rec.contiguous(), g_eo)
                if g_s.shape[1] != s.shape[1]:  # sender rows no edge references
                    pad = torch.zeros((g_s.shape[0], s.shape[1], g_s.shape[2]), device=g_s.device, dtype=g_s.dtype)
                    pad[:, : g_s.shape[1]] = g_s
                    g_s = pad
                if not self._is_sorted:
                    g_e = ops.gather_rows(g_e, self._inv_perm32)
                return (g_s, g_r, g_e, *[pg[n] for n in names])

        outs = ops.run_with_recompute(kernel_fn, torch_fn, [s3, r3, e3, *params], bwd_fn=bwd_fn)
        if not three_d:
            outs = [o[0] for o in outs]
        if self.update_edges:
            return outs[0], outs[1]
        return outs[0]

    def _stackable(self):
        return self._halo is None and self.update_edges and self._fusable() and self._is_sorted and not self.propagation

    @torch.no_grad()
    def forward_stacked(self, node_rep, edge_rep, first, last, proj_in=None, next_layer=None, keep_edges=False):
        """Inference-only entry for a layer inside a stack over ONE node set whose intermediate edge tensors are
        private to the stack (``GNNSequential`` with ``keep_edge_rep=False``): the last layer does not write its
        edge output (nobody reads it), a middle layer may update ``edge_rep`` in place (``first``: the incoming
        tensor belongs to the caller — e.g. the cached static embedding — and is never written).  ``keep_edges``: the last
        layer writes its edge output too, in place like a middle layer unless it is also the first.  Same values as
        ``forward``.  ``proj_in``: this layer's node projections, computed by the previous layer's node kernel;
        ``next_layer``: the following layer of the stack — when the library supports it for both, this call's node kernel
        also computes that layer's projections (csrc/fused.cu).  Returns ``(node_rep', edge_rep' | None, proj_next | None)``."""
        if self._halo is not None or not (self.update_edges and self._fusable() and self._is_sorted):
            assert proj_in is None
            return (*self.forward(node_rep, node_rep, edge_rep), None)
        self._check_inputs(node_rep, node_rep, edge_rep)
        _, (s3, r3, e3) = self._batchify(node_rep, node_rep, edge_rep)
        g = self._graph(r3.device)
        write_edges = keep_edges or not last
        # in place where the library supports the call shape (nlam_inet_inplace_supported), else out of place
        inplace = (not first) and write_edges and e3.is_contiguous()
        nxt = None
        if (next_layer is not None and isinstance(next_layer, InteractionNet) and next_layer._stackable()
                and self._stackable() and next_layer.num_rec == self.num_rec and r3.shape[0] > 0):
            fl = self._flags()
            if (ops.inet_chain_supported(g, self.edge_mlp, self.aggr_mlp, next_layer.edge_mlp, r3, fl)
                    and ops.inet_chain_supported(next_layer._graph(r3.device), next_layer.edge_mlp, next_layer.aggr_mlp, None, r3,
                                                 next_layer._flags())):
                nxt = next_layer.edge_mlp
        if proj_in is None and nxt is None:
            rec_out, edge_out, _ = ops.inet_fwd(g, self.edge_mlp, self.aggr_mlp, s3, r3, e3, write_edges, self._flags(),
                                                edge_inplace=inplace)
            return rec_out, edge_out, None
        rec_out, edge_out, _, proj_out = ops.inet_fwd(g, self.edge_mlp, self.aggr_mlp, s3, r3, e3, write_edges, self._flags(),
                                                      edge_inplace=inplace, proj_in=proj_in, next_edge_seq=nxt)
        return rec_out, edge_out, proj_out

    def _edge_stage_separable(self):
        """Can the edge stage of this layer run without its node update, so that a later kernel consumes the aggregate
        (``aggregate_only``, ``decode_step``)?  Needs an InteractionNet without edge update or halo, in CSR edge order,
        with H = 64 single-block MLPs."""
        return not (self._halo is not None or self.update_edges or self.propagation or not self._fusable()
                    or not self._is_sorted or self.edge_mlp[0].in_features != 192)

    @torch.no_grad()
    def decode_step(self, send_rep, rec_rep, edge_rep, out_seq, prev, boundary, bmask, diff_std, diff_mean, out_flags=0,
                    out=None, std_out=None):
        """Inference-only: this layer (the mesh->grid decoder) chained with ``out_seq`` and the forecast-step epilogue in two
        launches (``ops.decode_step``); neither the aggregate nor the updated receiver rows go to HBM.  Returns the new state,
        or None when the layer / graph / call shape has no such path (the caller then runs ``aggregate_only``).  ``std_out``:
        the predicted-std form of ``ops.decode_step``."""
        if not self._edge_stage_separable() or (out_flags & _lib.MATH_FP32):
            return None
        self._check_inputs(send_rep, rec_rep, edge_rep)
        _, (s3, r3, e3) = self._batchify(send_rep, rec_rep, edge_rep)
        return ops.decode_step(self._graph(r3.device), self.edge_mlp, self.aggr_mlp, out_seq, s3, r3, e3, prev, boundary, bmask,
                               diff_std, diff_mean, flags=self._flags() | out_flags, out=out, std_out=std_out)

    @torch.no_grad()
    def encode_step(self, embedder, grid_mlp, grid_inputs, rec_rep, edge_rep, want_grid_emb=False, second=None):
        """Inference-only, for the grid -> mesh layer of a forecast step: ``grid_emb = embedder(cat grid_inputs)``, this layer's
        node projections and ``grid_rep = grid_emb + grid_mlp(grid_emb)`` in one launch (``ops.encode``), then this layer's
        edge stage on those projections and its node update.  ``second``: another grid -> mesh layer on the same graph,
        receivers and edge features, with grid_emb as its senders (the hierarchical Graph-EFM's decoder g2m): the launch also
        computes its projections.  ``want_grid_emb``: the launch also stores grid_emb (Graph-EFM's decoder reads it; not with
        ``second``).  Returns ``(grid_rep, [rec_rep' of this layer (, of second)], grid_emb | None)``, or None when the layer /
        graph / call shape has no such path (the caller then runs the embedder, the layers and grid_mlp as separate calls)."""
        layers = [self] if second is None else [self, second]
        if not all(layer._edge_stage_separable() for layer in layers) or (second is not None and not self._same_edges(second)):
            return None
        _, (r3, e3) = self._batchify(rec_rep, edge_rep)
        if r3.shape[-2] != self.num_rec or e3.shape[-2] != self.num_edges or r3.device != self._src32.device:
            return None
        fl = embedder.nlam_flags | grid_mlp.nlam_flags
        for layer in layers:
            fl |= layer._flags()
        enc = ops.encode(self._graph(r3.device), embedder, grid_inputs, grid_mlp, self.edge_mlp, r3, e3, flags=fl,
                         want_emb=want_grid_emb, edge_seq_b=second.edge_mlp if second is not None else None)
        if enc is None:
            return None
        grid_rep, projs, grid_emb = enc
        B, G = grid_rep.shape[0], grid_rep.shape[1]
        outs = [ops.inet_fwd(layer._graph(r3.device), layer.edge_mlp, layer.aggr_mlp, proj[: B * G * 64].view(B, G, 64),
                             r3.expand(B, -1, -1), e3.expand(B, -1, -1), False, layer._flags(), proj_in=proj)[0]
                for layer, proj in zip(layers, projs)]
        return grid_rep, outs, grid_emb

    def _same_edges(self, other):
        """Does ``other`` have this layer's edge set?  Compared once per pair (outside any CUDA-graph capture: the first
        no-grad step runs eagerly)."""
        memo = self.__dict__.setdefault("_same_edges_memo", {})
        key = (id(other), other.edge_index.data_ptr(), self.edge_index.data_ptr())
        if key not in memo:
            memo[key] = (other.num_rec == self.num_rec and other.num_edges == self.num_edges
                         and torch.equal(other.edge_index.cpu(), self.edge_index.cpu()))
        return memo[key]

    @torch.no_grad()
    def aggregate_only(self, send_rep, rec_rep, edge_rep):
        """Inference-only: the edge stage of the layer (messages + aggregation) WITHOUT the node update; returns the (B, Nr, H)
        aggregate, or None when this layer / call shape has no such kernel path (the caller then runs ``forward``).  Used to
        chain the node update of the mesh->grid layer with the output MLP in one kernel (``ops.node_update_step``)."""
        if not self._edge_stage_separable():
            return None
        self._check_inputs(send_rep, rec_rep, edge_rep)
        _, (s3, r3, e3) = self._batchify(send_rep, rec_rep, edge_rep)
        try:
            _, _, aggr = ops.inet_fwd(self._graph(r3.device), self.edge_mlp, self.aggr_mlp, s3, r3, e3, False, self._flags(),
                                      edge_only=True)
        except _lib.NlamError:
            return None
        return aggr

    def propagate(self, edge_index, x=None, edge_attr=None, size=None):
        """PyG-style entry kept for API compatibility (reference tests call it directly,
        tests/test_gnn_layers.py:249,:290,:380): ``x`` is ``cat(rec_rep, send_rep)`` along the
        node dim, returns ``(aggregated, messages)`` in the layer's edge order."""
        if edge_index is not self.edge_index and not torch.equal(edge_index, self.edge_index):
            raise ValueError("propagate: only the layer's own edge_index is supported")
        rec = x[..., : self.num_rec, :]
        send = x[..., self.num_rec:, :]
        self._check_inputs(send, rec, edge_attr)
        names, params = self._param_list()
        three_d, (s3, r3, e3) = self._batchify(send, rec, edge_attr)

        def kernel_fn(s, r, e, *_p):
            return self._kernel_messages(s, r, e)

        def torch_fn(s, r, e, *p):
            return self._torch_messages(names, p, s, r, e)

        aggr, msg = ops.run_with_recompute(kernel_fn, torch_fn, [s3, r3, e3, *params])
        if not three_d:
            aggr, msg = aggr[0], msg[0]
        return aggr, msg

    def node_residual_target(self, rec_rep, edge_rep_aggr):
        """Base tensor of the node residual connection (reference gnn_layers.py:159-166)."""
        return rec_rep

    def extra_repr(self):
        return (f"E={self.num_edges}, num_rec={self.num_rec}, H={self.input_dim}, aggr={self.aggr}, "
                f"update_edges={self.update_edges}, math={self.math or _DEFAULT_MATH}")


class PropagationNet(InteractionNet):
    """InteractionNet variant that propagates sender information: mean aggregation is
    forced, messages are ``x_j + edge_mlp(...)`` and the node residual targets the aggregate
    (reference gnn_layers.py:192-249)."""

    propagation = True

    def __init__(self, edge_index, input_dim, update_edges=True, hidden_layers=1, hidden_dim=None,
                 edge_chunk_sizes=None, aggr_chunk_sizes=None, aggr="sum", math=None):
        super().__init__(edge_index, input_dim, update_edges=update_edges, hidden_layers=hidden_layers,
                         hidden_dim=hidden_dim, edge_chunk_sizes=edge_chunk_sizes,
                         aggr_chunk_sizes=aggr_chunk_sizes, aggr="mean", math=math)

    def node_residual_target(self, rec_rep, edge_rep_aggr):
        return edge_rep_aggr


GNN_TYPES = {
    "InteractionNet": InteractionNet,
    "PropagationNet": PropagationNet,
}


def get_gnn_class(gnn_type):
    """Look up a GNN class by name (reference gnn_layers.py:258-271)."""
    if gnn_type not in GNN_TYPES:
        raise ValueError(f"Unknown GNN type '{gnn_type}'. Available types: {list(GNN_TYPES.keys())}")
    return GNN_TYPES[gnn_type]
