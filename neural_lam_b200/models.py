"""Graph step predictors (GraphLAM / HiLAM) and the autoregressive forecaster with the
reference's structure, parameter names and forward semantics, running on the sm_90a kernels.

Reference files mirrored (neural_lam/models/...):
  step_predictors/base.py        StepPredictor: expand_to_batch :122-139, clamped update :335-396
  step_predictors/graph/base.py  BaseGraphModel.__init__ :31-178, forward :228-344
  step_predictors/graph/graph_lam.py     GraphLAM :28-126, process_step :157-188
  step_predictors/graph/hierarchical.py  BaseHiGraphModel :30-151, process_step :186-292
  step_predictors/graph/hi_lam.py        HiLAM :114-165, mesh_down_step :167-236,
                                         mesh_up_step :238-307, hi_processor_step :309-376
  forecasters/autoregressive.py  ARForecaster.forward :63-149

Differences that do not change results: the datastore argument is any object exposing the
few quantities the predictors read (``synthetic.SyntheticDatastore``; the xarray/zarr stack
is out of scope), the graph comes in as a dict of tensors (``synthetic.make_graph_spec`` /
``synthetic.load_graph``) instead of being read from ``datastore.root_path``, every edge set
is kept receiver-sorted, and input-independent embeddings are cached between steps while the
weights do not change (SURVEY.md section 8f item 1).
"""
import ctypes

import torch
from torch import nn

from . import _lib, ensemble, ops
from .gnn_layers import InteractionNet, get_gnn_class
from . import clamping
from .latent import (ConstantLatentEncoder, GraphLatentDecoder, GraphLatentEncoder, HiGraphLatentDecoder,
                     HiGraphLatentEncoder)
from .clamping import OutputClamp
from .networks import GNNSequential, make_mlp
from .synthetic import normalize_graph


def _sort_edges(edge_index, features):
    """Receiver-sort one edge set (stable), permuting its static features alike."""
    order = torch.sort(edge_index[1], stable=True).indices
    if torch.equal(order, torch.arange(order.numel())):
        return edge_index, features
    return edge_index[:, order], features[order]


class BufferList(nn.Module):
    """List of non-persistent buffers (reference neural_lam/utils/buffer_list.py:11)."""

    def __init__(self, tensors):
        super().__init__()
        self.n = len(tensors)
        for i, t in enumerate(tensors):
            self.register_buffer(f"b{i}", t, persistent=False)

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [getattr(self, f"b{k}") for k in range(self.n)[i]]
        if i < 0:
            i += self.n
        return getattr(self, f"b{i}")

    def __len__(self):
        return self.n

    def __iter__(self):
        return (getattr(self, f"b{i}") for i in range(self.n))


class StepPredictor(nn.Module):
    """One-step predictor ``(X_{t-1}, X_t, forcing_t) -> X_{t+1}`` (reference
    models/step_predictors/base.py)."""

    def __init__(self, datastore, output_std=False, output_clamping_lower=None, output_clamping_upper=None):
        super().__init__()
        self.register_buffer("grid_static_features", datastore.grid_static_features.float(), persistent=False)
        self.num_grid_nodes = self.grid_static_features.shape[0]
        self.num_state_vars = datastore.num_state_vars
        self.output_std = bool(output_std)
        self.grid_output_dim = 2 * self.num_state_vars if self.output_std else self.num_state_vars
        # output clamping (reference step_predictors/base.py:56-61, :181-334): {state variable name: physical limit}.
        # As in the reference (``prepare_clamping_params``, :279-301) the seven limit / index buffers are PERSISTENT
        # buffers of the predictor itself — empty when no limits are configured — so its checkpoints load strictly.
        clamp = OutputClamp(list(datastore.state_var_names), output_clamping_lower, output_clamping_upper,
                            datastore.state_mean, datastore.state_std)
        for name in clamping.BUFFER_NAMES:
            self.register_buffer(name, getattr(clamp, name))
        # per-variable form for the fused kernel (nlam_step_epilogue_clamped): kind 0 none / 1 sigmoid / 2 lower / 3 upper
        d = self.num_state_vars
        kind, lo, up = torch.zeros(d, dtype=torch.int32), torch.zeros(d), torch.zeros(d)
        kind[clamp.clamp_lower_upper_idx], lo[clamp.clamp_lower_upper_idx], up[clamp.clamp_lower_upper_idx] = (
            1, clamp.sigmoid_lower_lims, clamp.sigmoid_upper_lims)
        kind[clamp.clamp_lower_idx], lo[clamp.clamp_lower_idx] = 2, clamp.softplus_lower_lims
        kind[clamp.clamp_upper_idx], up[clamp.clamp_upper_idx] = 3, clamp.softplus_upper_lims
        for name, t in (("_clamp_kind", kind), ("_clamp_lo", lo), ("_clamp_up", up)):
            self.register_buffer(name, t, persistent=False)

    @property
    def predicts_std(self):
        return self.output_std

    def expand_to_batch(self, x, batch_size):
        """(N,d) -> (B,N,d) stride-0 view (reference step_predictors/base.py:122-139)."""
        return x.unsqueeze(0).expand(batch_size, -1, -1)

    @property
    def clamps_output(self):
        return clamping.clamp_active(self)

    def get_clamped_new_state(self, state_delta, prev_state):
        """``X_{t+1} = f(f^-1(X_t) + delta)`` for the variables with configured limits, the plain residual update for
        the others (reference step_predictors/base.py:335-396); with no limits the index lists are empty."""
        if self.clamps_output:
            return clamping.clamped_update(self, state_delta, prev_state)
        return prev_state + state_delta


class BaseGraphModel(StepPredictor):
    """Encode (g2m) - process (subclass) - decode (m2g) graph model."""

    def __init__(self, datastore, graph, hidden_dim=64, hidden_layers=1, processor_layers=4, mesh_aggr="sum",
                 output_std=False, g2m_gnn_type="InteractionNet", m2g_gnn_type="InteractionNet", math=None,
                 output_clamping_lower=None, output_clamping_upper=None, **_unused):
        super().__init__(datastore, output_std=output_std, output_clamping_lower=output_clamping_lower,
                         output_clamping_upper=output_clamping_upper)
        self.g2m_gnn_type, self.m2g_gnn_type = g2m_gnn_type, m2g_gnn_type
        self.register_buffer("diff_mean", datastore.state_diff_mean.float(), persistent=False)
        self.register_buffer("diff_std", datastore.state_diff_std.float(), persistent=False)
        self.hidden_dim, self.hidden_layers = hidden_dim, hidden_layers
        self.processor_layers, self.mesh_aggr = processor_layers, mesh_aggr
        self.math = math

        g = graph if graph.get("normalized") else normalize_graph(graph)
        self.hierarchical = bool(g["hierarchical"])
        self._register_graph(g)
        self.num_mesh_nodes, _ = self.get_num_mesh()
        self.grid_input_dim = datastore.grid_input_dim
        self.g2m_edges, g2m_dim = self.g2m_features.shape
        self.m2g_edges, m2g_dim = self.m2g_features.shape

        self.mlp_blueprint_end = [hidden_dim] * (hidden_layers + 1)
        self.grid_embedder = make_mlp([self.grid_input_dim] + self.mlp_blueprint_end)
        self.g2m_embedder = make_mlp([g2m_dim] + self.mlp_blueprint_end)
        self.m2g_embedder = make_mlp([m2g_dim] + self.mlp_blueprint_end)
        self.g2m_gnn = get_gnn_class(g2m_gnn_type)(self.g2m_edge_index, hidden_dim, hidden_layers=hidden_layers,
                                                   update_edges=False, math=math)
        self.encoding_grid_mlp = make_mlp([hidden_dim] + self.mlp_blueprint_end)
        self.m2g_gnn = get_gnn_class(m2g_gnn_type)(self.m2g_edge_index, hidden_dim, hidden_layers=hidden_layers,
                                                   update_edges=False, math=math)
        self.output_map = make_mlp([hidden_dim] * (hidden_layers + 1) + [self.grid_output_dim], layer_norm=False)
        self._static_cache = None
        self._set_mlp_flags()

    # -- graph registration (reference utils/graph.py:425-466: non-persistent buffers) -------
    def _register_graph(self, g):
        def reg(name, ei, feat):
            ei, feat = _sort_edges(ei.long(), feat.float())
            self.register_buffer(f"{name}_edge_index", ei, persistent=False)
            self.register_buffer(f"{name}_features", feat, persistent=False)

        reg("g2m", g["g2m_edge_index"], g["g2m_features"])
        reg("m2g", g["m2g_edge_index"], g["m2g_features"])
        if self.hierarchical:
            for name in ("m2m", "mesh_up", "mesh_down"):
                pairs = [_sort_edges(e.long(), f.float()) for e, f in zip(g[f"{name}_edge_index"], g[f"{name}_features"])]
                setattr(self, f"{name}_edge_index", BufferList([p[0] for p in pairs]))
                setattr(self, f"{name}_features", BufferList([p[1] for p in pairs]))
            self.mesh_static_features = BufferList([m.float() for m in g["mesh_static_features"]])
        else:
            reg("m2m", g["m2m_edge_index"], g["m2m_features"])
            self.register_buffer("mesh_static_features", g["mesh_static_features"].float(), persistent=False)

    def _set_mlp_flags(self):
        flag = {"auto": 0, None: None, "tf32": _lib.MATH_TF32, "fp32": _lib.MATH_FP32}[self.math]
        if flag is None:
            return
        for m in self.modules():
            if hasattr(m, "nlam_flags"):
                # embedders with tiny inputs always run exact; "tf32" is only forced on the GNNs
                m.nlam_flags = _lib.MATH_FP32 if self.math == "fp32" else 0

    # -- static (input independent) embeddings ----------------------------------------------
    def _static_param_version(self):
        # (version counter, storage address): ``p.data = new`` (EMA-style weight swaps) changes the address without
        # bumping the counter, in-place optimiser steps bump the counter without changing the address
        return tuple((p._version, p.data_ptr()) for p in self._static_params())

    def invalidate_static_cache(self):
        """Drop the cached input-independent embeddings (they are rebuilt on the next no-grad forward)."""
        self._static_cache = None

    def _static_params(self):
        raise NotImplementedError

    def _compute_static(self):
        raise NotImplementedError

    def static_embeddings(self):
        """Embeddings of static graph features.  The reference recomputes them every step
        (graph/base.py:289-295); they only depend on the weights, so in no-grad mode they are
        cached until a parameter changes."""
        if torch.is_grad_enabled():
            return self._compute_static()
        ver = self._static_param_version()
        if self._static_cache is None or self._static_cache[0] != ver or self._static_cache[1] != self.diff_std.device:
            self._static_cache = (ver, self.diff_std.device, self._compute_static())
        return self._static_cache[2]

    def get_num_mesh(self):
        raise NotImplementedError

    def process_step(self, mesh_rep, static):
        raise NotImplementedError

    def _encode(self, prev_state, prev_prev_state, forcing):
        """Grid embedder, grid -> mesh layer and encoding grid MLP (reference graph/base.py:275-310) ->
        (static embeddings, mesh_rep, grid_rep)."""
        B = prev_state.shape[0]
        # grid feature concat (base.py:275-283) is fused into the embedder kernel
        sources = [prev_state, prev_prev_state, forcing, self.expand_to_batch(self.grid_static_features, B)]
        if not torch.is_grad_enabled():
            # one launch for the embedder, the g2m node projections and the encoding grid MLP where the library covers the
            # shapes; the grid embedding never goes to HBM.  forward_with_boundary and the no-grad forward both take it, so the
            # eager and the captured step compute the same values
            st = self.static_embeddings()
            fused = self.g2m_gnn.encode_step(self.grid_embedder, self.encoding_grid_mlp, sources,
                                             self.expand_to_batch(st["mesh_emb"], B), self.expand_to_batch(st["g2m_emb"], B))
            if fused is not None:
                return st, fused[0], fused[1]
        grid_emb = self.grid_embedder.apply_rows(sources)
        st = self.static_embeddings()
        mesh_rep = self.g2m_gnn(grid_emb, self.expand_to_batch(st["mesh_emb"], B), self.expand_to_batch(st["g2m_emb"], B))
        grid_rep = self.encoding_grid_mlp.apply_rows([grid_emb], res=grid_emb)  # base.py:308-310
        return st, mesh_rep, grid_rep

    def forward(self, prev_state, prev_prev_state, forcing):
        """``(B,G,d_state), (B,G,d_state), (B,G,d_forcing) -> (new_state, pred_std|None)``
        (reference graph/base.py:228-344)."""
        B = prev_state.shape[0]
        st, mesh_rep, grid_rep = self._encode(prev_state, prev_prev_state, forcing)
        mesh_rep = self.process_step(mesh_rep, st)
        m2g_emb = self.expand_to_batch(st["m2g_emb"], B)
        inference = not torch.is_grad_enabled() and not self.output_std and not self.clamps_output
        if inference and hasattr(self.m2g_gnn, "decode_step"):
            # the fused decoder, as forward_with_boundary runs it: the eager and the captured step compute the same values
            fused = self.m2g_gnn.decode_step(mesh_rep, grid_rep, m2g_emb, self.output_map, prev_state, None, None, self.diff_std,
                                             self.diff_mean, out_flags=self.output_map.nlam_flags)
            if fused is not None:
                return fused, None
        grid_rep = self.m2g_gnn(mesh_rep, grid_rep, m2g_emb)
        if inference:
            # output_map + rescale (base.py:339) + residual (base.py:342) in one launch where the library fuses it
            fused = ops.rowmlp_step(self.output_map, grid_rep, prev_state, None, None, self.diff_std, self.diff_mean,
                                    flags=self.output_map.nlam_flags)
            if fused is not None:
                return fused, None
        net_output = self.output_map(grid_rep)
        if self.output_std:
            pred_delta_mean, pred_std_raw = net_output.chunk(2, dim=-1)
            pred_std = torch.nn.functional.softplus(pred_std_raw)
        else:
            pred_delta_mean, pred_std = net_output, None
        if not torch.is_grad_enabled():
            # rescale (base.py:339) + (clamped) residual update (base.py:342, step_predictors/base.py:366-396) in one kernel
            clamp = (self._clamp_kind, self._clamp_lo, self._clamp_up) if self.clamps_output else None
            return ops.step_epilogue(pred_delta_mean.contiguous(), prev_state, None, None, self.diff_std, self.diff_mean,
                                     clamp=clamp), pred_std
        rescaled = pred_delta_mean * self.diff_std + self.diff_mean
        return self.get_clamped_new_state(rescaled, prev_state), pred_std

    @torch.no_grad()
    def forward_with_boundary(self, prev_state, prev_prev_state, forcing, boundary_state, boundary_mask, out=None):
        """Inference step with the ARForecaster boundary mix (autoregressive.py:128-131) fused
        into the step epilogue kernel.  ``out``: optional preallocated (B,G,d) tensor for the new state."""
        assert not self.output_std
        B = prev_state.shape[0]
        st, mesh_rep, grid_rep = self._encode(prev_state, prev_prev_state, forcing)
        mesh_rep = self.process_step(mesh_rep, st)
        clamp = (self._clamp_kind, self._clamp_lo, self._clamp_up) if self.clamps_output else None
        m2g_emb = self.expand_to_batch(st["m2g_emb"], B)
        if clamp is None and hasattr(self.m2g_gnn, "aggregate_only"):
            # the whole decoder (edge projections, then edges + aggregation + node update + output_map + step epilogue in one
            # kernel) where the m2g graph has a uniform in-degree the kernel covers
            fused = self.m2g_gnn.decode_step(mesh_rep, grid_rep, m2g_emb, self.output_map, prev_state, boundary_state,
                                             boundary_mask, self.diff_std, self.diff_mean,
                                             out_flags=self.output_map.nlam_flags, out=out)
            if fused is not None:
                return fused
            # node update of the mesh->grid layer + output_map + step epilogue in one kernel: the updated grid
            # representation (which nothing else reads) never goes to HBM
            aggr = self.m2g_gnn.aggregate_only(mesh_rep, grid_rep, m2g_emb)
            if aggr is not None:
                fused = ops.node_update_step(self.m2g_gnn.aggr_mlp, self.output_map, grid_rep, aggr, prev_state, boundary_state,
                                             boundary_mask, self.diff_std, self.diff_mean,
                                             flags=self.output_map.nlam_flags, out=out)
                if fused is not None:
                    return fused
                grid_rep = self.m2g_gnn._kernel_node_update(grid_rep, aggr)
            else:
                grid_rep = self.m2g_gnn(mesh_rep, grid_rep, m2g_emb)
        else:
            grid_rep = self.m2g_gnn(mesh_rep, grid_rep, m2g_emb)
        if clamp is None:
            fused = ops.rowmlp_step(self.output_map, grid_rep, prev_state, boundary_state, boundary_mask, self.diff_std,
                                    self.diff_mean, flags=self.output_map.nlam_flags, out=out)
            if fused is not None:
                return fused
        net_output = self.output_map(grid_rep)
        # rescale + (clamped) update + boundary mix in one kernel
        return ops.step_epilogue(net_output, prev_state, boundary_state, boundary_mask, self.diff_std, self.diff_mean,
                                 out=out, clamp=clamp)


class GraphLAM(BaseGraphModel):
    """Flat (1-level or multiscale) mesh: ``processor_layers`` InteractionNets over m2m."""

    def __init__(self, datastore, graph, hidden_dim=64, hidden_layers=1, processor_layers=4, mesh_aggr="sum",
                 output_std=False, g2m_gnn_type="InteractionNet", m2g_gnn_type="InteractionNet", math=None,
                 **kwargs):
        super().__init__(datastore, graph, hidden_dim=hidden_dim, hidden_layers=hidden_layers,
                         processor_layers=processor_layers, mesh_aggr=mesh_aggr, output_std=output_std,
                         g2m_gnn_type=g2m_gnn_type, m2g_gnn_type=m2g_gnn_type, math=math,
                         output_clamping_lower=kwargs.get("output_clamping_lower"),
                         output_clamping_upper=kwargs.get("output_clamping_upper"))
        assert not self.hierarchical, "GraphLAM does not use a hierarchical mesh graph"
        mesh_dim = self.mesh_static_features.shape[1]
        m2m_dim = self.m2m_features.shape[1]
        self.mesh_embedder = make_mlp([mesh_dim] + self.mlp_blueprint_end)
        self.m2m_embedder = make_mlp([m2m_dim] + self.mlp_blueprint_end)
        self.processor = GNNSequential([
            InteractionNet(self.m2m_edge_index, hidden_dim, hidden_layers=hidden_layers, aggr=mesh_aggr, math=math)
            for _ in range(processor_layers)])
        self._set_mlp_flags()

    def get_num_mesh(self):
        return self.mesh_static_features.shape[0], 0

    def _static_params(self):
        return [p for m in (self.g2m_embedder, self.m2g_embedder, self.mesh_embedder, self.m2m_embedder)
                for p in m.parameters()]

    def _compute_static(self):
        return {"g2m_emb": self.g2m_embedder(self.g2m_features), "m2g_emb": self.m2g_embedder(self.m2g_features),
                "mesh_emb": self.mesh_embedder(self.mesh_static_features),
                "m2m_emb": self.m2m_embedder(self.m2m_features)}

    def embedd_mesh_nodes(self):
        return self.mesh_embedder(self.mesh_static_features)

    def process_step(self, mesh_rep, static=None):
        """reference graph/graph_lam.py:157-188"""
        static = static or self.static_embeddings()
        B = mesh_rep.shape[0]
        mesh_rep, _ = self.processor(mesh_rep, self.expand_to_batch(static["m2m_emb"], B), keep_edge_rep=False)
        return mesh_rep


class BaseHiGraphModel(BaseGraphModel):
    """Hierarchical mesh: per-level embedders, mesh-init (up) and read-out (down) GNNs."""

    def __init__(self, datastore, graph, hidden_dim=64, hidden_layers=1, processor_layers=4, mesh_aggr="sum",
                 output_std=False, g2m_gnn_type="InteractionNet", m2g_gnn_type="InteractionNet",
                 mesh_up_gnn_type="InteractionNet", mesh_down_gnn_type="InteractionNet", math=None, **kwargs):
        super().__init__(datastore, graph, hidden_dim=hidden_dim, hidden_layers=hidden_layers,
                         processor_layers=processor_layers, mesh_aggr=mesh_aggr, output_std=output_std,
                         g2m_gnn_type=g2m_gnn_type, m2g_gnn_type=m2g_gnn_type, math=math,
                         output_clamping_lower=kwargs.get("output_clamping_lower"),
                         output_clamping_upper=kwargs.get("output_clamping_upper"))
        assert self.hierarchical, "hierarchical models need a hierarchical mesh graph"
        self.mesh_up_gnn_type, self.mesh_down_gnn_type = mesh_up_gnn_type, mesh_down_gnn_type
        self.num_levels = len(self.mesh_static_features)
        self.level_mesh_sizes = [m.shape[0] for m in self.mesh_static_features]
        mesh_dim = self.mesh_static_features[0].shape[1]
        same_dim = self.m2m_features[0].shape[1]
        up_dim = self.mesh_up_features[0].shape[1]
        down_dim = self.mesh_down_features[0].shape[1]
        L = self.num_levels
        end = self.mlp_blueprint_end
        self.mesh_embedders = nn.ModuleList([make_mlp([mesh_dim] + end) for _ in range(L)])
        self.mesh_same_embedders = nn.ModuleList([make_mlp([same_dim] + end) for _ in range(L)])
        self.mesh_up_embedders = nn.ModuleList([make_mlp([up_dim] + end) for _ in range(L - 1)])
        self.mesh_down_embedders = nn.ModuleList([make_mlp([down_dim] + end) for _ in range(L - 1)])
        up_cls, down_cls = get_gnn_class(mesh_up_gnn_type), get_gnn_class(mesh_down_gnn_type)
        self.mesh_init_gnns = nn.ModuleList([
            up_cls(ei, hidden_dim, hidden_layers=hidden_layers, math=math) for ei in self.mesh_up_edge_index])
        self.mesh_read_gnns = nn.ModuleList([
            down_cls(ei, hidden_dim, hidden_layers=hidden_layers, update_edges=False, math=math)
            for ei in self.mesh_down_edge_index])

    def get_num_mesh(self):
        n = sum(m.shape[0] for m in self.mesh_static_features)
        return n, n - self.mesh_static_features[0].shape[0]

    def _static_params(self):
        mods = [self.g2m_embedder, self.m2g_embedder, *self.mesh_embedders, *self.mesh_same_embedders,
                *self.mesh_up_embedders, *self.mesh_down_embedders]
        return [p for m in mods for p in m.parameters()]

    def _compute_static(self):
        return {
            "g2m_emb": self.g2m_embedder(self.g2m_features), "m2g_emb": self.m2g_embedder(self.m2g_features),
            "mesh_emb": self.mesh_embedders[0](self.mesh_static_features[0]),
            "mesh_levels": [e(f) for e, f in zip(self.mesh_embedders[1:], self.mesh_static_features[1:])],
            "same": [e(f) for e, f in zip(self.mesh_same_embedders, self.m2m_features)],
            "up": [e(f) for e, f in zip(self.mesh_up_embedders, self.mesh_up_features)],
            "down": [e(f) for e, f in zip(self.mesh_down_embedders, self.mesh_down_features)],
        }

    def embedd_mesh_nodes(self):
        return self.mesh_embedders[0](self.mesh_static_features[0])

    def process_step(self, mesh_rep, static=None):
        """reference graph/hierarchical.py:186-292"""
        static = static or self.static_embeddings()
        B = mesh_rep.shape[0]
        ex = lambda t: self.expand_to_batch(t, B)  # noqa: E731
        levels = [mesh_rep] + [ex(t) for t in static["mesh_levels"]]
        same = [ex(t) for t in static["same"]]
        up = [ex(t) for t in static["up"]]
        down = [ex(t) for t in static["down"]]
        for l, gnn in enumerate(self.mesh_init_gnns, start=1):
            levels[l], up[l - 1] = gnn(levels[l - 1], levels[l], up[l - 1])
        levels, _, _, down = self.hi_processor_step(levels, same, up, down)
        for l, gnn in zip(range(self.num_levels - 2, -1, -1), reversed(self.mesh_read_gnns)):
            levels[l] = gnn(levels[l + 1], levels[l], down[l])
        return levels[0]

    def hi_processor_step(self, mesh_rep_levels, mesh_same_rep, mesh_up_rep, mesh_down_rep):
        raise NotImplementedError("hi_process_step not implemented")


class HiLAM(BaseHiGraphModel):
    """Hierarchical model with sequential down/up sweeps per processor layer
    (Hi-LAM, Oskarsson et al. 2023)."""

    def __init__(self, datastore, graph, **kwargs):
        super().__init__(datastore, graph, **kwargs)
        P = self.processor_layers
        self.mesh_down_gnns = nn.ModuleList([self.make_down_gnns() for _ in range(P)])
        self.mesh_down_same_gnns = nn.ModuleList([self.make_same_gnns() for _ in range(P)])
        self.mesh_up_gnns = nn.ModuleList([self.make_up_gnns() for _ in range(P)])
        self.mesh_up_same_gnns = nn.ModuleList([self.make_same_gnns() for _ in range(P)])
        self._set_mlp_flags()

    def make_same_gnns(self):
        return nn.ModuleList([InteractionNet(ei, self.hidden_dim, hidden_layers=self.hidden_layers, math=self.math)
                              for ei in self.m2m_edge_index])

    def make_up_gnns(self):
        cls = get_gnn_class(self.mesh_up_gnn_type)
        return nn.ModuleList([cls(ei, self.hidden_dim, hidden_layers=self.hidden_layers, math=self.math)
                              for ei in self.mesh_up_edge_index])

    def make_down_gnns(self):
        cls = get_gnn_class(self.mesh_down_gnn_type)
        return nn.ModuleList([cls(ei, self.hidden_dim, hidden_layers=self.hidden_layers, math=self.math)
                              for ei in self.mesh_down_edge_index])

    def mesh_down_step(self, levels, same, down, down_gnns, same_gnns):
        """reference graph/hi_lam.py:205-236"""
        levels[-1], same[-1] = same_gnns[-1](levels[-1], levels[-1], same[-1])
        for l, dg, sg in zip(range(self.num_levels - 2, -1, -1), reversed(down_gnns), reversed(same_gnns[:-1])):
            new_node, down[l] = dg(levels[l + 1], levels[l], down[l])
            levels[l], same[l] = sg(new_node, new_node, same[l])
        return levels, same, down

    def mesh_up_step(self, levels, same, up, up_gnns, same_gnns):
        """reference graph/hi_lam.py:277-307"""
        levels[0], same[0] = same_gnns[0](levels[0], levels[0], same[0])
        for l, (ug, sg) in enumerate(zip(up_gnns, same_gnns[1:]), start=1):
            new_node, up[l - 1] = ug(levels[l - 1], levels[l], up[l - 1])
            levels[l], same[l] = sg(new_node, new_node, same[l])
        return levels, same, up

    def hi_processor_step(self, levels, same, up, down):
        """reference graph/hi_lam.py:350-376"""
        for dg, dsg, ug, usg in zip(self.mesh_down_gnns, self.mesh_down_same_gnns, self.mesh_up_gnns,
                                    self.mesh_up_same_gnns):
            levels, same, down = self.mesh_down_step(levels, same, down, list(dg), list(dsg))
            levels, same, up = self.mesh_up_step(levels, same, up, list(ug), list(usg))
        return levels, same, up, down


class HiLAMParallel(BaseHiGraphModel):
    """Hierarchical model whose processor runs all same-level / up / down message passing of the mesh hierarchy
    as ONE InteractionNet over the concatenated node sets and edge sets, with separate MLPs per edge set and per
    level (reference graph/hi_lam_parallel.py: index offsets :89-122, processor :124-143,
    hi_processor_step :145-218)."""

    def __init__(self, datastore, graph, **kwargs):
        super().__init__(datastore, graph, **kwargs)
        first = [0]
        for size in self.level_mesh_sizes[:-1]:
            first.append(first[-1] + size)
        total = [ei + off for ei, off in zip(self.m2m_edge_index, first)]
        total += [torch.stack((ei[0] + first[l], ei[1] + first[l + 1])) for l, ei in enumerate(self.mesh_up_edge_index)]
        total += [torch.stack((ei[0] + first[l + 1], ei[1] + first[l])) for l, ei in enumerate(self.mesh_down_edge_index)]
        self.edge_split_sections = [ei.shape[1] for ei in total]
        total_edge_index = torch.cat(total, dim=1)
        self.processor = GNNSequential([
            InteractionNet(total_edge_index, self.hidden_dim, hidden_layers=self.hidden_layers,
                           edge_chunk_sizes=self.edge_split_sections, aggr_chunk_sizes=self.level_mesh_sizes,
                           math=self.math)
            for _ in range(self.processor_layers)])
        self._set_mlp_flags()

    def hi_processor_step(self, levels, same, up, down):
        """reference graph/hi_lam_parallel.py:186-218"""
        L = self.num_levels
        mesh_rep = torch.cat(levels, dim=1)
        edge_rep = torch.cat(list(same) + list(up) + list(down), dim=1)
        mesh_rep, edge_rep = self.processor(mesh_rep, edge_rep)
        levels = list(torch.split(mesh_rep, self.level_mesh_sizes, dim=1))
        sections = torch.split(edge_rep, self.edge_split_sections, dim=1)
        return levels, list(sections[:L]), list(sections[L:2 * L - 1]), list(sections[2 * L - 1:])


class BaseGraphEFM(BaseGraphModel):
    """Graph-EFM, the latent-variable ensemble forecaster (reference step_predictors/graph/graph_efm.py: BaseGraphEFM
    :25-471).  ``forward`` samples one step from the prior: grid embedding, prior over a latent on mesh nodes,
    reparameterised sample, decoder.  The variational posterior is ``self.encoder`` (conditioned on the target through
    ``embedd_grid_with_target``); the predictor computes no loss.

    Submodule names and persistent buffers are the reference's, so its state_dicts load strictly.  The graph registration
    and the cache of the weight-only embeddings are ``BaseGraphModel``'s; the encode-process-decode modules of
    ``BaseGraphModel.__init__`` are not built (``StepPredictor.__init__`` runs instead).  Subclasses define the mesh: its
    graph type, ``latent_spatial_dim``, the learnable prior, the weight-only embeddings and the no-grad ``_step``.

    Noise: ``latent_noise`` (B, latent_spatial_dim, latent_dim) is the standard normal ε of ``z = mean + ε * std``; without
    it ε is drawn with ``torch.randn`` on the default generator of the current device.  Under autograd the sample is
    composed from the module outputs in that order; the no-grad step runs the fused kernels where they cover the shapes."""

    samples_latent = True

    def __init__(self, datastore, graph, hidden_dim=64, hidden_layers=1, latent_dim=None, prior_layers=2, learn_prior=True,
                 prior_dist="isotropic", g2m_gnn_type="InteractionNet", m2g_gnn_type="InteractionNet", output_std=False,
                 output_clamping_lower=None, output_clamping_upper=None, math=None):
        StepPredictor.__init__(self, datastore, output_std=output_std, output_clamping_lower=output_clamping_lower,
                               output_clamping_upper=output_clamping_upper)
        self.g2m_gnn_type, self.m2g_gnn_type = g2m_gnn_type, m2g_gnn_type
        self.register_buffer("diff_mean", datastore.state_diff_mean.float(), persistent=False)
        self.register_buffer("diff_std", datastore.state_diff_std.float(), persistent=False)
        self.hidden_dim, self.hidden_layers, self.math = hidden_dim, hidden_layers, math
        g = graph if graph.get("normalized") else normalize_graph(graph)
        self.hierarchical = bool(g["hierarchical"])
        self.check_graph_type()
        self._register_graph(g)
        self.num_mesh_nodes, _ = self.get_num_mesh()
        self.grid_input_dim = self.grid_dim = datastore.grid_input_dim
        g2m_dim, m2g_dim = self.g2m_features.shape[1], self.m2g_features.shape[1]

        self.mlp_blueprint_end = [hidden_dim] * (hidden_layers + 1)
        self.grid_prev_embedder = make_mlp([self.grid_dim] + self.mlp_blueprint_end)
        self.grid_current_embedder = make_mlp([self.grid_dim + self.num_state_vars] + self.mlp_blueprint_end)
        self.g2m_embedder = make_mlp([g2m_dim] + self.mlp_blueprint_end)
        self.m2g_embedder = make_mlp([m2g_dim] + self.mlp_blueprint_end)
        self.latent_dim = latent_dim if latent_dim is not None else hidden_dim
        if learn_prior:
            self.prior_model = self.build_learnable_prior(prior_layers, prior_dist)
        else:
            self.prior_model = ConstantLatentEncoder(self.latent_dim, self.latent_spatial_dim, output_dist=prior_dist)
        self._static_cache = None

    def check_graph_type(self):
        raise NotImplementedError

    @property
    def latent_spatial_dim(self):
        raise NotImplementedError

    def build_learnable_prior(self, prior_layers, prior_dist):
        raise NotImplementedError

    def _graph_emb(self, batch_size):
        raise NotImplementedError

    def _grid_sources(self, prev_state, prev_prev_state, forcing):
        # Graph-EFM's order puts X_{t-1} first (graph_efm.py:386-394; GraphLAM puts X_t first)
        return [prev_prev_state, prev_state, forcing, self.expand_to_batch(self.grid_static_features, prev_state.shape[0])]

    def embedd_grid_and_graph(self, prev_state, prev_prev_state, forcing):
        """-> (grid_emb (B, G, H), graph_emb {g2m, m2g, mesh embeddings}) (graph_efm.py:364-413)"""
        grid_emb = self.grid_prev_embedder.apply_rows(self._grid_sources(prev_state, prev_prev_state, forcing))
        return grid_emb, self._graph_emb(prev_state.shape[0])

    def embedd_grid_with_target(self, prev_state, prev_prev_state, forcing, current_state):
        """Grid embedding including the target X_{t+1}, the input of the variational encoder (graph_efm.py:301-343)."""
        prev_prev, prev, forc, static = self._grid_sources(prev_state, prev_prev_state, forcing)
        # the row kernels take at most four sources: the last two columns blocks go in as one
        return self.grid_current_embedder.apply_rows([prev_prev, prev, forc, torch.cat((static, current_state), dim=-1)])

    def _noise(self, latent_noise, batch_size, device):
        shape = (batch_size, self.latent_spatial_dim, self.latent_dim)
        if latent_noise is None:
            return torch.randn(shape, device=device)
        if tuple(latent_noise.shape) != shape:
            raise ValueError(f"latent_noise: expected shape {shape}, got {tuple(latent_noise.shape)}")
        return latent_noise

    def forward(self, prev_state, prev_prev_state, forcing, latent_noise=None):
        """``(B,G,d_state) x 2, (B,G,d_forcing) -> (new_state, pred_std|None)``: one step sampled from the prior
        (graph_efm.py:415-471)."""
        if not torch.is_grad_enabled():
            return self._step(prev_state, prev_prev_state, forcing, latent_noise, None, None, None)
        grid_emb, graph_emb = self.embedd_grid_and_graph(prev_state, prev_prev_state, forcing)
        prior = self.prior_model(grid_emb, graph_emb=graph_emb)
        eps = self._noise(latent_noise, prev_state.shape[0], prev_state.device)
        latent_samples = prior.mean + eps * prior.stddev
        mean_delta, pred_std = self.decoder(grid_emb, latent_samples, graph_emb)
        rescaled = mean_delta * self.diff_std + self.diff_mean
        return self.get_clamped_new_state(rescaled, prev_state), pred_std

    @torch.no_grad()
    def forward_with_boundary(self, prev_state, prev_prev_state, forcing, boundary_state, boundary_mask, latent_noise=None,
                              out=None):
        """Inference step with the ARForecaster boundary mix fused into the step epilogue.  ``out``: optional preallocated
        (B,G,d) tensor for the new state."""
        assert not self.output_std
        return self._step(prev_state, prev_prev_state, forcing, latent_noise, boundary_state, boundary_mask, out)[0]

    def _step(self, prev_state, prev_prev_state, forcing, latent_noise, boundary, bmask, out):
        raise NotImplementedError

    def _sample_latent(self, mesh_rep, grid_emb, eps):
        """Prior parameters + sample + latent embedding: one launch where the library covers the shapes, else composed.
        ``mesh_rep``: the learned prior's representation on the latent's mesh nodes (None for a constant prior)."""
        prior, dec = self.prior_model, self.decoder
        if mesh_rep is not None:
            latent_emb = ops.latent_sample(prior.latent_param_map, dec.latent_embedder, mesh_rep, eps,
                                           flags=prior.latent_param_map.nlam_flags | dec.latent_embedder.nlam_flags)
            if latent_emb is not None:
                return latent_emb
        dist = prior.latent_param_map(mesh_rep) if mesh_rep is not None else prior.compute_dist_params(grid_emb)
        mean, std = prior.mean_std(dist)
        return dec.latent_embedder.apply_rows([mean + eps * std])

    def _decode(self, mesh_rep, grid_rep, m2g_emb, prev_state, boundary, bmask, out):
        """m2g + param_map + (clamped) step epilogue with the boundary mix: the fused decoder where the graph / shapes allow,
        else the launch chains ``BaseGraphModel.forward_with_boundary`` falls back to -> (new_state, pred_std|None)."""
        dec = self.decoder
        m2g, pm = dec.m2g_gnn, dec.param_map
        clamp = (self._clamp_kind, self._clamp_lo, self._clamp_up) if self.clamps_output else None
        if clamp is None and not self.output_std:
            fused = m2g.decode_step(mesh_rep, grid_rep, m2g_emb, pm, prev_state, boundary, bmask, self.diff_std, self.diff_mean,
                                    out_flags=pm.nlam_flags, out=out)
            if fused is not None:
                return fused, None
            aggr = m2g.aggregate_only(mesh_rep, grid_rep, m2g_emb)
            if aggr is not None:
                fused = ops.node_update_step(m2g.aggr_mlp, pm, grid_rep, aggr, prev_state, boundary, bmask, self.diff_std,
                                             self.diff_mean, flags=pm.nlam_flags, out=out)
                if fused is not None:
                    return fused, None
                grid_rep = m2g._kernel_node_update(grid_rep, aggr)
            else:
                grid_rep = m2g(mesh_rep, grid_rep, m2g_emb)
            fused = ops.rowmlp_step(pm, grid_rep, prev_state, boundary, bmask, self.diff_std, self.diff_mean,
                                    flags=pm.nlam_flags, out=out)
            if fused is not None:
                return fused, None
        else:
            grid_rep = m2g(mesh_rep, grid_rep, m2g_emb)
        net_output = pm(grid_rep)
        pred_std = None
        if self.output_std:
            net_output, std_raw = net_output.chunk(2, dim=-1)
            pred_std = torch.nn.functional.softplus(std_raw)
        return ops.step_epilogue(net_output.contiguous(), prev_state, boundary, bmask, self.diff_std, self.diff_mean, out=out,
                                 clamp=clamp), pred_std


class GraphEFMMultiScale(BaseGraphEFM):
    """Graph-EFM on a flat (multiscale) mesh (reference step_predictors/graph/graph_efm.py: GraphEFMMultiScale :796-1037):
    the latent lives on every mesh node; prior and variational posterior are ``GraphLatentEncoder``s, the decoder is a
    ``GraphLatentDecoder``."""

    def __init__(self, datastore, graph, hidden_dim=64, hidden_layers=1, latent_dim=None, prior_m2m_layers=2,
                 encoder_m2m_layers=2, decoder_m2m_layers=4, learn_prior=True, prior_dist="isotropic",
                 g2m_gnn_type="InteractionNet", m2g_gnn_type="InteractionNet", output_std=False,
                 output_clamping_lower=None, output_clamping_upper=None, math=None):
        super().__init__(datastore, graph, hidden_dim=hidden_dim, hidden_layers=hidden_layers, latent_dim=latent_dim,
                         prior_layers=prior_m2m_layers, learn_prior=learn_prior, prior_dist=prior_dist,
                         g2m_gnn_type=g2m_gnn_type, m2g_gnn_type=m2g_gnn_type, output_std=output_std,
                         output_clamping_lower=output_clamping_lower, output_clamping_upper=output_clamping_upper, math=math)
        self.mesh_embedder = make_mlp([self.mesh_static_features.shape[1]] + self.mlp_blueprint_end)
        self.m2m_embedder = make_mlp([self.m2m_features.shape[1]] + self.mlp_blueprint_end)
        self.encoder = GraphLatentEncoder(self.latent_dim, self.g2m_edge_index, self.m2m_edge_index, hidden_dim,
                                          encoder_m2m_layers, hidden_layers=hidden_layers, g2m_gnn_type=g2m_gnn_type,
                                          output_dist="diagonal", math=math)
        self.decoder = GraphLatentDecoder(self.g2m_edge_index, self.m2m_edge_index, self.m2g_edge_index, hidden_dim,
                                          self.latent_dim, self.num_state_vars, decoder_m2m_layers, hidden_layers=hidden_layers,
                                          g2m_gnn_type=g2m_gnn_type, m2g_gnn_type=m2g_gnn_type, output_std=bool(output_std),
                                          math=math)
        self._set_mlp_flags()

    def check_graph_type(self):
        if self.hierarchical:
            raise ValueError(f"{type(self).__name__} requires a flat mesh graph, but the graph is hierarchical")

    def build_learnable_prior(self, prior_layers, prior_dist):
        return GraphLatentEncoder(self.latent_dim, self.g2m_edge_index, self.m2m_edge_index, self.hidden_dim, prior_layers,
                                  hidden_layers=self.hidden_layers, g2m_gnn_type=self.g2m_gnn_type, output_dist=prior_dist,
                                  math=self.math)

    def get_num_mesh(self):
        return self.mesh_static_features.shape[0], 0

    @property
    def latent_spatial_dim(self):
        return self.num_mesh_nodes

    def _static_params(self):
        return [p for m in (self.g2m_embedder, self.m2g_embedder, self.mesh_embedder, self.m2m_embedder)
                for p in m.parameters()]

    def _compute_static(self):
        return {"g2m_emb": self.g2m_embedder(self.g2m_features), "m2g_emb": self.m2g_embedder(self.m2g_features),
                "mesh_emb": self.mesh_embedder(self.mesh_static_features),
                "m2m_emb": self.m2m_embedder(self.m2m_features)}

    def _graph_emb(self, batch_size):
        st = self.static_embeddings()
        return {k: self.expand_to_batch(st[f"{k}_emb"], batch_size) for k in ("g2m", "m2g", "mesh", "m2m")}

    def embedd_mesh(self, batch_size):
        """``mesh`` and ``m2m`` embeddings expanded to the batch (graph_efm.py:1015-1037)."""
        ge = self._graph_emb(batch_size)
        return {"mesh": ge["mesh"], "m2m": ge["m2m"]}

    @torch.no_grad()
    def _step(self, prev_state, prev_prev_state, forcing, latent_noise, boundary, bmask, out):
        """The no-grad step: (1) grid embedder, decoder grid MLP and the prior g2m's projections in one launch, (2) prior g2m,
        (3) prior m2m stack, (4) prior parameters + sample + latent embedding in one launch, (5) decoder g2m, (6) decoder
        m2m stack, (7) m2g + param_map + step epilogue.  Each fused launch falls back to its composition where the library
        does not cover the shapes."""
        B = prev_state.shape[0]
        ge = self._graph_emb(B)
        prior, dec = self.prior_model, self.decoder
        learned = isinstance(prior, GraphLatentEncoder)
        sources = self._grid_sources(prev_state, prev_prev_state, forcing)
        enc = None
        if learned:
            enc = prior.g2m_gnn.encode_step(self.grid_prev_embedder, dec.grid_update_mlp, sources, ge["mesh"], ge["g2m"],
                                            want_grid_emb=True)
        if enc is not None:
            mesh_rep, res_grid, grid_emb = enc
        else:
            grid_emb = self.grid_prev_embedder.apply_rows(sources)
            res_grid = dec.grid_update_mlp.apply_rows([grid_emb], res=grid_emb)
            mesh_rep = prior.g2m_gnn(grid_emb, ge["mesh"], ge["g2m"]) if learned else None
        eps = self._noise(latent_noise, B, prev_state.device)
        if learned:
            mesh_rep = prior.process_mesh(mesh_rep, ge["m2m"])
        latent_emb = self._sample_latent(mesh_rep, grid_emb, eps)
        mesh_rep = dec.mesh_step(grid_emb, latent_emb, ge)
        return self._decode(mesh_rep, res_grid, ge["m2g"], prev_state, boundary, bmask, out)


class GraphEFM(BaseGraphEFM):
    """Graph-EFM on a hierarchical mesh, the reference's default Graph-EFM (reference step_predictors/graph/graph_efm.py:
    GraphEFM :474-793): the latent lives on the top mesh level; prior and variational posterior are
    ``HiGraphLatentEncoder``s, the decoder is a ``HiGraphLatentDecoder``.  ``m2m_embedders`` exist only when some stack has
    intra-level layers (``embedd_m2m``)."""

    def __init__(self, datastore, graph, hidden_dim=64, hidden_layers=1, latent_dim=None, prior_intra_level_layers=2,
                 encoder_intra_level_layers=2, decoder_intra_level_layers=4, learn_prior=True, prior_dist="isotropic",
                 g2m_gnn_type="InteractionNet", m2g_gnn_type="InteractionNet", output_std=False,
                 output_clamping_lower=None, output_clamping_upper=None, math=None):
        super().__init__(datastore, graph, hidden_dim=hidden_dim, hidden_layers=hidden_layers, latent_dim=latent_dim,
                         prior_layers=prior_intra_level_layers, learn_prior=learn_prior, prior_dist=prior_dist,
                         g2m_gnn_type=g2m_gnn_type, m2g_gnn_type=m2g_gnn_type, output_std=output_std,
                         output_clamping_lower=output_clamping_lower, output_clamping_upper=output_clamping_upper, math=math)
        self.num_levels = len(self.mesh_static_features)
        self.level_mesh_sizes = [m.shape[0] for m in self.mesh_static_features]
        L, end = self.num_levels, self.mlp_blueprint_end
        mesh_dim = self.mesh_static_features[0].shape[1]
        m2m_dim = self.m2m_features[0].shape[1]
        up_dim, down_dim = self.mesh_up_features[0].shape[1], self.mesh_down_features[0].shape[1]
        self.mesh_embedders = nn.ModuleList([make_mlp([mesh_dim] + end) for _ in range(L)])
        self.mesh_up_embedders = nn.ModuleList([make_mlp([up_dim] + end) for _ in range(L - 1)])
        self.mesh_down_embedders = nn.ModuleList([make_mlp([down_dim] + end) for _ in range(L - 1)])
        self.embedd_m2m = max(prior_intra_level_layers, encoder_intra_level_layers, decoder_intra_level_layers) > 0
        if self.embedd_m2m:
            self.m2m_embedders = nn.ModuleList([make_mlp([m2m_dim] + end) for _ in range(L)])
        self.encoder = HiGraphLatentEncoder(self.latent_dim, self.g2m_edge_index, self.m2m_edge_index, self.mesh_up_edge_index,
                                            hidden_dim, encoder_intra_level_layers, hidden_layers=hidden_layers,
                                            g2m_gnn_type=g2m_gnn_type, output_dist="diagonal", math=math)
        self.decoder = HiGraphLatentDecoder(self.g2m_edge_index, self.m2m_edge_index, self.m2g_edge_index,
                                            self.mesh_up_edge_index, self.mesh_down_edge_index, hidden_dim, self.latent_dim,
                                            self.num_state_vars, decoder_intra_level_layers, hidden_layers=hidden_layers,
                                            g2m_gnn_type=g2m_gnn_type, m2g_gnn_type=m2g_gnn_type, output_std=bool(output_std),
                                            math=math)
        self._set_mlp_flags()

    def check_graph_type(self):
        if not self.hierarchical:
            raise ValueError(f"{type(self).__name__} requires a hierarchical mesh graph, but the graph is flat")

    def build_learnable_prior(self, prior_layers, prior_dist):
        return HiGraphLatentEncoder(self.latent_dim, self.g2m_edge_index, self.m2m_edge_index, self.mesh_up_edge_index,
                                    self.hidden_dim, prior_layers, hidden_layers=self.hidden_layers,
                                    g2m_gnn_type=self.g2m_gnn_type, output_dist=prior_dist, math=self.math)

    def get_num_mesh(self):
        n = sum(m.shape[0] for m in self.mesh_static_features)
        return n, n - self.mesh_static_features[0].shape[0]

    @property
    def latent_spatial_dim(self):
        return self.mesh_static_features[-1].shape[0]

    def _embedders(self):
        return {"mesh": (self.mesh_embedders, self.mesh_static_features),
                "mesh_up": (self.mesh_up_embedders, self.mesh_up_features),
                "mesh_down": (self.mesh_down_embedders, self.mesh_down_features),
                "m2m": (self.m2m_embedders if self.embedd_m2m else [], self.m2m_features)}

    def _static_params(self):
        mods = [self.g2m_embedder, self.m2g_embedder] + [m for embs, _ in self._embedders().values() for m in embs]
        return [p for m in mods for p in m.parameters()]

    def _compute_static(self):
        st = {"g2m": self.g2m_embedder(self.g2m_features), "m2g": self.m2g_embedder(self.m2g_features)}
        for k, (embs, feats) in self._embedders().items():
            st[k] = [e(f) for e, f in zip(embs, feats)]
        return st

    def _graph_emb(self, batch_size):
        ex = lambda t: self.expand_to_batch(t, batch_size)  # noqa: E731
        return {k: ([ex(t) for t in v] if isinstance(v, list) else ex(v)) for k, v in self.static_embeddings().items()}

    def embedd_mesh(self, batch_size):
        """``mesh``, ``m2m`` (empty without intra-level layers), ``mesh_up`` and ``mesh_down`` embeddings per level, expanded
        to the batch (graph_efm.py:746-793)."""
        ge = self._graph_emb(batch_size)
        return {k: ge[k] for k in ("mesh", "mesh_up", "mesh_down", "m2m")}

    @torch.no_grad()
    def _step(self, prev_state, prev_prev_state, forcing, latent_noise, boundary, bmask, out):
        """The no-grad step: (1) grid embedder, decoder grid MLP and the projections of both g2m layers (the prior's and the
        decoder's: both have the static level-0 embedding as receivers) in one launch, then both g2m layers on their
        projections, (2) the prior's sweep up the hierarchy, (3) prior parameters + sample + latent embedding in one launch,
        (4) the decoder's up and down sweeps, (5) m2g + param_map + step epilogue.  With a constant prior the launch of (1)
        serves the decoder's g2m alone.  Each fused launch falls back to its composition where the library does not cover
        the shapes."""
        B = prev_state.shape[0]
        ge = self._graph_emb(B)
        prior, dec = self.prior_model, self.decoder
        learned = isinstance(prior, HiGraphLatentEncoder)
        sources = self._grid_sources(prev_state, prev_prev_state, forcing)
        mesh0, g2m = ge["mesh"][0], ge["g2m"]
        grid_emb = prior_rep = None
        if learned:
            enc = prior.g2m_gnn.encode_step(self.grid_prev_embedder, dec.grid_update_mlp, sources, mesh0, g2m,
                                            second=dec.g2m_gnn)
            if enc is not None:
                prior_rep, res_grid, dec_rep = enc
        else:
            enc = dec.g2m_gnn.encode_step(self.grid_prev_embedder, dec.grid_update_mlp, sources, mesh0, g2m)
            if enc is not None:
                dec_rep, res_grid = enc
        if enc is None:
            grid_emb = self.grid_prev_embedder.apply_rows(sources)
            res_grid = dec.grid_update_mlp.apply_rows([grid_emb], res=grid_emb)
            prior_rep = prior.g2m_gnn(grid_emb, mesh0, g2m) if learned else None
            dec_rep = dec.g2m_gnn(grid_emb, mesh0, g2m)
        eps = self._noise(latent_noise, B, prev_state.device)
        if learned:
            prior_rep = prior.process_mesh(prior_rep, ge)
        elif grid_emb is None:  # the constant prior reads only the batch size and device of its input
            grid_emb = res_grid
        latent_emb = self._sample_latent(prior_rep, grid_emb, eps)
        mesh_rep = dec.mesh_step(dec_rep, latent_emb, ge)
        return self._decode(mesh_rep, res_grid, ge["m2g"], prev_state, boundary, bmask, out)


MODELS = {"graph_lam": GraphLAM, "hi_lam": HiLAM, "hi_lam_parallel": HiLAMParallel}


def _boundary_blocks(mask, max_blocks=8, min_saving=0.2):
    """Row runs of a (G,) boundary mask as copy blocks ``(start node, run length, pitch, count)``: ``count`` runs of
    ``run length`` nodes, ``pitch`` nodes apart (count == 1: a single run).  None when the mask is not worth compacting
    (everything selected, too fragmented for a handful of strided copies, or the strips do not tile the grid evenly)."""
    import os
    if os.environ.get("NLAM_NO_BOUNDARY_COMPACTION"):
        return None
    m = (mask.reshape(-1) > 0).to("cpu").numpy().astype("int8")
    G = m.shape[0]
    if G == 0 or m.sum() == 0 or m.sum() > (1.0 - min_saving) * G:
        return None
    import numpy as np
    d = np.diff(np.concatenate([[0], m, [0]]))
    starts, ends = np.nonzero(d == 1)[0], np.nonzero(d == -1)[0]
    runs = list(zip(starts.tolist(), (ends - starts).tolist()))
    blocks, j = [], 0
    while j < len(runs):
        s0, l0 = runs[j]
        n = 1
        if j + 1 < len(runs) and runs[j + 1][1] == l0:
            pitch = runs[j + 1][0] - s0
            while j + n < len(runs) and runs[j + n][1] == l0 and runs[j + n][0] == s0 + n * pitch:
                n += 1
            # a 3-D copy needs the slice stride (G nodes per sample) to be a whole number of pitches
            if n > 1 and (G % pitch != 0 or l0 > pitch or n > G // pitch or l0 < 4):  # (runs of a few bytes: not worth it)
                n = 1
        if n > 1:
            blocks.append((s0, l0, pitch, n))
        else:
            blocks.append((s0, l0, 0, 1))
        j += n
        if len(blocks) > max_blocks:
            return None
    return blocks


class ARForecaster(nn.Module):
    """Autoregressive rollout with boundary overwrite (reference
    models/forecasters/autoregressive.py:63-149).  ``forward`` keeps the reference semantics;
    ``rollout_graphed`` replays one CUDA-graph-captured forecast step per AR step (inference)."""

    def __init__(self, predictor, datastore):
        super().__init__()
        self.predictor = predictor
        bm = datastore.boundary_mask.float()
        self.register_buffer("boundary_mask", bm, persistent=False)
        self.register_buffer("interior_mask", 1.0 - bm, persistent=False)
        self._graph = None

    @property
    def predicts_std(self):
        return self.predictor.predicts_std

    def forward(self, init_states, forcing_features, boundary_states):
        """init_states (B,2,G,d), forcing (B,T,G,f), boundary (B,T,G,d) -> (prediction (B,T,G,d), std|None)"""
        prev_prev_state, prev_state = init_states[:, 0], init_states[:, 1]
        preds, stds = [], []
        for i in range(forcing_features.shape[1]):
            pred_state, pred_std = self.predictor(prev_state, prev_prev_state, forcing_features[:, i])
            new_state = self.boundary_mask * boundary_states[:, i] + self.interior_mask * pred_state
            preds.append(new_state)
            if pred_std is not None:
                stds.append(pred_std)
            prev_prev_state, prev_state = prev_state, new_state
        return torch.stack(preds, dim=1), (torch.stack(stds, dim=1) if stds else None)

    # ---- inference fast path: one captured CUDA graph per (B, shapes) ----------------------
    @torch.no_grad()
    def capture(self, batch_size):
        """Capture the forecast step (predictor + boundary mix) into CUDA graphs operating on static buffers.
        The states live in a ring of three buffers — step k reads prev_prev = state[k%3], prev = state[(k+1)%3] and
        writes the new state into state[(k+2)%3] — so the autoregressive feedback costs no copies; the three
        rotations are three graphs sharing one memory pool.  Returns the dict of static buffers
        (``forcing``, ``boundary``, ``state``)."""
        p = self.predictor
        bufs = self._step_buffers(batch_size)
        p.static_embeddings()  # materialise the weight-only embeddings outside the graph
        graphs = self._capture_ring(lambda k: self._one_step(bufs, k))
        self._graph = (batch_size, graphs, bufs)
        # the graphs hold the cached static embeddings and every weight BY ADDRESS: remember what they were captured
        # against so that a later weight update / load_state_dict / .to() triggers a re-capture instead of a stale replay
        self._graph_key = self._capture_key(batch_size)
        self._graph_static = p._static_cache  # keeps the captured embedding tensors alive while the graphs exist
        self._phase = 0
        return bufs

    def _step_buffers(self, batch_size):
        """The static buffers of a captured step on ``batch_size`` rows: ``forcing``, ``boundary``, the ``state`` ring and,
        for a sampling predictor, ``latent_noise``."""
        p = self.predictor
        dev = self.boundary_mask.device
        G, d, f = p.num_grid_nodes, p.num_state_vars, p.grid_input_dim - 2 * p.num_state_vars - p.grid_static_features.shape[1]
        bufs = {"forcing": torch.zeros(batch_size, G, f, device=dev), "boundary": torch.zeros(batch_size, G, d, device=dev),
                "state": [torch.zeros(batch_size, G, d, device=dev) for _ in range(3)]}
        if getattr(p, "samples_latent", False):
            # a predictor that samples: every captured step first refills this buffer from the default generator of the
            # device, so each replay draws fresh noise and torch.cuda.manual_seed makes a sequence of replays reproducible
            bufs["latent_noise"] = torch.zeros(batch_size, p.latent_spatial_dim, p.latent_dim, device=dev)
        return bufs

    def _capture_ring(self, step):
        """Warm ``step(0)`` up twice on a side stream, then capture ``step(k)`` for the three rotations of the state ring
        into three CUDA graphs sharing one memory pool."""
        dev = self.boundary_mask.device
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(2):  # warm up allocator / lazy handles
                step(0)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        graphs = []
        for k in range(3):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=graphs[0].pool() if graphs else None):
                step(k)
            graphs.append(g)
        return graphs

    def _capture_key(self, batch_size):
        p = self.predictor
        return (batch_size, self.boundary_mask.device, p._static_param_version(),
                tuple(q.data_ptr() for q in p.parameters()))

    def _ensure_captured(self, batch_size):
        if self._graph is None or getattr(self, "_graph_key", None) != self._capture_key(batch_size):
            self._io = None
            self.capture(batch_size)

    def _one_step(self, bufs, k):
        st = bufs["state"]
        noise = bufs.get("latent_noise")
        if noise is None:
            return self.predictor.forward_with_boundary(st[(k + 1) % 3], st[k % 3], bufs["forcing"], bufs["boundary"],
                                                        self.boundary_mask, out=st[(k + 2) % 3])
        noise.normal_()
        return self.predictor.forward_with_boundary(st[(k + 1) % 3], st[k % 3], bufs["forcing"], bufs["boundary"],
                                                    self.boundary_mask, latent_noise=noise, out=st[(k + 2) % 3])

    def set_state(self, prev_prev_state, prev_state):
        """Load the two initial states into the captured step's state ring."""
        _, _, bufs = self._graph
        bufs["state"][0].copy_(prev_prev_state)
        bufs["state"][1].copy_(prev_state)
        self._phase = 0

    def replay_step(self):
        """Replay one captured forecast step on the static ``forcing`` / ``boundary`` buffers; returns the buffer
        holding the new state (valid until two further steps have been replayed)."""
        _, graphs, bufs = self._graph
        k = self._phase
        graphs[k].replay()
        self._phase = (k + 1) % 3
        return bufs["state"][(k + 2) % 3]

    @torch.no_grad()
    def rollout_graphed(self, init_states, forcing_features, boundary_states):
        """Same result as ``forward`` (no std), replaying the captured step graphs."""
        B, T = forcing_features.shape[0], forcing_features.shape[1]
        self._ensure_captured(B)
        _, _, bufs = self._graph
        out = torch.empty(B, T, *init_states.shape[2:], device=init_states.device)
        self.set_state(init_states[:, 0], init_states[:, 1])
        for i in range(T):
            bufs["forcing"].copy_(forcing_features[:, i])
            bufs["boundary"].copy_(boundary_states[:, i])
            out[:, i].copy_(self.replay_step())
        return out

    # ---- ensemble forecasts of a sampling predictor: K members per initial condition, reduced on the device ----------
    def _capture_ensemble(self, B, K, with_scores):
        """Capture the ensemble step for B initial conditions of K members: expand the step's forcing and boundary
        (B rows each) to the B·K member rows in one broadcast copy each, run the predictor step on the B·K rows with fresh
        noise (``_one_step``, as ``capture`` does) and reduce the new states with ``ens_stats_kernel``.  Kept apart from
        ``capture``'s graphs: neither evicts the other."""
        p = self.predictor
        dev = self.boundary_mask.device
        bufs = self._step_buffers(B * K)
        G, d, f = bufs["boundary"].shape[1], bufs["boundary"].shape[2], bufs["forcing"].shape[2]
        bufs.update({"ens_forcing": torch.zeros(B, G, f, device=dev), "ens_boundary": torch.zeros(B, G, d, device=dev),
                     "mean": torch.zeros(B, G, d, device=dev), "std": torch.zeros(B, G, d, device=dev)})
        if with_scores:
            bufs.update({"target": torch.zeros(B, G, d, device=dev), "scores": torch.zeros(B, d, 4, device=dev),
                         "workspace": torch.zeros(ensemble.workspace_bytes(B, G, d), dtype=torch.uint8, device=dev)})
        interior = self.interior_mask.reshape(-1).contiguous()

        def step(k):
            bufs["forcing"].view(B, K, G, f).copy_(bufs["ens_forcing"].unsqueeze(1).expand(B, K, G, f))
            bufs["boundary"].view(B, K, G, d).copy_(bufs["ens_boundary"].unsqueeze(1).expand(B, K, G, d))
            self._one_step(bufs, k)
            ensemble.launch(bufs["state"][(k + 2) % 3].view(B, K, G, d), interior, bufs["mean"], bufs["std"],
                            target=bufs.get("target"), scores=bufs.get("scores"), workspace=bufs.get("workspace"))

        p.static_embeddings()
        graphs = self._capture_ring(step)
        self._ens = {"key": (B, K, with_scores) + self._capture_key(B * K), "graphs": graphs, "bufs": bufs,
                     "static": p._static_cache, "interior": interior}

    @torch.no_grad()
    def rollout_ensemble(self, init_states, forcing_features, boundary_states, members, targets=None):
        """Ensemble forecast of a sampling predictor (Graph-EFM), reduced on the device: ``members`` forecasts per initial
        condition, each with its own latent noise, of which only the ensemble mean and spread are stored.

        ``init_states`` (B, 2, G, d), ``forcing_features`` (B, T, G, f), ``boundary_states`` (B, T, G, d) and the optional
        ``targets`` (B, T, G, d) are per initial condition, on the device.  Returns ``(mean, std, scores)``: mean and std
        (B, T, G, d) over the members (``ensemble.ensemble_stats``), and with ``targets`` an ``ensemble.EnsembleScores`` of
        (B, T, d) interior-grid means, else None.  In the reference's evaluation loop the targets are the boundary tensor
        (module.py:389-391), so the same tensor may be passed twice.

        Each step replays one captured graph: the member expansion of that step's forcing and boundary, the predictor step
        on B·members rows with fresh noise per replay (as ``rollout_graphed`` draws it: after the same
        ``torch.cuda.manual_seed`` the members are ``rollout_graphed``'s rows on the inputs expanded to B·members rows) and
        ``ens_stats_kernel``.  Only B rows of forcing and boundary enter per step."""
        p = self.predictor
        if not getattr(p, "samples_latent", False):
            raise ValueError(f"rollout_ensemble needs a predictor that samples its latent (Graph-EFM), got {type(p).__name__}")
        if isinstance(members, bool) or not isinstance(members, int) or not 2 <= members <= ensemble.MAX_MEMBERS:
            raise ValueError(f"rollout_ensemble: members must be an int in 2 .. {ensemble.MAX_MEMBERS}, got {members!r}")
        G, d = p.num_grid_nodes, p.num_state_vars
        if forcing_features.dim() != 4 or forcing_features.shape[2] != G:
            raise ValueError(f"forcing_features: expected (B, T, {G}, f), got {tuple(forcing_features.shape)}")
        B, T = forcing_features.shape[0], forcing_features.shape[1]
        want = {"init_states": (init_states, (B, 2, G, d)), "boundary_states": (boundary_states, (B, T, G, d))}
        if targets is not None:
            want["targets"] = (targets, (B, T, G, d))
        for name, (t, shape) in want.items():
            if tuple(t.shape) != shape:
                raise ValueError(f"{name}: expected shape {shape}, got {tuple(t.shape)}")
        K, with_scores = members, targets is not None
        ens = getattr(self, "_ens", None)
        if ens is None or ens["key"] != (B, K, with_scores) + self._capture_key(B * K):
            self._capture_ensemble(B, K, with_scores)
        graphs, bufs = self._ens["graphs"], self._ens["bufs"]
        dev = init_states.device
        mean = torch.empty(B, T, G, d, device=dev)
        std = torch.empty(B, T, G, d, device=dev)
        scores = torch.empty(B, T, d, 4, device=dev) if with_scores else None
        st = bufs["state"]
        st[0].view(B, K, G, d).copy_(init_states[:, 0].unsqueeze(1).expand(B, K, G, d))
        st[1].view(B, K, G, d).copy_(init_states[:, 1].unsqueeze(1).expand(B, K, G, d))
        for i in range(T):
            bufs["ens_forcing"].copy_(forcing_features[:, i])
            bufs["ens_boundary"].copy_(boundary_states[:, i])
            if with_scores:
                bufs["target"].copy_(targets[:, i])
            graphs[i % 3].replay()
            mean[:, i].copy_(bufs["mean"])
            std[:, i].copy_(bufs["std"])
            if with_scores:
                scores[:, i].copy_(bufs["scores"])
        return mean, std, (ensemble.EnsembleScores.from_means(scores, K) if with_scores else None)

    @torch.no_grad()
    def host_io_bytes_per_step(self, B):
        """(host->device, device->host) bytes ``rollout_from_host`` moves per AR step of B forecasts: the forcing, the rows of
        the boundary state the boundary mask selects, and the prediction."""
        self._ensure_captured(B)
        _, _, bufs = self._graph
        G, d_state = bufs["boundary"].shape[1], bufs["boundary"].shape[2]
        blocks = _boundary_blocks(self.boundary_mask)
        bnd_rows = G if blocks is None else sum(rlen * count for _, rlen, _, count in blocks)
        return B * (G * bufs["forcing"].shape[2] + bnd_rows * d_state) * 4, B * G * d_state * 4

    def rollout_from_host(self, init_states, forcing_features, boundary_states, out=None):
        """Inference rollout with HOST tensors (ideally pinned).  Every AR step copies that step's
        forcing + boundary states host->device, replays the captured step graph and copies the
        predicted state device->host.  The PCIe transfers run on their own streams, double
        buffered, so that H2D of step i+1 and D2H of step i-1 overlap the kernels of step i;
        nothing synchronises with the host until the end.  Shapes as in ``forward``; returns the
        (B,T,G,d) prediction on the host (``out`` if given)."""
        B, T = forcing_features.shape[0], forcing_features.shape[1]
        dev = self.boundary_mask.device
        self._ensure_captured(B)
        _, _, bufs = self._graph
        if out is None:
            out = torch.empty(B, T, *init_states.shape[2:], dtype=torch.float32, pin_memory=True)
        if getattr(self, "_io", None) is None or self._io["B"] != B:
            self._io = {
                "B": B, "s_in": torch.cuda.Stream(device=dev), "s_out": torch.cuda.Stream(device=dev),
                "forc": [torch.empty_like(bufs["forcing"]) for _ in range(2)],
                # zero-filled: with a compact boundary transfer the interior rows are never written (and multiplied by a
                # zero mask in the step epilogue)
                "bnd": [torch.zeros_like(bufs["boundary"]) for _ in range(2)],
                "out": [torch.empty_like(bufs["boundary"]) for _ in range(2)],
                "bnd_blocks": _boundary_blocks(self.boundary_mask),
            }
        io = self._io
        main = torch.cuda.current_stream(dev)
        s_in, s_out = io["s_in"], io["s_out"]
        s_in.wait_stream(main)
        s_out.wait_stream(main)
        in_ready = [torch.cuda.Event() for _ in range(2)]
        in_free = [torch.cuda.Event() for _ in range(2)]
        out_ready = [torch.cuda.Event() for _ in range(2)]
        out_free = [torch.cuda.Event() for _ in range(2)]

        def copy_step(dev_t, host_t, i, stream, to_device):
            """step-i slice of a (B, T, G, F) host tensor <-> a dense (B, G, F) device tensor: ONE strided copy"""
            row = host_t.shape[2] * host_t.shape[3] * 4
            hp = host_t.data_ptr() + i * row
            args = (dev_t.data_ptr(), row, hp, host_t.stride(0) * 4) if to_device else (hp, host_t.stride(0) * 4, dev_t.data_ptr(), row)
            _lib.check(_lib.lib().nlam_memcpy2d_async(*args, row, B, 1 if to_device else 0, ctypes.c_void_p(stream.cuda_stream)))

        def sliceable(t):  # (B, T, G, F) with dense (G, F) blocks, steps G*F apart: slices along T of a dense tensor qualify
            return (t.dtype == torch.float32 and not t.is_cuda and t.dim() == 4 and t.stride(3) == 1
                    and t.stride(2) == t.shape[3] and t.stride(1) == t.shape[2] * t.shape[3]
                    and t.stride(0) % (t.shape[2] * t.shape[3]) == 0)

        dense = all(sliceable(t) for t in (forcing_features, boundary_states, out))

        def copy_boundary(dev_t, host_t, i, stream):
            """only the rows the boundary mask selects (new = mask*boundary + (1-mask)*prediction never reads the others):
            the blocks of ``_boundary_blocks`` — a run of nodes per sample, or equally spaced runs (the strips left and
            right of the interior) as one 3-D copy"""
            Bh, Th, G, F = host_t.shape
            L = _lib.lib()
            sp = ctypes.c_void_p(stream.cuda_stream)
            for start, rlen, pitch, count in io["bnd_blocks"]:
                hp = host_t.data_ptr() + (i * G + start) * F * 4
                dp = dev_t.data_ptr() + start * F * 4
                if count == 1:
                    _lib.check(L.nlam_memcpy2d_async(dp, G * F * 4, hp, host_t.stride(0) * 4, rlen * F * 4, Bh, 1, sp))
                else:
                    _lib.check(L.nlam_memcpy3d_async(dp, pitch * F * 4, G // pitch, hp, pitch * F * 4,
                                                     host_t.stride(0) // (pitch * F), rlen * F * 4, count, Bh, 1, sp))

        def h2d(i):
            k = i & 1
            with torch.cuda.stream(s_in):
                if i >= 2:
                    s_in.wait_event(in_free[k])
                if dense:
                    copy_step(io["forc"][k], forcing_features, i, s_in, True)
                    if io["bnd_blocks"] is not None:
                        copy_boundary(io["bnd"][k], boundary_states, i, s_in)
                    else:
                        copy_step(io["bnd"][k], boundary_states, i, s_in, True)
                else:
                    for b in range(B):  # per-sample slices of (B,T,G,F) host tensors are contiguous
                        io["forc"][k][b].copy_(forcing_features[b, i], non_blocking=True)
                        io["bnd"][k][b].copy_(boundary_states[b, i], non_blocking=True)
                in_ready[k].record(s_in)

        for b in range(B):
            bufs["state"][0][b].copy_(init_states[b, 0], non_blocking=True)
            bufs["state"][1][b].copy_(init_states[b, 1], non_blocking=True)
        self._phase = 0
        h2d(0)
        for i in range(T):
            k = i & 1
            if i + 1 < T:
                h2d(i + 1)
            main.wait_event(in_ready[k])
            bufs["forcing"].copy_(io["forc"][k])
            bufs["boundary"].copy_(io["bnd"][k])
            in_free[k].record(main)
            new_state = self.replay_step()
            if i >= 2:
                main.wait_event(out_free[k])
            io["out"][k].copy_(new_state)
            out_ready[k].record(main)
            with torch.cuda.stream(s_out):
                s_out.wait_event(out_ready[k])
                if dense:
                    copy_step(io["out"][k], out, i, s_out, False)
                else:
                    for b in range(B):
                        out[b, i].copy_(io["out"][k][b], non_blocking=True)
                out_free[k].record(s_out)
        main.wait_stream(s_out)
        main.wait_stream(s_in)
        main.synchronize()
        return out
