"""Latent encoders and decoders of Graph-EFM on a flat and on a hierarchical mesh, with the reference's structure, parameter
names and forward semantics (reference neural_lam/models/latent/: base_encoder.py, graph_encoder.py, constant_encoder.py,
base_decoder.py, graph_decoder.py, hi_graph_encoder.py, hi_graph_decoder.py).  The modules hold parameters and compose the
library's MLP, InteractionNet and PropagationNet kernels; the fused inference steps of ``models.GraphEFMMultiScale`` and
``models.GraphEFM`` reach into them (``latent_param_map``, ``latent_embedder``, ...).
"""
import torch
from torch import distributions as tdists
from torch import nn

from .gnn_layers import InteractionNet, PropagationNet, get_gnn_class
from .networks import GNNSequential, make_mlp


def _m2m_stack(edge_index, m2m_layers, hidden_layers, hidden_dim, math):
    """``make_gnn_seq`` of the reference (utils/networks.py:43-106) with the model's math mode; None for no layers."""
    if m2m_layers <= 0:
        return None
    return GNNSequential([InteractionNet(edge_index, hidden_dim, hidden_layers=hidden_layers, math=math)
                         for _ in range(m2m_layers)])


class BaseLatentEncoder(nn.Module):
    """Maps a grid representation to a Gaussian over a latent variable on mesh nodes (reference base_encoder.py:9-94):
    ``"isotropic"`` outputs the mean (unit std), ``"diagonal"`` the mean and ``1e-4 + softplus(raw)``."""

    def __init__(self, latent_dim, output_dist="isotropic"):
        super().__init__()
        self.output_dist = output_dist
        if output_dist == "isotropic":
            self.output_dim = latent_dim
        elif output_dist == "diagonal":
            self.output_dim = 2 * latent_dim
            self.latent_std_eps = 1e-4
        else:
            raise ValueError(f"Unknown encoder output distribution: {output_dist}")

    def compute_dist_params(self, grid_rep, *args, **kwargs):
        raise NotImplementedError("compute_dist_params not implemented")

    def mean_std(self, dist_params):
        """Raw parameters (..., output_dim) -> (mean, std), as ``forward`` builds its Normal."""
        if self.output_dist == "diagonal":
            mean, std_raw = dist_params.chunk(2, dim=-1)
            return mean, self.latent_std_eps + nn.functional.softplus(std_raw)
        return dist_params, torch.ones_like(dist_params)

    def forward(self, grid_rep, **kwargs):
        """-> ``torch.distributions.Normal`` with batch shape (B, num_mesh_nodes, latent_dim)."""
        return tdists.Normal(*self.mean_std(self.compute_dist_params(grid_rep, **kwargs)))


class GraphLatentEncoder(BaseLatentEncoder):
    """g2m GNN, ``m2m_layers`` on-mesh InteractionNets (None for 0) and ``latent_param_map`` (Linear-SiLU-Linear, no
    LayerNorm) on a flat graph (reference graph_encoder.py:11-105)."""

    def __init__(self, latent_dim, g2m_edge_index, m2m_edge_index, hidden_dim, m2m_layers, hidden_layers=1,
                 g2m_gnn_type="InteractionNet", output_dist="isotropic", math=None):
        super().__init__(latent_dim, output_dist)
        self.g2m_gnn = get_gnn_class(g2m_gnn_type)(g2m_edge_index, hidden_dim, hidden_layers=hidden_layers,
                                                   update_edges=False, math=math)
        self.m2m_gnns = _m2m_stack(m2m_edge_index, m2m_layers, hidden_layers, hidden_dim, math)
        self.latent_param_map = make_mlp([hidden_dim] * (hidden_layers + 1) + [self.output_dim], layer_norm=False)

    def process_mesh(self, mesh_rep, m2m_emb):
        """The on-mesh stack (identity without one); the final edge representation is discarded."""
        if self.m2m_gnns is not None:
            mesh_rep, _ = self.m2m_gnns(mesh_rep, m2m_emb, keep_edge_rep=False)
        return mesh_rep

    def compute_dist_params(self, grid_rep, graph_emb, **kwargs):
        """graph_emb: ``mesh`` (B, N_mesh, H), ``g2m`` (B, M_g2m, H), ``m2m`` (B, M_m2m, H) -> (B, N_mesh, output_dim)"""
        mesh_rep = self.g2m_gnn(grid_rep, graph_emb["mesh"], graph_emb["g2m"])
        return self.latent_param_map(self.process_mesh(mesh_rep, graph_emb["m2m"]))


class ConstantLatentEncoder(BaseLatentEncoder):
    """Input-independent prior: zero raw parameters, i.e. N(0, 1) (isotropic) or N(0, 1e-4 + softplus(0)) (diagonal)
    (reference constant_encoder.py:10-62)."""

    def __init__(self, latent_dim, num_mesh_nodes, output_dist="isotropic"):
        super().__init__(latent_dim, output_dist)
        self.num_mesh_nodes = num_mesh_nodes

    def compute_dist_params(self, grid_rep, **kwargs):
        return torch.zeros(grid_rep.shape[0], self.num_mesh_nodes, self.output_dim, device=grid_rep.device)


class BaseGraphLatentDecoder(nn.Module):
    """The decoder's grid-side MLPs: ``grid_update_mlp`` (residual update of the grid representation, the m2g receivers),
    ``latent_embedder`` and ``param_map`` (reference base_decoder.py:10-171).  Subclasses define ``combine_with_latent``."""

    def __init__(self, hidden_dim, latent_dim, num_state_vars, hidden_layers=1, output_std=True):
        super().__init__()
        self.grid_update_mlp = make_mlp([hidden_dim] * (hidden_layers + 2))
        self.latent_embedder = make_mlp([latent_dim] + [hidden_dim] * (hidden_layers + 1))
        self.output_std = output_std
        output_dim = 2 * num_state_vars if output_std else num_state_vars
        self.param_map = make_mlp([hidden_dim] * (hidden_layers + 1) + [output_dim], layer_norm=False)

    def combine_with_latent(self, original_grid_rep, latent_rep, residual_grid_rep, graph_emb):
        raise NotImplementedError("combine_with_latent not implemented")

    def forward(self, grid_rep, latent_samples, graph_emb):
        """-> (mean_delta (B, G, d_state), pred_std (B, G, d_state) or None)"""
        latent_emb = self.latent_embedder(latent_samples)
        residual_grid_rep = self.grid_update_mlp.apply_rows([grid_rep], res=grid_rep)
        state_params = self.param_map(self.combine_with_latent(grid_rep, latent_emb, residual_grid_rep, graph_emb))
        if self.output_std:
            mean_delta, std_raw = state_params.chunk(2, dim=-1)
            return mean_delta, nn.functional.softplus(std_raw)
        return state_params, None


class GraphLatentDecoder(BaseGraphLatentDecoder):
    """Grid representation + latent sample on the mesh -> next-state increment (and std) on the grid, through g2m (the
    embedded latent as receivers), ``m2m_layers`` on-mesh InteractionNets and m2g onto ``grid_rep + grid_update_mlp(grid_rep)``
    (reference base_decoder.py:10-171, graph_decoder.py:11-134)."""

    def __init__(self, g2m_edge_index, m2m_edge_index, m2g_edge_index, hidden_dim, latent_dim, num_state_vars, m2m_layers,
                 hidden_layers=1, g2m_gnn_type="InteractionNet", m2g_gnn_type="InteractionNet", output_std=True, math=None):
        super().__init__(hidden_dim, latent_dim, num_state_vars, hidden_layers=hidden_layers, output_std=output_std)
        self.g2m_gnn = get_gnn_class(g2m_gnn_type)(g2m_edge_index, hidden_dim, hidden_layers=hidden_layers,
                                                   update_edges=False, math=math)
        self.m2m_gnns = _m2m_stack(m2m_edge_index, m2m_layers, hidden_layers, hidden_dim, math)
        self.m2g_gnn = get_gnn_class(m2g_gnn_type)(m2g_edge_index, hidden_dim, hidden_layers=hidden_layers,
                                                   update_edges=False, math=math)

    def mesh_step(self, grid_rep, latent_emb, graph_emb):
        """g2m (senders grid_rep, receivers the embedded latent) and the on-mesh stack -> mesh representation."""
        mesh_rep = self.g2m_gnn(grid_rep, latent_emb, graph_emb["g2m"])
        if self.m2m_gnns is not None:
            mesh_rep, _ = self.m2m_gnns(mesh_rep, graph_emb["m2m"], keep_edge_rep=False)
        return mesh_rep

    def combine_with_latent(self, original_grid_rep, latent_rep, residual_grid_rep, graph_emb):
        return self.m2g_gnn(self.mesh_step(original_grid_rep, latent_rep, graph_emb), residual_grid_rep, graph_emb["m2g"])


def _check_levels(cls, m2m_edge_index):
    if len(m2m_edge_index) < 2:
        flat = "GraphLatentEncoder" if cls == "HiGraphLatentEncoder" else "GraphLatentDecoder"
        raise ValueError(f"{cls} requires at least 2 mesh levels (got {len(m2m_edge_index)}). Use {flat} for flat graphs.")


def _level_stacks(edge_indices, layers, hidden_layers, hidden_dim, math):
    """One intra-level stack per edge set, or None for no layers (reference hi_graph_encoder.py:101-115)."""
    if layers <= 0:
        return None
    return nn.ModuleList([_m2m_stack(ei, layers, hidden_layers, hidden_dim, math) for ei in edge_indices])


class HiGraphLatentEncoder(BaseLatentEncoder):
    """Latent encoder on a hierarchical mesh: g2m onto level 0, then up the hierarchy with PropagationNets
    (``mesh_up_gnns``), each level followed by ``intra_level_layers`` InteractionNets (``intra_level_gnns``, None for 0);
    the distribution is read out on the top level by ``latent_param_map`` (reference hi_graph_encoder.py:14-175)."""

    def __init__(self, latent_dim, g2m_edge_index, m2m_edge_index, mesh_up_edge_index, hidden_dim, intra_level_layers,
                 hidden_layers=1, g2m_gnn_type="InteractionNet", output_dist="isotropic", math=None):
        super().__init__(latent_dim, output_dist)
        _check_levels("HiGraphLatentEncoder", m2m_edge_index)
        self.g2m_gnn = get_gnn_class(g2m_gnn_type)(g2m_edge_index, hidden_dim, hidden_layers=hidden_layers,
                                                   update_edges=False, math=math)
        self.mesh_up_gnns = nn.ModuleList([
            PropagationNet(ei, hidden_dim, hidden_layers=hidden_layers, update_edges=False, math=math)
            for ei in mesh_up_edge_index])
        self.intra_level_gnns = _level_stacks(list(m2m_edge_index), intra_level_layers, hidden_layers, hidden_dim, math)
        self.latent_param_map = make_mlp([hidden_dim] * (hidden_layers + 1) + [self.output_dim], layer_norm=False)

    def _intra(self, level, mesh_rep, graph_emb):
        if self.intra_level_gnns is not None:
            mesh_rep, _ = self.intra_level_gnns[level](mesh_rep, graph_emb["m2m"][level], keep_edge_rep=False)
        return mesh_rep

    def process_mesh(self, mesh_rep, graph_emb):
        """Level-0 representation after g2m -> top-level representation: the intra-level stack of level 0, then per level
        the up-step and that level's stack (hi_graph_encoder.py:152-173)."""
        mesh_rep = self._intra(0, mesh_rep, graph_emb)
        for level, up_gnn in enumerate(self.mesh_up_gnns, start=1):
            mesh_rep = up_gnn(mesh_rep, graph_emb["mesh"][level], graph_emb["mesh_up"][level - 1])
            mesh_rep = self._intra(level, mesh_rep, graph_emb)
        return mesh_rep

    def compute_dist_params(self, grid_rep, graph_emb, **kwargs):
        """graph_emb: ``mesh``, ``m2m``, ``mesh_up`` lists over levels, ``g2m`` -> (B, N_top, output_dim)"""
        mesh_rep = self.g2m_gnn(grid_rep, graph_emb["mesh"][0], graph_emb["g2m"])
        return self.latent_param_map(self.process_mesh(mesh_rep, graph_emb))


class HiGraphLatentDecoder(BaseGraphLatentDecoder):
    """Latent decoder on a hierarchical mesh: g2m onto the static level-0 embedding, an up sweep (intra-level stack, then
    an InteractionNet up-step; the last up-step's receivers are the embedded latent on the top level), the top level's
    stack, a down sweep (PropagationNet down-step onto the up sweep's level representation, then the intra-level stack on
    the up sweep's edge representation of that level) and m2g (reference hi_graph_decoder.py:18-270)."""

    def __init__(self, g2m_edge_index, m2m_edge_index, m2g_edge_index, mesh_up_edge_index, mesh_down_edge_index, hidden_dim,
                 latent_dim, num_state_vars, intra_level_layers, hidden_layers=1, g2m_gnn_type="InteractionNet",
                 m2g_gnn_type="InteractionNet", output_std=True, math=None):
        super().__init__(hidden_dim, latent_dim, num_state_vars, hidden_layers=hidden_layers, output_std=output_std)
        _check_levels("HiGraphLatentDecoder", m2m_edge_index)
        self.g2m_gnn = get_gnn_class(g2m_gnn_type)(g2m_edge_index, hidden_dim, hidden_layers=hidden_layers,
                                                   update_edges=False, math=math)
        self.m2g_gnn = get_gnn_class(m2g_gnn_type)(m2g_edge_index, hidden_dim, hidden_layers=hidden_layers,
                                                   update_edges=False, math=math)
        self.mesh_up_gnns = nn.ModuleList([
            InteractionNet(ei, hidden_dim, hidden_layers=hidden_layers, update_edges=False, math=math)
            for ei in mesh_up_edge_index])
        self.mesh_down_gnns = nn.ModuleList([
            PropagationNet(ei, hidden_dim, hidden_layers=hidden_layers, update_edges=False, math=math)
            for ei in mesh_down_edge_index])
        m2m = list(m2m_edge_index)
        self.intra_up_gnns = _level_stacks(m2m, intra_level_layers, hidden_layers, hidden_dim, math)
        self.intra_down_gnns = _level_stacks(m2m[:-1], intra_level_layers, hidden_layers, hidden_dim, math)

    def mesh_step(self, mesh_rep, latent_emb, graph_emb):
        """Level-0 representation after g2m + embedded latent -> level-0 representation after the down sweep
        (hi_graph_decoder.py:220-264).  The up sweep's edge representations go to the down sweep's stacks; in no-grad mode
        the up stacks keep them on the stacked path (``GNNSequential(keep_stacked=True)``)."""
        levels, edges = [], []
        receivers = list(graph_emb["mesh"][1:-1]) + [latent_emb]
        for level, (up_gnn, up_emb, rec) in enumerate(zip(self.mesh_up_gnns, graph_emb["mesh_up"], receivers)):
            edge_rep = None
            if self.intra_up_gnns is not None:
                mesh_rep, edge_rep = self.intra_up_gnns[level](mesh_rep, graph_emb["m2m"][level], keep_stacked=True)
            levels.append(mesh_rep)
            edges.append(edge_rep)
            mesh_rep = up_gnn(mesh_rep, rec, up_emb)
        if self.intra_up_gnns is not None:
            mesh_rep, _ = self.intra_up_gnns[-1](mesh_rep, graph_emb["m2m"][-1], keep_edge_rep=False)
        for level in reversed(range(len(self.mesh_down_gnns))):
            mesh_rep = self.mesh_down_gnns[level](mesh_rep, levels[level], graph_emb["mesh_down"][level])
            if self.intra_down_gnns is not None:
                mesh_rep, _ = self.intra_down_gnns[level](mesh_rep, edges[level], keep_edge_rep=False)
        return mesh_rep

    def combine_with_latent(self, original_grid_rep, latent_rep, residual_grid_rep, graph_emb):
        mesh_rep = self.g2m_gnn(original_grid_rep, graph_emb["mesh"][0], graph_emb["g2m"])
        return self.m2g_gnn(self.mesh_step(mesh_rep, latent_rep, graph_emb), residual_grid_rep, graph_emb["m2g"])
