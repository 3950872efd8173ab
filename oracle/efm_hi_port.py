"""CPU restatement (oracle) of the Graph-EFM step on a HIERARCHICAL mesh (the reference's ``GraphEFM``) with an explicit
noise sample.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  Built from ``reference_port.mlp`` / ``interaction_net`` and the
flat-mesh helpers of ``oracle/efm_port.py`` (grid embedding, ``mean_std``), so it runs in fp32, fp64, under
``reference_port.tf32_matmul()`` and on the GPU; parameters are a flat ``{state_dict key: tensor}`` dict of
``models.GraphEFM``.
"""
import torch

from .efm_port import _cast, _gnn, grid_embedding, mean_std
from .reference_port import _expand, clamped_new_state, mlp

# Reference files (neural_lam/models/...): step_predictors/graph/graph_efm.py (GraphEFM.embedd_mesh :746-793),
# latent/hi_graph_encoder.py:148-175, latent/hi_graph_decoder.py:216-270.  ``graph`` holds the per-level lists
# ``mesh_static_features``, ``m2m_features`` / ``m2m_edge_index``, ``mesh_up_*`` and ``mesh_down_*`` of the model's buffers;
# ``cfg``: dict(hidden_layers, prior_intra_level_layers, encoder_intra_level_layers, decoder_intra_level_layers, learn_prior,
# prior_dist, g2m_gnn_type, m2g_gnn_type, output_std, clamp, num_top_nodes, latent_dim).


def _cast_hi(graph, dt):
    return {k: ([t.to(dt) if t.is_floating_point() else t for t in v] if isinstance(v, (list, tuple)) else v)
            for k, v in _cast(graph, dt).items()}


def hi_static_embeddings(params, g, cfg):
    """graph_efm.py:364-413 (g2m, m2g) and :746-793 (per level; ``m2m`` empty without ``m2m_embedders``)"""
    hl = cfg.get("hidden_layers", 1)
    st = {"g2m": mlp(g["g2m_features"], params, "g2m_embedder", hl), "m2g": mlp(g["m2g_features"], params, "m2g_embedder", hl)}
    for k, emb, feats in (("mesh", "mesh_embedders", "mesh_static_features"), ("mesh_up", "mesh_up_embedders", "mesh_up_features"),
                          ("mesh_down", "mesh_down_embedders", "mesh_down_features"), ("m2m", "m2m_embedders", "m2m_features")):
        st[k] = [mlp(f, params, f"{emb}.{l}", hl) for l, f in enumerate(g[feats]) if f"{emb}.{l}.0.weight" in params]
    return st


def _intra(params, prefix, ei, mesh, edge, layers, hl):
    """``make_gnn_seq`` stack of ``layers`` InteractionNets over one level -> (mesh, edge) (utils/networks.py:93-106)"""
    for i in range(layers):
        mesh, edge = _gnn(params, f"{prefix}.module_{i}", ei, mesh, mesh, edge, hl)
    return mesh, edge


def hi_graph_latent_encoder(params, prefix, g, cfg, grid_rep, st, layers, dist):
    """HiGraphLatentEncoder -> (mean, std) on the top level (hi_graph_encoder.py:148-175)."""
    hl, B = cfg.get("hidden_layers", 1), grid_rep.shape[0]
    mesh = _gnn(params, f"{prefix}.g2m_gnn", g["g2m_edge_index"], grid_rep, _expand(st["mesh"][0], B), _expand(st["g2m"], B), hl,
                cfg.get("g2m_gnn_type", "InteractionNet"), update_edges=False)
    mesh, _ = _intra(params, f"{prefix}.intra_level_gnns.0", g["m2m_edge_index"][0], mesh,
                     _expand(st["m2m"][0], B) if layers else None, layers, hl)
    for level in range(1, len(g["mesh_static_features"])):
        mesh = _gnn(params, f"{prefix}.mesh_up_gnns.{level - 1}", g["mesh_up_edge_index"][level - 1], mesh,
                    _expand(st["mesh"][level], B), _expand(st["mesh_up"][level - 1], B), hl, "PropagationNet",
                    update_edges=False)
        mesh, _ = _intra(params, f"{prefix}.intra_level_gnns.{level}", g["m2m_edge_index"][level], mesh,
                         _expand(st["m2m"][level], B) if layers else None, layers, hl)
    return mean_std(mlp(mesh, params, f"{prefix}.latent_param_map", hl, layer_norm=False), dist)


def hi_prior(params, g, cfg, grid_emb, st):
    """the prior's (mean, std) on the top level: HiGraphLatentEncoder, or the constant prior's zeros through ``mean_std``"""
    if cfg.get("learn_prior", True):
        return hi_graph_latent_encoder(params, "prior_model", g, cfg, grid_emb, st, cfg["prior_intra_level_layers"],
                                       cfg.get("prior_dist", "isotropic"))
    z = grid_emb.new_zeros(grid_emb.shape[0], cfg["num_top_nodes"],
                           cfg["latent_dim"] * (2 if cfg.get("prior_dist") == "diagonal" else 1))
    return mean_std(z, cfg.get("prior_dist", "isotropic"))


def hi_decoder(params, g, cfg, grid_emb, z, st):
    """HiGraphLatentDecoder -> (mean_delta, pred_std|None) (base_decoder.py:145-171, hi_graph_decoder.py:216-270)."""
    hl, B = cfg.get("hidden_layers", 1), grid_emb.shape[0]
    layers = cfg["decoder_intra_level_layers"]
    L = len(g["mesh_static_features"])
    latent_emb = mlp(z, params, "decoder.latent_embedder", hl)
    res_grid = grid_emb + mlp(grid_emb, params, "decoder.grid_update_mlp", hl)
    # g2m onto the static level-0 embedding (hi_graph_decoder.py:216-218)
    mesh = _gnn(params, "decoder.g2m_gnn", g["g2m_edge_index"], grid_emb, _expand(st["mesh"][0], B), _expand(st["g2m"], B), hl,
                cfg.get("g2m_gnn_type", "InteractionNet"), update_edges=False)
    # up sweep; the last up-step's receivers are the embedded latent (:223-245)
    receivers = [_expand(m, B) for m in st["mesh"][1:-1]] + [latent_emb]
    levels, edges = [], []
    for level in range(L - 1):
        mesh, edge = _intra(params, f"decoder.intra_up_gnns.{level}", g["m2m_edge_index"][level], mesh,
                            _expand(st["m2m"][level], B) if layers else None, layers, hl)
        levels.append(mesh)
        edges.append(edge)
        mesh = _gnn(params, f"decoder.mesh_up_gnns.{level}", g["mesh_up_edge_index"][level], mesh, receivers[level],
                    _expand(st["mesh_up"][level], B), hl, update_edges=False)
    # top level (:247-251)
    mesh, _ = _intra(params, f"decoder.intra_up_gnns.{L - 1}", g["m2m_edge_index"][L - 1], mesh,
                     _expand(st["m2m"][L - 1], B) if layers else None, layers, hl)
    # down sweep onto the up sweep's representations (:253-264)
    for level in reversed(range(L - 1)):
        mesh = _gnn(params, f"decoder.mesh_down_gnns.{level}", g["mesh_down_edge_index"][level], mesh, levels[level],
                    _expand(st["mesh_down"][level], B), hl, "PropagationNet", update_edges=False)
        mesh, _ = _intra(params, f"decoder.intra_down_gnns.{level}", g["m2m_edge_index"][level], mesh, edges[level], layers, hl)
    grid = _gnn(params, "decoder.m2g_gnn", g["m2g_edge_index"], mesh, res_grid, _expand(st["m2g"], B), hl,
                cfg.get("m2g_gnn_type", "InteractionNet"), update_edges=False)
    out = mlp(grid, params, "decoder.param_map", hl, layer_norm=False)
    if cfg.get("output_std"):
        mean_delta, raw = out.chunk(2, dim=-1)
        return mean_delta, torch.nn.functional.softplus(raw)
    return out, None


def efm_hi_step(params, graph, cfg, prev_state, prev_prev_state, forcing, eps):
    """One ``GraphEFM.forward`` with the prior sample ``z = mean + eps * std`` on the top level ->
    dict(pred, pred_std, prior_mean, prior_std, z)."""
    dt = prev_state.dtype
    g = _cast_hi(graph, dt)
    st = hi_static_embeddings(params, g, cfg)
    grid_emb = grid_embedding(params, g, cfg, prev_state, prev_prev_state, forcing)
    mean, std = hi_prior(params, g, cfg, grid_emb, st)
    z = mean + eps.to(dt) * std
    mean_delta, pred_std = hi_decoder(params, g, cfg, grid_emb, z, st)
    delta = mean_delta * g["diff_std"] + g["diff_mean"]
    clamp = cfg.get("clamp")
    if clamp:
        pred = clamped_new_state(delta, prev_state, clamp["names"], clamp["lower"], clamp["upper"], clamp["state_mean"].to(dt),
                                 clamp["state_std"].to(dt))
    else:
        pred = prev_state + delta
    return dict(pred=pred, pred_std=pred_std, prior_mean=mean, prior_std=std, z=z)


def efm_hi_posterior(params, graph, cfg, prev_state, prev_prev_state, forcing, target):
    """GraphEFM's variational encoder's (mean, std) given the target X_{t+1} (graph_efm.py:301-343, ``"diagonal"``)."""
    g = _cast_hi(graph, prev_state.dtype)
    st = hi_static_embeddings(params, g, cfg)
    grid_cur = grid_embedding(params, g, cfg, prev_state, prev_prev_state, forcing, target=target)
    return hi_graph_latent_encoder(params, "encoder", g, cfg, grid_cur, st, cfg["encoder_intra_level_layers"], "diagonal")
