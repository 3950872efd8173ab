"""CPU restatement (oracle) of the Graph-EFM step on a flat mesh with an explicit noise sample.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  Built from ``reference_port.mlp`` / ``interaction_net`` (so it runs
in fp32, fp64 and under ``reference_port.tf32_matmul()``); parameters are a flat ``{state_dict key: tensor}`` dict of
``GraphEFMMultiScale``.  Reference files (neural_lam/models/...): step_predictors/graph/graph_efm.py (embedding :364-413,
forward :415-471, target embedding :301-343), latent/graph_encoder.py:102-105, latent/base_encoder.py:85-94,
latent/constant_encoder.py:57-62, latent/base_decoder.py:145-171, latent/graph_decoder.py:127-134.

``graph``: the tensors the model registers (``g2m_edge_index``, ``m2m_features``, ``diff_std``, ...); ``cfg``: dict(
hidden_layers, prior_m2m_layers, encoder_m2m_layers, decoder_m2m_layers, learn_prior, prior_dist, g2m_gnn_type,
m2g_gnn_type, output_std, clamp (as in reference_port.graph_model_forward), num_mesh_nodes, latent_dim).
"""
import torch

from .reference_port import _expand, clamped_new_state, interaction_net, mlp


def _cast(graph, dt):
    return {k: (v.to(dt) if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in graph.items()}


def _gnn(params, prefix, ei, send, rec, edge, hl, gnn_type="InteractionNet", update_edges=True):
    return interaction_net(params, ei, send, rec, edge, prefix=prefix, hidden_layers=hl, update_edges=update_edges,
                           propagation=(gnn_type == "PropagationNet"))


def static_embeddings(params, g, cfg):
    hl = cfg.get("hidden_layers", 1)
    return {k: mlp(g[f"{src}"], params, f"{k}_embedder", hl)
            for k, src in (("g2m", "g2m_features"), ("m2g", "m2g_features"), ("mesh", "mesh_static_features"),
                           ("m2m", "m2m_features"))}


def grid_embedding(params, g, cfg, prev_state, prev_prev_state, forcing, target=None):
    """grid_prev_embedder (or grid_current_embedder with the target appended) on the EFM-order concatenation."""
    B = prev_state.shape[0]
    feats = [prev_prev_state, prev_state, forcing, _expand(g["grid_static_features"], B)]
    name = "grid_prev_embedder"
    if target is not None:
        feats.append(target)
        name = "grid_current_embedder"
    return mlp(torch.cat(feats, dim=-1), params, name, cfg.get("hidden_layers", 1))


def mean_std(dist_params, dist):
    """base_encoder.py:85-94"""
    if dist == "diagonal":
        mean, raw = dist_params.chunk(2, dim=-1)
        return mean, 1e-4 + torch.nn.functional.softplus(raw)
    return dist_params, torch.ones_like(dist_params)


def graph_latent_encoder(params, prefix, g, cfg, grid_rep, st, m2m_layers, dist):
    """GraphLatentEncoder -> (mean, std) (graph_encoder.py:102-105)."""
    hl, B = cfg.get("hidden_layers", 1), grid_rep.shape[0]
    mesh = _gnn(params, f"{prefix}.g2m_gnn", g["g2m_edge_index"], grid_rep, _expand(st["mesh"], B), _expand(st["g2m"], B), hl,
                cfg.get("g2m_gnn_type", "InteractionNet"), update_edges=False)
    edge = _expand(st["m2m"], B)
    for i in range(m2m_layers):
        mesh, edge = _gnn(params, f"{prefix}.m2m_gnns.module_{i}", g["m2m_edge_index"], mesh, mesh, edge, hl)
    return mean_std(mlp(mesh, params, f"{prefix}.latent_param_map", hl, layer_norm=False), dist)


def prior(params, g, cfg, grid_emb, st):
    """the prior's (mean, std): GraphLatentEncoder, or the constant prior's zeros through ``mean_std``"""
    if cfg.get("learn_prior", True):
        return graph_latent_encoder(params, "prior_model", g, cfg, grid_emb, st, cfg["prior_m2m_layers"],
                                    cfg.get("prior_dist", "isotropic"))
    z = grid_emb.new_zeros(grid_emb.shape[0], cfg["num_mesh_nodes"],
                           cfg["latent_dim"] * (2 if cfg.get("prior_dist") == "diagonal" else 1))
    return mean_std(z, cfg.get("prior_dist", "isotropic"))


def decoder(params, g, cfg, grid_emb, z, st):
    """GraphLatentDecoder -> (mean_delta, pred_std|None) (base_decoder.py:145-171, graph_decoder.py:127-134)."""
    hl, B = cfg.get("hidden_layers", 1), grid_emb.shape[0]
    latent_emb = mlp(z, params, "decoder.latent_embedder", hl)
    res_grid = grid_emb + mlp(grid_emb, params, "decoder.grid_update_mlp", hl)
    mesh = _gnn(params, "decoder.g2m_gnn", g["g2m_edge_index"], grid_emb, latent_emb, _expand(st["g2m"], B), hl,
                cfg.get("g2m_gnn_type", "InteractionNet"), update_edges=False)
    edge = _expand(st["m2m"], B)
    for i in range(cfg["decoder_m2m_layers"]):
        mesh, edge = _gnn(params, f"decoder.m2m_gnns.module_{i}", g["m2m_edge_index"], mesh, mesh, edge, hl)
    grid = _gnn(params, "decoder.m2g_gnn", g["m2g_edge_index"], mesh, res_grid, _expand(st["m2g"], B), hl,
                cfg.get("m2g_gnn_type", "InteractionNet"), update_edges=False)
    out = mlp(grid, params, "decoder.param_map", hl, layer_norm=False)
    if cfg.get("output_std"):
        mean_delta, raw = out.chunk(2, dim=-1)
        return mean_delta, torch.nn.functional.softplus(raw)
    return out, None


def efm_step(params, graph, cfg, prev_state, prev_prev_state, forcing, eps):
    """One ``GraphEFMMultiScale.forward`` with the prior sample ``z = mean + eps * std`` ->
    dict(pred, pred_std, prior_mean, prior_std, z)."""
    dt = prev_state.dtype
    g = _cast(graph, dt)
    st = static_embeddings(params, g, cfg)
    grid_emb = grid_embedding(params, g, cfg, prev_state, prev_prev_state, forcing)
    mean, std = prior(params, g, cfg, grid_emb, st)
    z = mean + eps.to(dt) * std
    mean_delta, pred_std = decoder(params, g, cfg, grid_emb, z, st)
    delta = mean_delta * g["diff_std"] + g["diff_mean"]
    clamp = cfg.get("clamp")
    if clamp:
        pred = clamped_new_state(delta, prev_state, clamp["names"], clamp["lower"], clamp["upper"], clamp["state_mean"].to(dt),
                                 clamp["state_std"].to(dt))
    else:
        pred = prev_state + delta
    return dict(pred=pred, pred_std=pred_std, prior_mean=mean, prior_std=std, z=z)


def efm_posterior(params, graph, cfg, prev_state, prev_prev_state, forcing, target):
    """The variational encoder's (mean, std) given the target X_{t+1} (graph_efm.py:301-343, ``output_dist="diagonal"``)."""
    g = _cast(graph, prev_state.dtype)
    st = static_embeddings(params, g, cfg)
    grid_cur = grid_embedding(params, g, cfg, prev_state, prev_prev_state, forcing, target=target)
    return graph_latent_encoder(params, "encoder", g, cfg, grid_cur, st, cfg["encoder_m2m_layers"], "diagonal")
