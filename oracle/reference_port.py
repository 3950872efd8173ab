"""CPU restatement (oracle) of the Neural-LAM GNN message-passing hot path.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``): never imported by the
product package.  Pure ``torch`` CPU ops written out explicitly (no
``torch.nn`` modules, no torch_geometric), usable in fp32 ("reference
equivalent") and fp64 ("ground truth").  All parameters come in as a flat
``{name: tensor}`` dict using the reference's ``state_dict`` key names.

Each function cites the reference code it follows (paths relative to
``/root/reference``).
"""
import contextlib
import math

import torch

# --------------------------------------------------------------------------------------------------
# The reference's GPU configuration: ``torch.set_float32_matmul_precision("high")`` whenever CUDA is
# available (train_model.py:484-488) = TF32 tensor-core matmuls: both operands rounded to TF32 (10
# explicit mantissa bits), products accumulated in fp32.  ``tf32_matmul()`` makes ``mlp`` emulate that on
# the CPU, so that "the error of the reference's own GPU configuration" is a number the tests can state
# without a GPU run of the reference.  In fp64 the operands are rounded to TF32 and the products summed in
# fp64: a reference for kernels whose only intended rounding is that of their TF32 operands.
# ``mode="rz"`` (truncation toward zero, what a tensor core does with fp32 bits it is handed unrounded) exists
# so that tests can tell the two rounding modes apart.
# --------------------------------------------------------------------------------------------------
_TF32 = None  # None (exact matmuls) or the rounding mode of the operands: "rna" | "rz"


@contextlib.contextmanager
def tf32_matmul(enabled=True, mode="rna"):
    global _TF32
    assert mode in ("rna", "rz"), mode
    old, _TF32 = _TF32, (mode if enabled else None)
    try:
        yield
    finally:
        _TF32 = old


def round_tf32(x, mode="rna"):
    """-> x rounded to TF32 (10 explicit mantissa bits), same dtype.  ``"rna"``: to nearest, ties away from zero;
    ``"rz"``: toward zero.  fp32 rounds on the 13 dropped mantissa bits; fp64 rounds its own value (never through
    fp32 first)."""
    assert mode in ("rna", "rz"), mode
    if x.dtype == torch.float32:
        bits = x.contiguous().view(torch.int32)
        if mode == "rna":
            bits = bits + 0x1000
        return (bits & ~0x1FFF).view(torch.float32)
    assert x.dtype == torch.float64, x.dtype
    m, e = torch.frexp(x)                  # x = m * 2^e, 0.5 <= |m| < 1: 11 significant bits = |m| * 2^11 in [1024, 2048)
    q = m.abs() * 2048.0
    q = torch.floor(q + 0.5) if mode == "rna" else torch.floor(q)
    return torch.ldexp(torch.copysign(q, m), (e - 11).to(torch.float64))


# ---------------------------------------------------------------------------
# MLP  (neural_lam/utils/networks.py:27-40)
# ---------------------------------------------------------------------------
def mlp(x, params, prefix, hidden_layers=1, layer_norm=True, eps=1e-5):
    """``make_mlp`` network: Linear -> SiLU -> ... -> Linear [-> LayerNorm].

    networks.py:31-35 (Linear + SiLU on all but the last Linear), :37-38
    (LayerNorm(blueprint[-1]), torch defaults eps=1e-5, affine).
    ``nn.Sequential`` indices: Linear k sits at ``2*k``; LayerNorm at
    ``2*hidden_layers + 1``.
    """
    h = x
    for k in range(hidden_layers + 1):
        w = params[f"{prefix}.{2 * k}.weight"].to(h.dtype)
        b = params[f"{prefix}.{2 * k}.bias"].to(h.dtype)
        if _TF32 is not None and h.dtype in (torch.float32, torch.float64):
            h = round_tf32(h, _TF32) @ round_tf32(w, _TF32).t() + b
        else:
            h = h @ w.t() + b
        if k != hidden_layers:
            h = h * torch.sigmoid(h)  # SiLU
    if layer_norm:
        g = params[f"{prefix}.{2 * hidden_layers + 1}.weight"].to(h.dtype)
        bb = params[f"{prefix}.{2 * hidden_layers + 1}.bias"].to(h.dtype)
        mu = h.mean(dim=-1, keepdim=True)
        var = ((h - mu) ** 2).mean(dim=-1, keepdim=True)  # biased, as LayerNorm
        h = (h - mu) / torch.sqrt(var + eps) * g + bb
    return h


def split_mlps(x, params, prefix, chunk_sizes, **kw):
    """``SplitMLPs.forward`` (gnn_layers.py:305-324): split dim -2, one MLP per
    chunk (``{prefix}.mlps.{k}``), concatenate."""
    outs = []
    start = 0
    for k, n in enumerate(chunk_sizes):
        outs.append(mlp(x[..., start : start + n, :], params, f"{prefix}.mlps.{k}", **kw))
        start += n
    assert start == x.shape[-2]
    return torch.cat(outs, dim=-2)


# ---------------------------------------------------------------------------
# InteractionNet / PropagationNet  (neural_lam/gnn_layers.py)
# ---------------------------------------------------------------------------
def scatter_aggregate(messages, receivers, num_rec, aggr):
    """PyG 2.3.1 ``SumAggregation`` / ``MeanAggregation`` as reached from
    gnn_layers.py:188: zero-filled ``(…, num_rec, H)`` + ``scatter_add_`` over the
    node dim (-2); mean divides by the in-degree clamped to >= 1."""
    size = list(messages.shape)
    size[-2] = num_rec
    out = messages.new_zeros(size)
    out.index_add_(messages.dim() - 2, receivers, messages)
    if aggr == "mean":
        cnt = messages.new_zeros(num_rec)
        cnt.index_add_(0, receivers, messages.new_ones(receivers.numel()))
        out = out / cnt.clamp(min=1).unsqueeze(-1)
    return out


def interaction_net(
    params,
    edge_index,
    send_rep,
    rec_rep,
    edge_rep,
    prefix="",
    aggr="sum",
    update_edges=True,
    propagation=False,
    hidden_layers=1,
    edge_chunk_sizes=None,
    aggr_chunk_sizes=None,
    return_internals=False,
):
    """``InteractionNet.forward`` (gnn_layers.py:110-157) /
    ``PropagationNet`` (gnn_layers.py:192-249).

    ``edge_index`` is the ORIGINAL zero-based ``(2, E)`` index (row 0 senders in
    their own node set, row 1 receivers), i.e. the constructor argument
    (gnn_layers.py:23-26), not the offset buffer.
    """
    p = (prefix + ".") if prefix else ""
    if propagation:
        aggr = "mean"  # gnn_layers.py:219-229
    senders = edge_index[0].long()
    receivers = edge_index[1].long()
    num_rec = int(receivers.max()) + 1  # gnn_layers.py:73
    assert rec_rep.shape[-2] == num_rec

    # propagate (gnn_layers.py:144-147): gather sender/receiver rows
    x_j = send_rep.index_select(send_rep.dim() - 2, senders)
    x_i = rec_rep.index_select(rec_rep.dim() - 2, receivers)
    # message (gnn_layers.py:168-172): edge_mlp(cat(edge_attr, x_j, x_i))
    edge_in = torch.cat((edge_rep, x_j, x_i), dim=-1)
    if edge_chunk_sizes is None:
        msg = mlp(edge_in, params, p + "edge_mlp", hidden_layers)
    else:
        msg = split_mlps(edge_in, params, p + "edge_mlp", edge_chunk_sizes, hidden_layers=hidden_layers)
    if propagation:
        msg = x_j + msg  # gnn_layers.py:249
    # aggregate (gnn_layers.py:175-189)
    edge_rep_aggr = scatter_aggregate(msg, receivers, num_rec, aggr)
    # node update (gnn_layers.py:148)
    node_in = torch.cat((rec_rep, edge_rep_aggr), dim=-1)
    if aggr_chunk_sizes is None:
        rec_diff = mlp(node_in, params, p + "aggr_mlp", hidden_layers)
    else:
        rec_diff = split_mlps(node_in, params, p + "aggr_mlp", aggr_chunk_sizes, hidden_layers=hidden_layers)
    # residual (gnn_layers.py:151; target :159-166 / :231-239)
    base = edge_rep_aggr if propagation else rec_rep
    new_rec = base + rec_diff
    if return_internals:
        return new_rec, edge_rep + msg, edge_rep_aggr, msg
    if update_edges:
        return new_rec, edge_rep + msg  # gnn_layers.py:153-155
    return new_rec


# ---------------------------------------------------------------------------
# Step predictors
# ---------------------------------------------------------------------------
def _expand(x, batch_size):
    """``expand_to_batch`` (models/step_predictors/base.py:122-139)."""
    return x.unsqueeze(0).expand(batch_size, -1, -1)


def graph_model_forward(params, graph, cfg, prev_state, prev_prev_state, forcing, prefix=""):
    """``BaseGraphModel.forward`` (models/step_predictors/graph/base.py:228-344)
    with ``GraphLAM.process_step`` (graph/graph_lam.py:157-188) or
    ``BaseHiGraphModel.process_step`` + ``HiLAM.hi_processor_step``
    (graph/hierarchical.py:186-292, graph/hi_lam.py:167-376).

    ``graph`` holds the tensors ``load_graph`` registers (utils/graph.py:146-422);
    ``cfg`` = dict(model="graph_lam"|"hi_lam", hidden_layers, processor_layers,
    mesh_aggr, gnn types).  No clamping limits (step_predictors/base.py:366-396
    with empty index lists reduces to ``prev_state + delta``), no output_std.
    """
    p = (prefix + ".") if prefix else ""
    dt = prev_state.dtype
    hl = cfg.get("hidden_layers", 1)
    B = prev_state.shape[0]
    g = {k: ([t.to(dt) if t.is_floating_point() else t for t in v] if isinstance(v, (list, tuple)) else (v.to(dt) if v.is_floating_point() else v)) for k, v in graph.items()}

    def gnn(name, ei, send, rec, edge, **kw):
        kind = kw.pop("gnn_type", "InteractionNet")
        return interaction_net(
            params, ei, send, rec, edge, prefix=p + name, hidden_layers=hl,
            propagation=(kind == "PropagationNet"), **kw,
        )

    # base.py:275-283 grid feature concat, :286 embed, :289-295 static embedders
    grid_features = torch.cat(
        (prev_state, prev_prev_state, forcing, _expand(g["grid_static_features"], B)), dim=-1
    )
    grid_emb = mlp(grid_features, params, p + "grid_embedder", hl)
    g2m_emb = mlp(g["g2m_features"], params, p + "g2m_embedder", hl)
    m2g_emb = mlp(g["m2g_features"], params, p + "m2g_embedder", hl)
    hierarchical = cfg["model"] != "graph_lam"  # "hi_lam" | "hi_lam_parallel"
    if hierarchical:
        mesh_emb = mlp(g["mesh_static_features"][0], params, p + "mesh_embedders.0", hl)
    else:
        mesh_emb = mlp(g["mesh_static_features"], params, p + "mesh_embedder", hl)
    # base.py:298-310 encode
    mesh_rep = gnn(
        "g2m_gnn", g["g2m_edge_index"], grid_emb, _expand(mesh_emb, B), _expand(g2m_emb, B),
        update_edges=False, gnn_type=cfg.get("g2m_gnn_type", "InteractionNet"),
    )
    grid_rep = grid_emb + mlp(grid_emb, params, p + "encoding_grid_mlp", hl)

    if not hierarchical:
        # graph_lam.py:176-188
        m2m_emb = _expand(mlp(g["m2m_features"], params, p + "m2m_embedder", hl), B)
        edge = m2m_emb
        for i in range(cfg["processor_layers"]):
            mesh_rep, edge = gnn(
                f"processor.module_{i}", g["m2m_edge_index"], mesh_rep, mesh_rep, edge,
                aggr=cfg.get("mesh_aggr", "sum"),
            )
    else:
        L = len(g["mesh_static_features"])
        up_t = cfg.get("mesh_up_gnn_type", "InteractionNet")
        down_t = cfg.get("mesh_down_gnn_type", "InteractionNet")
        # hierarchical.py:205-237
        levels = [mesh_rep] + [
            _expand(mlp(g["mesh_static_features"][l], params, p + f"mesh_embedders.{l}", hl), B)
            for l in range(1, L)
        ]
        same = [_expand(mlp(g["m2m_features"][l], params, p + f"mesh_same_embedders.{l}", hl), B) for l in range(L)]
        up = [_expand(mlp(g["mesh_up_features"][l], params, p + f"mesh_up_embedders.{l}", hl), B) for l in range(L - 1)]
        down = [_expand(mlp(g["mesh_down_features"][l], params, p + f"mesh_down_embedders.{l}", hl), B) for l in range(L - 1)]
        # hierarchical.py:241-262 mesh init (up sweep)
        for l in range(1, L):
            levels[l], up[l - 1] = gnn(
                f"mesh_init_gnns.{l - 1}", g["mesh_up_edge_index"][l - 1], levels[l - 1], levels[l], up[l - 1],
                gnn_type=up_t,
            )
        if cfg["model"] == "hi_lam_parallel":
            # hi_lam_parallel.py:89-122 (offset concatenation) and :186-218: ONE InteractionNet per layer over
            # all levels / edge sets with per-section MLPs (SplitMLPs)
            sizes = [t.shape[-2] for t in levels]
            first = [0]
            for n in sizes[:-1]:
                first.append(first[-1] + n)
            total = [ei + off for ei, off in zip(g["m2m_edge_index"], first)]
            total += [torch.stack((ei[0] + first[l], ei[1] + first[l + 1])) for l, ei in enumerate(g["mesh_up_edge_index"])]
            total += [torch.stack((ei[0] + first[l + 1], ei[1] + first[l])) for l, ei in enumerate(g["mesh_down_edge_index"])]
            sections = [ei.shape[1] for ei in total]
            tei = torch.cat(total, dim=1)
            mesh_all = torch.cat(levels, dim=1)
            edge_all = torch.cat(same + up + down, dim=1)
            for k in range(cfg["processor_layers"]):
                mesh_all, edge_all = interaction_net(
                    params, tei, mesh_all, mesh_all, edge_all, prefix=p + f"processor.module_{k}", hidden_layers=hl,
                    edge_chunk_sizes=sections, aggr_chunk_sizes=sizes)
            levels = list(torch.split(mesh_all, sizes, dim=1))
            parts = torch.split(edge_all, sections, dim=1)
            same, up, down = list(parts[:L]), list(parts[L:2 * L - 1]), list(parts[2 * L - 1:])
        # hi_lam.py:350-376
        for k in range(cfg["processor_layers"] if cfg["model"] == "hi_lam" else 0):
            # mesh_down_step hi_lam.py:205-236
            levels[-1], same[-1] = gnn(f"mesh_down_same_gnns.{k}.{L - 1}", g["m2m_edge_index"][L - 1], levels[-1], levels[-1], same[-1])
            for l in range(L - 2, -1, -1):
                new_node, down[l] = gnn(
                    f"mesh_down_gnns.{k}.{l}", g["mesh_down_edge_index"][l], levels[l + 1], levels[l], down[l],
                    gnn_type=down_t,
                )
                levels[l], same[l] = gnn(f"mesh_down_same_gnns.{k}.{l}", g["m2m_edge_index"][l], new_node, new_node, same[l])
            # mesh_up_step hi_lam.py:277-307
            levels[0], same[0] = gnn(f"mesh_up_same_gnns.{k}.0", g["m2m_edge_index"][0], levels[0], levels[0], same[0])
            for l in range(1, L):
                new_node, up[l - 1] = gnn(
                    f"mesh_up_gnns.{k}.{l - 1}", g["mesh_up_edge_index"][l - 1], levels[l - 1], levels[l], up[l - 1],
                    gnn_type=up_t,
                )
                levels[l], same[l] = gnn(f"mesh_up_same_gnns.{k}.{l}", g["m2m_edge_index"][l], new_node, new_node, same[l])
        # hierarchical.py:271-289 read-out (down sweep, update_edges=False)
        for l in range(L - 2, -1, -1):
            levels[l] = gnn(
                f"mesh_read_gnns.{l}", g["mesh_down_edge_index"][l], levels[l + 1], levels[l], down[l],
                update_edges=False, gnn_type=down_t,
            )
        mesh_rep = levels[0]

    # base.py:316-322 decode + output map (no LayerNorm, base.py:172-175)
    grid_rep = gnn(
        "m2g_gnn", g["m2g_edge_index"], mesh_rep, grid_rep, _expand(m2g_emb, B),
        update_edges=False, gnn_type=cfg.get("m2g_gnn_type", "InteractionNet"),
    )
    net_output = mlp(grid_rep, params, p + "output_map", hl, layer_norm=False)
    pred_std = None
    if cfg.get("output_std"):
        # base.py:324-334: mean | raw std halves, softplus on the std half (not rescaled)
        net_output, std_raw = net_output.chunk(2, dim=-1)
        pred_std = torch.nn.functional.softplus(std_raw)
    # base.py:339 rescale; :342 / step_predictors/base.py:366 residual (clamped where limits are configured)
    delta = net_output * g["diff_std"] + g["diff_mean"]
    clamp = cfg.get("clamp")
    if clamp:
        new_state = clamped_new_state(delta, prev_state, clamp["names"], clamp["lower"], clamp["upper"],
                                      clamp["state_mean"].to(dt), clamp["state_std"].to(dt))
    else:
        new_state = prev_state + delta
    if cfg.get("return_std"):
        return new_state, pred_std
    return new_state


def ar_rollout(params, graph, cfg, init_states, forcing_features, boundary_states, prefix="predictor"):
    """``ARForecaster.forward`` (models/forecasters/autoregressive.py:113-149).  Returns the stacked prediction, or
    ``(prediction, pred_std)`` when ``cfg["return_std"]`` (std None for predictors without one, :142-148)."""
    dt = init_states.dtype
    bm = graph["boundary_mask"].to(dt)
    im = 1.0 - bm
    prev_prev, prev = init_states[:, 0], init_states[:, 1]
    preds, stds = [], []
    for i in range(forcing_features.shape[1]):
        pred = graph_model_forward(params, graph, cfg, prev, prev_prev, forcing_features[:, i], prefix=prefix)
        if cfg.get("return_std"):
            pred, std = pred
            if std is not None:
                stds.append(std)
        new = bm * boundary_states[:, i] + im * pred  # autoregressive.py:128-131
        preds.append(new)
        prev_prev, prev = prev, new
    if cfg.get("return_std"):
        return torch.stack(preds, dim=1), (torch.stack(stds, dim=1) if stds else None)
    return torch.stack(preds, dim=1)


def algorithmic_bytes_inet(B, Ns, Nr, E, H, update_edges, same_nodes):
    """SURVEY.md section 8(d): algorithmic HBM bytes of one InteractionNet call
    (fp32, forward)."""
    nodes_read = (Nr if same_nodes else (Ns + Nr))
    reads = 4 * H * B * (nodes_read + E)
    writes = 4 * H * B * (Nr + (E if update_edges else 0))
    index = 4 * E + 4 * (Nr + 1)
    weights = 4 * (7 * H * H + 8 * H)
    return reads + writes + index + weights


def flops_inet(B, Nr, E, H):
    """SURVEY.md section 8(d): forward FLOPs (LayerNorm/SiLU excluded)."""
    return B * (8 * H * H * E + 6 * H * H * Nr)


# ---------------------------------------------------------------------------------------------------
# Output clamping (models/step_predictors/base.py:181-396 with utils/tensor.py:7-81)
# ---------------------------------------------------------------------------------------------------
def ref_inverse_softplus(x, beta=1.0, threshold=20.0):
    """utils/tensor.py:7-50."""
    x_clamped = torch.clamp(x, min=torch.log(torch.tensor(1e-6 + 1)) / beta, max=threshold / beta)
    non_linear_part = torch.log(torch.expm1(x_clamped * beta)) / beta
    below_threshold = x * beta <= threshold
    return torch.where(below_threshold, non_linear_part, x)


def ref_inverse_sigmoid(x):
    """utils/tensor.py:53-81."""
    x_clamped = torch.clamp(x, min=1e-6, max=1 - 1e-6)
    return torch.log(x_clamped / (1 - x_clamped))


def clamped_new_state(state_delta, prev_state, names, lower, upper, state_mean, state_std):
    """``prepare_clamping_params`` + ``get_clamped_new_state`` (step_predictors/base.py:181-396): per state variable
    with both limits a scaled sigmoid, lower-only / upper-only a shifted softplus, applied as f(f^-1(X_t) + delta);
    limits standardised with the state statistics (:229-234); sharpness 1 and centre 0 (:217-220)."""
    new_state = prev_state + state_delta
    for i, n in enumerate(names):
        has_lo, has_up = n in lower, n in upper
        if not (has_lo or has_up):
            continue
        lo = (lower[n] - state_mean[i]) / state_std[i] if has_lo else None
        up = (upper[n] - state_mean[i]) / state_std[i] if has_up else None
        x, d = prev_state[:, :, i], state_delta[:, :, i]
        if has_lo and has_up:
            z = 0 + ref_inverse_sigmoid((x - lo) / (up - lo)) / 1 + d                       # :316-322
            new_state[:, :, i] = lo + (up - lo) * torch.sigmoid(1 * (z - 0))              # :296-300
        elif has_lo:
            z = ref_inverse_softplus(x - lo, beta=1) + 0 + d                              # :323-328
            new_state[:, :, i] = lo + torch.nn.functional.softplus(z - 0, beta=1)         # :301-306
        else:
            z = -ref_inverse_softplus(up - x, beta=1) + 0 + d                             # :329-334
            new_state[:, :, i] = up - torch.nn.functional.softplus(0 - z, beta=1)         # :307-312
    return new_state
