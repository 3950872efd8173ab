"""Parity of the wgmma (TF32 tensor-core) kernels, through the C ABI, against the CPU oracle.

Stated tolerance (TF32 inputs, fp32 accumulate; LayerNorm outputs are O(1)):
  * |kernel - fp64 oracle| <= 1e-2 absolute per InteractionNet call, and
  * <= max(3x the error the REFERENCE's own GPU configuration makes on the same inputs, 4e-3):
    the reference error is that of the oracle op sequence run by torch on the GPU with TF32
    matmuls enabled, as the reference enables them whenever CUDA is available (reference
    neural_lam/train_model.py:484-488); 4e-3 is the floor for shapes where cuBLAS does not
    actually take a TF32 path (e.g. single-row GEMV).
"""
import pytest
import torch

import neural_lam_b200 as nlb
from neural_lam_b200 import _lib, models, ops, synthetic
from oracle import reference_port as rp

pytestmark = pytest.mark.gpu
DEV = "cuda"
ABS_TOL = 1e-2


def _ref_tf32_err(fn64, fn_gpu):
    """error of the reference-style torch TF32 GPU evaluation vs the fp64 oracle"""
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        got = fn_gpu()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    want = fn64()
    if isinstance(got, torch.Tensor):
        got, want = (got,), (want,)
    return max((g.double().cpu() - w).abs().max().item() for g, w in zip(got, want)), want


def _graph(ns, nr, ne, seed, sort):
    g = torch.Generator().manual_seed(seed)
    ei = torch.stack([torch.randint(0, ns, (ne,), generator=g), torch.randint(0, nr, (ne,), generator=g)])
    ei[1, -1] = nr - 1
    if sort:
        ei = ei[:, torch.sort(ei[1], stable=True).indices]
    return ei


CASES = [
    # name, ns, nr, ne, B, update_edges, aggr, same nodes, sorted, expanded edge
    ("sum_upd", 50, 30, 400, 2, True, "sum", False, True, False),
    ("mean_noupd", 50, 30, 400, 2, False, "mean", False, True, False),
    ("m2m_same", 200, 200, 1800, 3, True, "sum", True, True, False),
    ("unsorted", 60, 40, 500, 2, True, "sum", False, False, False),
    ("expanded_edge", 60, 40, 500, 3, True, "sum", False, True, True),
    ("empty_receivers", 40, 600, 300, 2, True, "sum", False, True, False),
    ("single_tile", 5, 4, 10, 1, True, "sum", False, True, False),
    ("deg128", 300, 3, 300, 2, False, "sum", False, True, False),
    # batch-broadcast edge features, no edge update, large sender set -> tc_edge_bcast_kernel
    ("bcast_g2m", 3000, 200, 2500, 3, False, "sum", False, True, True),
    ("bcast_mean_b1", 3000, 200, 2500, 1, False, "mean", False, True, True),
    ("bcast_many_items", 60000, 3000, 40000, 5, False, "sum", False, True, True),
    ("bcast_deg100", 2000, 3, 300, 4, False, "sum", False, True, True),
    ("bcast_empty_receivers", 5000, 900, 400, 2, False, "sum", False, True, True),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_edge_and_node_kernels_vs_oracle(case):
    name, ns, nr, ne, B, upd, aggr, same, srt, expand = case
    ei = _graph(ns, nr, ne, 1, srt)
    torch.manual_seed(0)
    net = nlb.InteractionNet(ei, 64, update_edges=upd, aggr=aggr, math="tf32")
    with torch.no_grad():
        for p in net.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    send = torch.randn(B, ns, 64)
    rec = send if same else torch.randn(B, nr, 64)
    if name.startswith("bcast"):  # grid -> mesh shape: receivers and edge features are batch-broadcast static embeddings
        rec = torch.randn(1, nr, 64).expand(B, -1, -1)
    edge = torch.randn(1 if expand else B, ne, 64)
    sd = dict(net.state_dict())
    sd64 = {k: v.double() for k, v in sd.items()}
    sdg = {k: v.to(DEV) for k, v in sd.items()}

    def f64():
        return rp.interaction_net(sd64, ei, send.double(), rec.double(), edge.double().expand(B, -1, -1), aggr=aggr,
                                  update_edges=upd)

    def fgpu():
        return rp.interaction_net(sdg, ei.to(DEV), send.to(DEV), rec.to(DEV), edge.to(DEV).expand(B, -1, -1),
                                  aggr=aggr, update_edges=upd)

    ref_err, want = _ref_tf32_err(f64, fgpu)
    net = net.to(DEV)
    rec_dev = (send if same else rec).to(DEV)
    if name.startswith("bcast"):
        rec_dev = rec[:1].to(DEV).expand(B, -1, -1)  # stride-0 batch, as expand_to_batch hands it over
    with torch.no_grad(), ops.profile_launches() as prof:
        got = net(send.to(DEV), rec_dev, edge.to(DEV).expand(B, -1, -1))
    if name.startswith("bcast"):
        assert "tc_edge_bcast_kernel" in prof.names(), prof.names()
    assert not any("simt" in n for n in prof.names()), prof.names()
    got = got if isinstance(got, tuple) else (got,)
    err = max((g.double().cpu() - w).abs().max().item() for g, w in zip(got, want))
    assert err <= ABS_TOL, (name, err)
    assert err <= max(3 * ref_err, 4e-3), (name, err, ref_err)


GEN_CASES = [
    # name, class, H, ns, nr, ne, B, update_edges, aggr, expanded edge
    ("h128_sum_upd", "InteractionNet", 128, 300, 200, 1500, 2, True, "sum", False),
    ("h128_mean_noupd_bcast", "InteractionNet", 128, 300, 200, 1500, 3, False, "mean", True),
    ("h256_sum_upd", "InteractionNet", 256, 200, 150, 900, 2, True, "sum", False),
    ("h256_b1_many_tiles", "InteractionNet", 256, 5000, 3000, 20000, 1, True, "sum", False),
    ("h128_prop", "PropagationNet", 128, 120, 80, 700, 2, True, "sum", False),
    ("h64_prop", "PropagationNet", 64, 120, 80, 700, 2, True, "sum", False),
    ("h64_prop_noupd", "PropagationNet", 64, 120, 80, 700, 2, False, "sum", True),
]


@pytest.mark.parametrize("case", GEN_CASES, ids=[c[0] for c in GEN_CASES])
def test_generic_tensor_core_path_vs_oracle(case):
    """H = 128 / 256 (BASELINE configs 3-5) and PropagationNet: the generic wgmma Linear kernel (tc7.cu) — node
    projections, two edge layers, CSR segment sum, two node layers — against the fp64 oracle, same bound as above."""
    name, cls, H, ns, nr, ne, B, upd, aggr, expand = case
    ei = _graph(ns, nr, ne, 3, True)
    torch.manual_seed(0)
    net = getattr(nlb, cls)(ei, H, update_edges=upd, aggr=aggr, math="tf32")
    with torch.no_grad():
        for p in net.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    send, rec = torch.randn(B, ns, H), torch.randn(B, nr, H)
    edge = torch.randn(1 if expand else B, ne, H)
    prop = cls == "PropagationNet"
    sd = dict(net.state_dict())
    sd64 = {k: v.double() for k, v in sd.items()}
    sdg = {k: v.to(DEV) for k, v in sd.items()}

    def f64():
        return rp.interaction_net(sd64, ei, send.double(), rec.double(), edge.double().expand(B, -1, -1), aggr=aggr,
                                  update_edges=upd, propagation=prop)

    def fgpu():
        return rp.interaction_net(sdg, ei.to(DEV), send.to(DEV), rec.to(DEV), edge.to(DEV).expand(B, -1, -1), aggr=aggr,
                                  update_edges=upd, propagation=prop)

    ref_err, want = _ref_tf32_err(f64, fgpu)
    net = net.to(DEV)
    with torch.no_grad(), ops.profile_launches() as prof:
        got = net(send.to(DEV), rec.to(DEV), edge.to(DEV).expand(B, -1, -1))
    names = prof.names()
    assert any(n.startswith("tc_linear_kernel") for n in names) and not any("rowmlp_simt" in n for n in names), names
    got = got if isinstance(got, tuple) else (got,)
    err = max((g.double().cpu() - w).abs().max().item() for g, w in zip(got, want))
    print(f"{name}: err {err:.3e} (reference TF32 config {ref_err:.3e}); launches {names}")
    assert err <= ABS_TOL, (name, err)
    assert err <= max(3 * ref_err, 4e-3), (name, err, ref_err)


GEN_ROW_CASES = [
    ("h128_embed", [128, 128, 128], [(2, 700, 128)], None, True),
    ("h128_node_res", [256, 128, 128], [(2, 333, 128), (2, 333, 128)], 0, True),
    ("h256_node_res_aggr", [512, 256, 256], [(1, 1000, 256), (1, 1000, 256)], 1, True),
    ("h256_bcast_in", [256, 256, 256], [(500, 256)], None, True),
    ("h128_output_map_17", [128, 128, 17], [(2, 400, 128)], None, False),
    ("h128_grid_embedder_56", [56, 128, 128], [(2, 400, 17), (2, 400, 17), (2, 400, 18), (400, 4)], None, True),
    ("h256_edge_embedder_3", [4, 256, 256], [(900, 4)], None, True),
]


@pytest.mark.parametrize("case", GEN_ROW_CASES, ids=[c[0] for c in GEN_ROW_CASES])
def test_generic_row_mlp_vs_oracle(case):
    name, blueprint, shapes, res_i, ln = case
    torch.manual_seed(1)
    mlp = nlb.make_mlp(blueprint, layer_norm=ln)
    srcs = [torch.randn(*sh) for sh in shapes]
    sd64 = {f"m.{k}": v.double() for k, v in mlp.state_dict().items()}
    B = max((t.shape[0] for t in srcs if t.dim() == 3), default=1)
    cat64 = torch.cat([(t if t.dim() == 3 else t.unsqueeze(0).expand(B, -1, -1)).double() for t in srcs], dim=-1)
    want = rp.mlp(cat64, sd64, "m", 1, layer_norm=ln)
    if res_i is not None:
        want = want + srcs[res_i].double()
    mlp = mlp.to(DEV)
    mlp.nlam_flags = _lib.MATH_TF32
    with torch.no_grad(), ops.profile_launches() as prof:
        got = mlp.apply_rows([t.to(DEV) for t in srcs], res=None if res_i is None else srcs[res_i].to(DEV))
    assert all(n.startswith(("tc_linear_kernel", "pack_rows")) for n in prof.names()), prof.names()
    got = got if got.dim() == 3 else got.unsqueeze(0)
    err = (got.double().cpu() - want).abs().max().item()
    print(f"{name}: err {err:.3e}")
    assert err <= ABS_TOL, (name, err)


def test_tf32_requested_but_unsupported_raises_and_auto_falls_back():
    ei = _graph(50, 3, 500, 0, True)  # in-degree > 128: outside the tensor-core tile table
    for H, ok_auto in ((64, True), (16, True)):
        net_auto = nlb.InteractionNet(ei, H, math="auto").to(DEV)
        x = [torch.randn(50, H, device=DEV), torch.randn(3, H, device=DEV), torch.randn(500, H, device=DEV)]
        r, e = net_auto(*x)
        r_o, e_o = rp.interaction_net({k: v.cpu() for k, v in net_auto.state_dict().items()}, ei, *[t.cpu() for t in x])
        torch.testing.assert_close(r.cpu(), r_o, rtol=2e-5, atol=2e-5)  # exact-fp32 kernels were used
        net_tf = nlb.InteractionNet(ei, H, math="tf32").to(DEV)
        with pytest.raises(_lib.NlamError, match="not supported by the tensor-core"):
            net_tf(*x)


ROW_CASES = [
    ("embed_ln", [64, 64, 64], [(3, 300, 64)], None, True),
    ("embed_res", [64, 64, 64], [(2, 1000, 64)], 0, True),
    ("node_res_rec", [128, 64, 64], [(2, 777, 64), (2, 777, 64)], 0, True),
    ("node_res_aggr", [128, 64, 64], [(2, 130, 64), (2, 130, 64)], 1, True),
    ("node_bcast", [128, 64, 64], [(257, 64), (3, 257, 64)], None, True),
    ("output_map_17", [64, 64, 17], [(2, 500, 64)], None, False),
    ("grid_embedder_56", [56, 64, 64], [(2, 400, 17), (2, 400, 17), (2, 400, 18), (400, 4)], None, True),
    ("one_row", [64, 64, 64], [(1, 1, 64)], None, True),
    # row kernel, several tiles per CTA, partial last tile
    ("enc_many_tiles", [64, 64, 64], [(2, 128 * 300 + 77, 64)], 0, True),
    ("node_many_tiles", [128, 64, 64], [(2, 128 * 200 + 3, 64), (2, 128 * 200 + 3, 64)], 0, True),
    ("node_res_aggr_many", [128, 64, 64], [(2, 128 * 160 + 9, 64), (2, 128 * 160 + 9, 64)], 1, True),
    # narrow inputs staged by bulk copies + repack (rows % 4 == 0; otherwise the element-wise loader), narrow output
    ("embedder_many_tiles", [56, 64, 64], [(2, 128 * 200 + 8, 17), (2, 128 * 200 + 8, 17), (2, 128 * 200 + 8, 18),
                                           (128 * 200 + 8, 4)], None, True),
    ("embedder_rows_not_mult4", [56, 64, 64], [(2, 401, 17), (2, 401, 17), (2, 401, 18), (401, 4)], None, True),
    ("output_map_many_tiles", [64, 64, 17], [(3, 128 * 200 + 5, 64)], None, False),
    ("narrow_in_narrow_out", [20, 64, 9], [(2, 1000, 13), (2, 1000, 7)], None, False),
    # a source whose width is a multiple of 4 starting at a column that is not (grid embedder, d_state 5, d_forcing 12)
    ("embedder_unaligned_offset", [24, 64, 64], [(2, 700, 5), (2, 700, 5), (2, 700, 12), (700, 2)], None, True),
]


@pytest.mark.parametrize("case", ROW_CASES, ids=[c[0] for c in ROW_CASES])
def test_row_kernel_vs_oracle(case):
    name, bp, shapes, res_idx, ln = case
    torch.manual_seed(0)
    m = nlb.make_mlp(bp, layer_norm=ln)
    with torch.no_grad():
        for p in m.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    srcs = [torch.randn(*s) for s in shapes]
    B = max([s.shape[0] for s in srcs if s.dim() == 3], default=1)
    cat = torch.cat([s if s.dim() == 3 else s.unsqueeze(0).expand(B, -1, -1) for s in srcs], dim=-1)
    res = None if res_idx is None else srcs[res_idx]
    p64 = {f"m.{k}": v.double() for k, v in m.state_dict().items()}
    pg = {f"m.{k}": v.to(DEV) for k, v in m.state_dict().items()}

    def f64():
        y = rp.mlp(cat.double(), p64, "m", layer_norm=ln)
        return y if res is None else y + res.double()

    def fgpu():
        y = rp.mlp(cat.to(DEV), pg, "m", layer_norm=ln)
        return y if res is None else y + res.to(DEV)

    ref_err, (want,) = _ref_tf32_err(f64, fgpu)
    m = m.to(DEV)
    ds = [s.to(DEV) for s in srcs]
    with torch.no_grad():
        got = ops.rowmlp(m, ds, res=None if res_idx is None else ds[res_idx], flags=_lib.MATH_TF32)
    err = (got.double().cpu().reshape(want.shape) - want).abs().max().item()
    assert err <= ABS_TOL, (name, err)
    assert err <= max(3 * ref_err, 4e-3), (name, err, ref_err)


@pytest.mark.parametrize("kind", ["graph_lam", "hi_lam"])
def test_model_rollout_tf32_vs_oracle(kind):
    """Whole forecast steps (hidden 64 -> every GNN / grid MLP on the tensor-core kernels), 2 AR
    steps, against the fp64 oracle; bound = 3x the reference-style torch TF32 GPU error."""
    spec = synthetic.make_graph_spec(30, 27, hierarchical=(kind == "hi_lam"))
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=2)
    torch.manual_seed(42)
    cls = models.HiLAM if kind == "hi_lam" else models.GraphLAM
    m = cls(ds, spec, hidden_dim=64, processor_layers=2, math="auto")
    fc = models.ARForecaster(m, ds)
    from test_models import _oracle_graph

    g = _oracle_graph(m, fc)
    cfg = dict(model=kind, hidden_layers=1, processor_layers=2, mesh_aggr="sum")
    G = m.num_grid_nodes
    gen = torch.Generator().manual_seed(123)
    B, T = 2, 2
    init, forc, bnd = torch.randn(B, 2, G, 17, generator=gen), torch.randn(B, T, G, 18, generator=gen), torch.randn(B, T, G, 17, generator=gen)
    params = {f"predictor.{k}": v for k, v in m.state_dict().items()}
    gd = {k: ([t.to(DEV) for t in v] if isinstance(v, list) else v.to(DEV)) for k, v in g.items()}

    def f64():
        return rp.ar_rollout({k: v.double() for k, v in params.items()}, g, cfg, init.double(), forc.double(), bnd.double())

    def fgpu():
        return rp.ar_rollout({k: v.to(DEV) for k, v in params.items()}, gd, cfg, init.to(DEV), forc.to(DEV), bnd.to(DEV))

    ref_err, (want,) = _ref_tf32_err(f64, fgpu)
    fc = fc.to(DEV)
    n0 = _lib.lib().nlam_launch_count()
    with torch.no_grad():
        got, _ = fc(init.to(DEV), forc.to(DEV), bnd.to(DEV))
        got_g = fc.rollout_graphed(init.to(DEV), forc.to(DEV), bnd.to(DEV))
    assert _lib.lib().nlam_launch_count() > n0
    err = (got.double().cpu() - want).abs().max().item()
    assert err <= 5e-2 and err <= max(3 * ref_err, 1e-2), (err, ref_err)
    torch.testing.assert_close(got_g, got, rtol=1e-6, atol=1e-6)


def test_split_and_k192_edge_forms_vs_oracle():
    """Both forms of the first edge Linear against the fp64 oracle, each picked by rule 2 of the edge path (DESIGN §4.1) on
    graphs either side of its threshold at B = 3, ns = nr = 300 (2.5 x 1800 node rows = 4500 edge rows): split (node
    projections in tc_rowlinear_kernel, then the K = 64 edge GEMM) for 2600 edges, K = 192 on raw gathered rows
    (tc_edge_kernel) for 1000."""
    B, ns, nr = 3, 300, 300
    for ne, split in ((2600, True), (1000, False)):
        ei = _graph(ns, nr, ne, 1, sort=True)
        for upd, aggr in ((True, "sum"), (False, "mean")):
            torch.manual_seed(0)
            net = nlb.InteractionNet(ei, 64, update_edges=upd, aggr=aggr, math="tf32")
            send, edge = torch.randn(B, ns, 64), torch.randn(B, ne, 64)
            want = rp.interaction_net({k: v.double() for k, v in net.state_dict().items()}, ei, send.double(), send.double(),
                                      edge.double(), aggr=aggr, update_edges=upd)
            net = net.to(DEV)
            with torch.no_grad(), ops.profile_launches() as prof:
                got = net(send.to(DEV), send.to(DEV), edge.to(DEV))
            edge_label = "tc_edge3_kernel" if upd else "tc_edge_rmw_kernel"
            labels = ["tc_rowlinear_kernel", edge_label] if split else ["tc_edge_kernel"]
            assert prof.names() == labels + ["tc_rowmlp_kernel"], (ne, upd, prof.names())
            got = got if isinstance(got, tuple) else (got,)
            want = want if isinstance(want, tuple) else (want,)
            err = max((a.double().cpu() - b).abs().max().item() for a, b in zip(got, want))
            assert err < 1e-2, (ne, upd, err)


def _ell_graph(ns, nr, d, seed):
    """Every receiver has exactly d incoming edges (mesh->grid: d = 4, mesh-down: d = 1)."""
    g = torch.Generator().manual_seed(seed)
    rcv = torch.arange(nr).repeat_interleave(d)
    snd = torch.randint(0, ns, (nr * d,), generator=g)
    return torch.stack([snd, rcv])


ELL_CASES = [
    # name, ns, nr, d, B, aggr, expanded edge, broadcast receivers
    # at most 128 distinct senders per 128 receivers: gathered sender rows repeat within and across neighbouring tiles
    ("win_d4", 50, 30, 4, 2, "sum", False, False),
    ("win_d4_mean_tail", 100, 1000, 4, 3, "mean", False, False),
    ("win_d1_always", 5000, 128 * 20 + 5, 1, 2, "sum", False, False),
    ("win_d8_bcast_rec", 64, 300, 8, 2, "sum", False, True),
    ("win_multi_tile_per_cta", 120, 128 * 150 + 17, 4, 2, "sum", True, False),
    # random senders out of thousands: nearly every gathered sender row is a different one
    ("gather_d5", 2000, 128 * 150 + 17, 5, 2, "sum", False, False),
    ("gather_d2_B1", 4000, 129, 2, 1, "mean", False, False),
    ("gather_d3_expand", 3000, 500, 3, 3, "sum", True, False),
]


@pytest.mark.parametrize("case", ELL_CASES, ids=[c[0] for c in ELL_CASES])
def test_uniform_degree_edge_path_vs_oracle(case):
    """Uniform in-degree edge sets with update_edges=False take the uniform-degree edge path (tc_ell_window_kernel)."""
    name, ns, nr, d, B, aggr, expand, bcast = case
    ei = _ell_graph(ns, nr, d, 1)
    torch.manual_seed(0)
    net = nlb.InteractionNet(ei, 64, update_edges=False, aggr=aggr, math="tf32")
    with torch.no_grad():
        for p in net.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    send = torch.randn(B, ns, 64)
    rec = torch.randn(1 if bcast else B, nr, 64)
    edge = torch.randn(1 if expand else B, nr * d, 64)
    sd = dict(net.state_dict())
    sd64 = {k: v.double() for k, v in sd.items()}
    sdg = {k: v.to(DEV) for k, v in sd.items()}

    def f64():
        return rp.interaction_net(sd64, ei, send.double(), rec.double().expand(B, -1, -1),
                                  edge.double().expand(B, -1, -1), aggr=aggr, update_edges=False)

    def fgpu():
        return rp.interaction_net(sdg, ei.to(DEV), send.to(DEV), rec.to(DEV).expand(B, -1, -1),
                                  edge.to(DEV).expand(B, -1, -1), aggr=aggr, update_edges=False)

    ref_err, want = _ref_tf32_err(f64, fgpu)
    net = net.to(DEV)
    graph = net._graph(next(net.parameters()).device)
    assert graph.uniform_degree == d
    with torch.no_grad(), ops.profile_launches() as prof:
        got = net(send.to(DEV), rec.to(DEV).expand(B, -1, -1), edge.to(DEV).expand(B, -1, -1))
    assert "tc_ell_window_kernel" in prof.names(), prof.names()
    err = (got.double().cpu() - want[0]).abs().max().item()
    assert err <= ABS_TOL, (name, err)
    assert err <= max(3 * ref_err, 4e-3), (name, err, ref_err)


@pytest.mark.parametrize("with_boundary", [False, True])
def test_fused_output_map_step_epilogue(with_boundary):
    """nlam_rowmlp_step_fwd: output_map + rescale + residual (+ boundary mix) in one launch (reference
    graph/base.py:322-342, forecasters/autoregressive.py:128-131) against the fp64 formula on the oracle MLP."""
    torch.manual_seed(0)
    B, G, D = 3, 128 * 40 + 12, 17
    m = nlb.make_mlp([64, 64, D], layer_norm=False)
    x, prev, bnd = torch.randn(B, G, 64), torch.randn(B, G, D), torch.randn(B, G, D)
    mask = (torch.rand(G) < 0.3).float()
    std, mean = torch.rand(D) + 0.5, torch.randn(D)
    y = rp.mlp(x.double(), {f"m.{k}": v.double() for k, v in m.state_dict().items()}, "m", layer_norm=False)
    want = prev.double() + (y * std.double() + mean.double())
    if with_boundary:
        mk = mask.double()[None, :, None]
        want = mk * bnd.double() + (1 - mk) * want
    m = m.to(DEV)
    n0 = _lib.lib().nlam_launch_count()
    with torch.no_grad():
        got = ops.rowmlp_step(m, x.to(DEV), prev.to(DEV), bnd.to(DEV) if with_boundary else None,
                              mask.to(DEV) if with_boundary else None, std.to(DEV), mean.to(DEV))
    assert got is not None, "the TF32 path must fuse this shape"
    assert _lib.lib().nlam_launch_count() == n0 + 1
    err = (got.double().cpu() - want).abs().max().item()
    assert err <= ABS_TOL, err
    if with_boundary:  # boundary nodes are copied exactly
        sel = mask.bool()
        assert torch.equal(got.cpu()[:, sel], bnd[:, sel])
    # the exact-fp32 mode does not fuse: callers fall back to the two kernels
    assert ops.rowmlp_step(m, x.to(DEV), prev.to(DEV), None, None, std.to(DEV), mean.to(DEV), flags=_lib.MATH_FP32) is None


RMW_CASES = [
    # name, n nodes, n edges, B
    ("small_b1", 60, 500, 1),
    ("ragged_b3", 300, 2600, 3),
    ("empty_receivers", 900, 5000, 2),
    ("many_items", 4000, 36000, 5),   # > 148 work items: CTA ranges start in the middle of a tile's batches
    ("deg100", 40, 4000, 4),
]


@pytest.mark.parametrize("case", RMW_CASES, ids=[c[0] for c in RMW_CASES])
def test_inplace_edge_update_kernel(case):
    """tc_edge_rmw_kernel: e += m written over the edge tensor (edge_out aliases edge) and the no-edge-output
    mode, against the out-of-place kernel (tc_edge3_kernel) on the same inputs and against the fp64 oracle."""
    name, nn_, ne, B = case
    ei = _graph(nn_, nn_, ne, 3, True)
    if name == "empty_receivers":  # two thirds of the nodes receive nothing
        gen = torch.Generator().manual_seed(3)
        ei = torch.stack([torch.randint(0, nn_, (ne,), generator=gen), 3 * torch.randint(0, nn_ // 3, (ne,), generator=gen)])
        ei[1, -1] = nn_ - 1
        ei = ei[:, torch.sort(ei[1], stable=True).indices]
    torch.manual_seed(1)
    net = nlb.InteractionNet(ei, 64, update_edges=True, math="tf32")
    with torch.no_grad():
        for p in net.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    x = torch.randn(B, nn_, 64)
    edge = torch.randn(B, ne, 64)
    want = rp.interaction_net({k: v.double() for k, v in net.state_dict().items()}, ei, x.double(), x.double(),
                              edge.double(), update_edges=True)
    net = net.to(DEV)
    g = net._graph(torch.device(DEV, torch.cuda.current_device()))
    xs, e0 = x.to(DEV), edge.to(DEV)
    flags = net._flags()
    with torch.no_grad():
        with ops.profile_launches() as prof:
            rec_a, edge_a, _ = ops.inet_fwd(g, net.edge_mlp, net.aggr_mlp, xs, xs, e0, True, flags)  # out of place
        assert "tc_edge3_kernel" in prof.names(), prof.names()
        e_in = e0.clone()
        with ops.profile_launches() as prof:
            rec_b, edge_b, _ = ops.inet_fwd(g, net.edge_mlp, net.aggr_mlp, xs, xs, e_in, True, flags, edge_inplace=True)
        assert "tc_edge_rmw_kernel" in prof.names(), prof.names()
        assert edge_b.data_ptr() == e_in.data_ptr()
        with ops.profile_launches() as prof:
            rec_c, edge_c, _ = ops.inet_fwd(g, net.edge_mlp, net.aggr_mlp, xs, xs, e0, False, flags)  # no edge output
        assert "tc_edge_rmw_kernel" in prof.names() and edge_c is None
    torch.cuda.synchronize()
    # same TF32 products; only fp32 summation orders differ between the kernels
    assert (edge_b - edge_a).abs().max().item() <= 2e-5
    # (the aggregates differ in their last bits, which can flip the TF32 rounding of the node update's inputs)
    assert (rec_b - rec_a).abs().max().item() <= 2e-3
    assert (rec_c - rec_a).abs().max().item() <= 2e-3
    err = max((rec_b.double().cpu() - want[0]).abs().max().item(), (edge_b.double().cpu() - want[1]).abs().max().item())
    assert err <= ABS_TOL, (name, err)
    # a batch-broadcast edge tensor can not be updated in place: the library must refuse the alias
    if B > 1:
        eb = e0[:1].expand(B, -1, -1)
        with torch.no_grad():
            _, edge_d, _ = ops.inet_fwd(g, net.edge_mlp, net.aggr_mlp, xs, xs, eb, True, flags, edge_inplace=True)
        assert edge_d.data_ptr() != eb.data_ptr()


def test_stack_updates_private_edge_tensor_in_place():
    """GNNSequential with keep_edge_rep=False (GraphLAM.process_step): first layer out of place (its input is the
    caller's), middle layers in place, last layer without edge output — same values as the plain layer-by-layer
    evaluation, input untouched."""
    from neural_lam_b200.networks import make_gnn_seq
    ei = _graph(500, 500, 4500, 5, True)
    torch.manual_seed(2)
    seq = make_gnn_seq(ei, 4, 1, 64).to(DEV)
    x = torch.randn(3, 500, 64, device=DEV)
    e_static = torch.randn(1, 4500, 64, device=DEV)
    e_in = e_static.expand(3, -1, -1)
    keep = e_static.clone()
    with torch.no_grad():
        want, _ = seq(x, e_in, keep_edge_rep=True)
        with ops.profile_launches() as prof:
            got, e_none = seq(x, e_in, keep_edge_rep=False)
    assert e_none is None
    assert prof.names().count("tc_edge_rmw_kernel") == 3 and prof.names().count("tc_edge3_kernel") == 1, prof.names()
    # the node kernel of layers 1-3 also computes the next layer's node projections: one projection launch (layer 1)
    # and one plain node update (layer 4) remain
    assert prof.names().count("tc_node_proj_kernel") == 3 and prof.names().count("tc_rowlinear_kernel") == 1, prof.names()
    assert len(prof.names()) == 9, prof.names()
    assert torch.equal(e_static, keep)
    assert (got - want).abs().max().item() <= 5e-3


@pytest.mark.parametrize("with_boundary,B,G", [(True, 3, 1000), (False, 1, 128), (True, 2, 40 * 128 + 36)])
def test_chained_node_update_output_map_step_epilogue(with_boundary, B, G):
    """tc_node_out_kernel: node update of the mesh->grid layer + output_map + forecast-step epilogue in one launch, against the
    two-kernel path (row-kernel node update, then output_map + epilogue) on the same inputs: same TF32 products, same fp32
    formulas — the intermediate only stays in shared memory."""
    from neural_lam_b200.networks import make_mlp
    torch.manual_seed(3)
    ei = _graph(50, G, 4 * G, 2, True)
    net = nlb.InteractionNet(ei, 64, update_edges=False, math="tf32").to(DEV)
    out_map = make_mlp([64, 64, 17], layer_norm=False).to(DEV)
    with torch.no_grad():
        for p in list(net.parameters()) + list(out_map.parameters()):
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    rec = torch.randn(B, G, 64, device=DEV)
    aggr = torch.randn(B, G, 64, device=DEV)
    prev = torch.randn(B, G, 17, device=DEV)
    bnd = torch.randn(B, G, 17, device=DEV) if with_boundary else None
    mask = (torch.rand(G, 1, device=DEV) < 0.3).float() if with_boundary else None
    std, mean = torch.rand(17, device=DEV) + 0.5, torch.randn(17, device=DEV)
    with torch.no_grad():
        with ops.profile_launches() as prof:
            got = ops.node_update_step(net.aggr_mlp, out_map, rec, aggr, prev, bnd, mask, std, mean)
        assert got is not None and prof.names() == ["tc_node_out_kernel"], prof.names()
        grid2 = net._kernel_node_update(rec, aggr)
        want = ops.rowmlp_step(out_map, grid2, prev, bnd, mask, std, mean)
        assert want is not None
    torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-6)
    # and against plain torch in fp64 (TF32 tolerance)
    sd = {k: v.double().cpu() for k, v in net.state_dict().items()}
    x = torch.cat([rec, aggr], -1).double().cpu()
    h = torch.nn.functional.silu(x @ sd["aggr_mlp.0.weight"].T + sd["aggr_mlp.0.bias"])
    y = torch.nn.functional.layer_norm(h @ sd["aggr_mlp.2.weight"].T + sd["aggr_mlp.2.bias"], (64,),
                                       sd["aggr_mlp.3.weight"], sd["aggr_mlp.3.bias"])
    g2 = rec.double().cpu() + y
    od = {k: v.double().cpu() for k, v in out_map.state_dict().items()}
    o = torch.nn.functional.silu(g2 @ od["0.weight"].T + od["0.bias"]) @ od["2.weight"].T + od["2.bias"]
    new = prev.double().cpu() + o * std.double().cpu() + mean.double().cpu()
    if with_boundary:
        m = mask.double().cpu()
        new = m * bnd.double().cpu() + (1 - m) * new
    assert (got.double().cpu() - new).abs().max().item() < 2e-2


@pytest.mark.parametrize("cls_name,H", [("InteractionNet", 64), ("PropagationNet", 64), ("InteractionNet", 128)])
def test_split_mlps_layer_on_tensor_cores(cls_name, H):
    """SplitMLPs layers (reference gnn_layers.py:274-324; HiLAMParallel's per-level MLPs): every chunk's edge MLP runs as
    gather-pack + two launches of the generic wgmma Linear kernel, the node MLPs on the row-MLP kernels — no SIMT math."""
    cls = getattr(nlb, cls_name)
    ns, nr, ne, B = 70, 50, 600, 2
    ei = _graph(ns, nr, ne, 4, False)  # chunks are defined on the layer's own (unsorted) edge order
    torch.manual_seed(5)
    ech, ach = [250, 350], [20, 30]
    net = cls(ei, H, edge_chunk_sizes=ech, aggr_chunk_sizes=ach, math="tf32")
    send, rec, edge = torch.randn(B, ns, H), torch.randn(B, nr, H), torch.randn(B, ne, H)
    prop = cls_name == "PropagationNet"
    want = rp.interaction_net({k: v.double() for k, v in net.state_dict().items()}, ei, send.double(), rec.double(),
                              edge.double(), propagation=prop, aggr="mean" if prop else "sum",
                              edge_chunk_sizes=ech, aggr_chunk_sizes=ach)
    net = net.to(DEV)
    with torch.no_grad(), ops.profile_launches() as prof:
        got = net(send.to(DEV), rec.to(DEV), edge.to(DEV))
    assert not any("simt" in n for n in prof.names()), prof.names()
    assert any(n.startswith("tc_linear") for n in prof.names()), prof.names()
    err = max((g.double().cpu() - w).abs().max().item() for g, w in zip(got, want))
    assert err <= 2e-2, err


@pytest.mark.parametrize("B,N", [(1, 100), (3, 500), (2, 128 * 3 + 5)])
def test_node_kernel_with_next_layer_projections(B, N):
    """tc_node_proj_kernel through nlam_inet_fwd_chain: layer 1 produces the node projections of layer 2's edge MLP in its node kernel, layer
    2 consumes them — against the unchained calls on the same inputs (same TF32 products: results agree to fp32 rounding)."""
    ei = _graph(N, N, 9 * N, 7, True)
    torch.manual_seed(4)
    l1 = nlb.InteractionNet(ei, 64, math="tf32").to(DEV)
    l2 = nlb.InteractionNet(ei, 64, math="tf32").to(DEV)
    with torch.no_grad():
        for p in list(l1.parameters()) + list(l2.parameters()):
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    x = torch.randn(B, N, 64, device=DEV)
    e = torch.randn(B, 9 * N, 64, device=DEV)
    with torch.no_grad():
        x1, e1 = l1(x, x, e)
        x2, e2 = l2(x1, x1, e1)
        with ops.profile_launches() as prof:
            y1, f1, proj = l1.forward_stacked(x, e.clone(), first=True, last=False, next_layer=l2)
            assert proj is not None and proj.shape == (2, B, N, 64)
            y2, f2, none = l2.forward_stacked(y1, f1, first=False, last=True, proj_in=proj)
        assert none is None and f2 is None
    assert prof.names().count("tc_node_proj_kernel") == 1 and prof.names().count("tc_rowlinear_kernel") == 1, prof.names()
    assert (y1 - x1).abs().max().item() <= 1e-5 and (f1 - e1).abs().max().item() <= 1e-5
    assert (y2 - x2).abs().max().item() <= 2e-3
    # the projections themselves against fp64
    w = l2.edge_mlp[0].weight.double().cpu()
    b = l2.edge_mlp[0].bias.double().cpu()
    ps = y1.double().cpu() @ w[:, 64:128].T
    pr = y1.double().cpu() @ w[:, 128:192].T + b
    assert (proj[0].double().cpu() - ps).abs().max().item() <= 1e-2
    assert (proj[1].double().cpu() - pr).abs().max().item() <= 1e-2
