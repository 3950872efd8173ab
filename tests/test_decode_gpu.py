"""The fused mesh -> grid decoder (``ops.decode_step``: tc_rowlinear_kernel for the edge projections, then tc_decode_kernel
for the edge MLP, the per-receiver aggregation, the node update, output_map and the forecast-step epilogue).

Bounds:
  * against the fp64 oracle: |err| <= max(3 x the error of the reference's own TF32 GPU configuration, 4e-3) and <= 1e-2
    (DESIGN.md §2, as in test_tc_kernels.py);
  * against the three-launch path (edge-only InteractionNet, then tc_node_out_kernel) on the same inputs: 2e-3.  Both
    compute the same TF32 products; the fused kernel adds P_e + P_s + P_r and the d messages of a receiver in another
    order, and a last-bit difference of the aggregate can flip the TF32 rounding of a node-MLP operand (one TF32 ulp,
    2^-11 relative, of an O(1) input);
  * the operand rounding: ||got - ref_rna|| <= 0.6 ||got - ref_rz|| on tailed operands (test_tf32_rounding_gpu.py B).
"""
import pytest
import torch

import neural_lam_b200 as nlb
from neural_lam_b200 import models, ops, synthetic
from neural_lam_b200.networks import make_mlp
from oracle import reference_port as rp
from test_tc_kernels import _ell_graph, _graph
from test_tf32_rounding_gpu import RATIO, _inputs, _p64, _tail_params

pytestmark = pytest.mark.gpu
DEV = "cuda"
ABS_TOL = 1e-2
VS_OLD_TOL = 2e-3
D = 17
DECODER = ["tc_rowlinear_kernel", "tc_decode_kernel"]


def _setup(ei, ns, nr, B, aggr="sum", boundary=True, seed=0, tailed=False, d_out=D, send_rows=None, bcast=()):
    """``send_rows``: rows of the sender tensor (default ``ns``); ``bcast``: inputs ("send", "rec") given as a stride-0
    expansion of one batch element"""
    torch.manual_seed(seed)
    net = nlb.InteractionNet(ei, 64, update_edges=False, aggr=aggr, math="tf32")
    out_map = make_mlp([64, 64, d_out], layer_norm=False)
    ne = ei.shape[1]
    shapes = [(B, send_rows or ns, 64), (B, nr, 64), (1, ne, 64), (B, nr, d_out), (B, nr, d_out)]
    if tailed:
        _tail_params(net, seed + 1)
        _tail_params(out_map, seed + 2)
        send, rec, edge, prev, bnd = _inputs(shapes, seed + 3)
    else:
        with torch.no_grad():
            for p in list(net.parameters()) + list(out_map.parameters()):
                if p.dim() == 1:
                    p.add_(0.1 * torch.randn_like(p))
        send, rec, edge, prev, bnd = (torch.randn(sh) for sh in shapes)
    send = send[:1].expand(B, -1, -1) if "send" in bcast else send
    rec = rec[:1].expand(B, -1, -1) if "rec" in bcast else rec
    gen = torch.Generator().manual_seed(seed + 4)
    mask = (torch.rand(nr, generator=gen) < 0.3).float()
    std, mean = torch.rand(d_out, generator=gen) + 0.5, torch.randn(d_out, generator=gen)
    return dict(ei=ei, B=B, aggr=aggr, net=net, out_map=out_map, send=send, rec=rec, edge=edge, prev=prev,
                bnd=bnd if boundary else None, mask=mask if boundary else None, std=std, mean=mean)


def _oracle(c, dev, dtype):
    """the decoder through the oracle's op sequence (fp64 on the CPU, or the reference's fp32 GPU configuration)"""
    pn = {k: v.to(dev, dtype) for k, v in _p64(c["net"]).items()}
    po = {k: v.to(dev, dtype) for k, v in _p64(c["out_map"], "m").items()}
    t = {k: c[k].to(dev, dtype) for k in ("send", "rec", "edge", "prev", "std", "mean")}
    grid = rp.interaction_net(pn, c["ei"].to(dev), t["send"], t["rec"], t["edge"].expand(c["B"], -1, -1), aggr=c["aggr"],
                              update_edges=False)
    new = t["prev"] + rp.mlp(grid, po, "m", layer_norm=False) * t["std"] + t["mean"]
    if c["bnd"] is not None:
        mk = c["mask"].to(dev, dtype)[None, :, None]
        new = mk * c["bnd"].to(dev, dtype) + (1 - mk) * new
    return new


def _to_dev(t):
    if t is not None and t.dim() == 3 and t.shape[0] > 1 and t.stride(0) == 0:  # a batch broadcast stays one on the device
        return t[:1].to(DEV).expand_as(t)
    return t.to(DEV) if t is not None else None


def _on_gpu(c):
    net, out_map = c["net"].to(DEV), c["out_map"].to(DEV)
    g = {k: _to_dev(c[k]) for k in ("send", "rec", "edge", "prev", "bnd", "mask", "std", "mean")}
    return net, out_map, g


def _fused(c):
    net, out_map, g = _on_gpu(c)
    with torch.no_grad(), ops.profile_launches() as prof:
        got = net.decode_step(g["send"], g["rec"], g["edge"], out_map, g["prev"], g["bnd"], g["mask"], g["std"], g["mean"])
    return got, prof.names()


def _three_launches(c):
    """the decoder as the model ran it before: edge-only InteractionNet (projections + tc_ell_window_kernel), then
    tc_node_out_kernel"""
    net, out_map, g = _on_gpu(c)
    with torch.no_grad(), ops.profile_launches() as prof:
        aggr = net.aggregate_only(g["send"], g["rec"], g["edge"])
        got = ops.node_update_step(net.aggr_mlp, out_map, g["rec"], aggr, g["prev"], g["bnd"], g["mask"], g["std"], g["mean"])
    return got, prof.names()


def test_decode_rounds_operands_to_nearest():
    c = _setup(_ell_graph(100, 1000, 4, 1), 100, 1000, 3, tailed=True, boundary=False)
    got, names = _fused(c)
    assert names == DECODER, names
    with torch.no_grad():
        with rp.tf32_matmul(mode="rna"):
            rna = _oracle(c, "cpu", torch.float64)
        with rp.tf32_matmul(mode="rz"):
            rz = _oracle(c, "cpu", torch.float64)
    got = got.double().cpu()
    d_rna, d_rz = (got - rna).norm().item(), (got - rz).norm().item()
    err = (got - rna).abs().max().item()
    print(f"\ndecode: ||got - ref_rna|| / ||got - ref_rz|| = {d_rna / d_rz:.3f}; max |got - ref_rna| {err:.3e}")
    assert err <= ABS_TOL, err
    assert d_rna <= RATIO * d_rz, (d_rna, d_rz)


CASES = [
    # name, n senders, n receivers, in-degree, B, aggregation, boundary
    ("d1_sum", 300, 1000, 1, 3, "sum", True),
    ("d2_mean_b1", 500, 777, 2, 1, "mean", False),
    ("d4_sum", 200, 1000, 4, 3, "sum", True),
    ("d4_mean_full_items", 200, 64 * 20, 4, 3, "mean", False),
    ("d8_sum_b1", 100, 1000, 8, 1, "sum", True),
    ("d8_mean", 100, 500, 8, 3, "mean", True),
]


def _check_case(name, c):
    """the fused decoder on the inputs of ``_setup`` against the fp64 oracle and the three-launch path; a rerun is equal
    bit for bit and boundary rows are copied exactly"""
    with torch.no_grad():
        want = _oracle(c, "cpu", torch.float64)
        old = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = True
        try:
            ref_err = (_oracle(c, DEV, torch.float32).double().cpu() - want).abs().max().item()
        finally:
            torch.backends.cuda.matmul.allow_tf32 = old
    got, names = _fused(c)
    assert names == DECODER, names
    again, _ = _fused(c)
    assert torch.equal(got, again), "two runs of the fused decoder differ"
    err = (got.double().cpu() - want).abs().max().item()
    old_got, old_names = _three_launches(c)
    assert "tc_decode_kernel" not in old_names and old_names[-1] == "tc_node_out_kernel", old_names
    vs_old = (got - old_got).abs().max().item()
    print(f"\n{name}: max |err| vs fp64 oracle {err:.3e} (reference TF32 configuration {ref_err:.3e}); "
          f"max |fused - three-launch| {vs_old:.3e}")
    assert err <= ABS_TOL, err
    assert err <= max(3 * ref_err, 4e-3), (err, ref_err)
    assert vs_old <= VS_OLD_TOL, vs_old
    if c["bnd"] is not None:  # boundary rows are copied exactly
        sel = c["mask"].bool()
        assert torch.equal(got.cpu()[:, sel], c["bnd"][:, sel])


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_decode_vs_oracle_and_three_launch_path(case):
    name, ns, nr, d, B, aggr, boundary = case
    _check_case(name, _setup(_ell_graph(ns, nr, d, 2), ns, nr, B, aggr=aggr, boundary=boundary))


def _multi_item_shape(B):
    """Receivers for a decoder call at batch B in which every warp group of tc_decode_kernel runs at least 3 items, the last
    round is partial and the last 64-receiver block is partial.  Returns (n_rec, n_items, warp groups of the launch)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_blocks = -(-6 * sms // B)  # 3 items for each of 2 warp groups on every SM
    # a partial last round; an odd item count (odd B) also leaves one warp group of a CTA without a last item
    while (n_blocks * B) % (2 * sms) == 0 or (B % 2 == 1 and n_blocks % 2 == 0):
        n_blocks += 1
    n_items = n_blocks * B
    grid = min((n_items + 1) // 2, sms)  # as tc_decode launches it: CTAs of two warp groups, at most one per SM
    return 64 * (n_blocks - 1) + 37, n_items, 2 * grid


NS_MULTI = 600
MULTI_ITEM = [
    # name, in-degree, B, aggregation
    ("d1_sum_b5", 1, 5, "sum"),
    ("d1_mean_b32", 1, 32, "mean"),
    ("d2_mean_b5", 2, 5, "mean"),
    ("d2_sum_b32", 2, 32, "sum"),
    ("d4_sum_b5", 4, 5, "sum"),
    ("d4_mean_b32", 4, 32, "mean"),
    ("d8_mean_b5", 8, 5, "mean"),
    ("d8_sum_b32", 8, 32, "sum"),
]


@pytest.mark.parametrize("case", MULTI_ITEM, ids=[c[0] for c in MULTI_ITEM])
def test_decode_multi_item(case):
    """Every warp group runs several items: the cross-item prefetch of receiver rows and sender indices, the reuse of the
    warp group's named barriers and shared operands by later items, and a partial receiver block that is not a warp
    group's first item.  Items run batch-fastest (item i: block i / B, batch element i % B) on warp group i % groups."""
    name, d, B, aggr = case
    nr, n_items, groups = _multi_item_shape(B)
    assert n_items // groups >= 3, (n_items, groups)  # the fewest items a warp group runs
    assert n_items % groups != 0 and nr % 64 != 0 and n_items - B >= groups, (nr, n_items, groups)
    assert B % 2 == 0 or n_items % 2 == 1
    print(f"\n{name}: {nr} receivers, {n_items} items on {groups} warp groups")
    _check_case(name, _setup(_ell_graph(NS_MULTI, nr, d, 4), NS_MULTI, nr, B, aggr=aggr))


@pytest.mark.parametrize("B", [5, 32])
def test_decode_multi_item_batch_permutation(B):
    """Permuting the batch permutes the output bit for bit (the decoder has no reduction across the batch)."""
    nr, _, _ = _multi_item_shape(B)
    c = _setup(_ell_graph(NS_MULTI, nr, 4, 5), NS_MULTI, nr, B)
    perm = torch.arange(B).flip(0).roll(2)
    assert not torch.equal(perm, torch.arange(B))
    got, names = _fused(c)
    assert names == DECODER, names
    got_p, _ = _fused(dict(c, **{k: c[k][perm] for k in ("send", "rec", "prev", "bnd")}))
    want = got[perm.to(DEV)]
    bad = [b for b in range(B) if not torch.equal(got_p[b], want[b])]
    assert not bad, f"permuted positions {bad} differ (max |diff| {(got_p - want).abs().max().item():.3e})"


CALL_SHAPES = [
    # name, options of _setup
    ("bcast_send", dict(bcast=("send",))),
    ("bcast_rec", dict(bcast=("rec",))),
    ("bcast_send_rec", dict(bcast=("send", "rec"))),
    ("send_rows_n_send_plus_37", dict(send_rows=300 + 37)),
    ("d_out_1", dict(d_out=1)),
    ("d_out_63", dict(d_out=63)),
]


@pytest.mark.parametrize("case", CALL_SHAPES, ids=[c[0] for c in CALL_SHAPES])
def test_decode_call_shapes(case):
    """Call shapes tc_decode handles with code of its own: stride-0 senders (one P_s for the batch) and receivers (P_r and
    the residual from one element), a sender tensor with more rows than the graph's senders, and the narrowest and widest
    output the kernel accepts (D < 64; columns >= D of the last bias are zero-padded)."""
    name, kw = case
    ns, nr, B = 300, 777, 5
    c = _setup(_ell_graph(ns, nr, 4, 6), ns, nr, B, **kw)
    _check_case(name, c)
    _, _, g = _on_gpu(c)
    for k in kw.get("bcast", ()):
        assert g[k].stride(0) == 0, k
    assert c["net"]._graph(g["rec"].device).n_send == ns
    assert g["send"].shape[1] == kw.get("send_rows", ns) and g["prev"].shape[2] == kw.get("d_out", D)


@pytest.mark.parametrize("kind", ["degree3", "non_uniform", "halo"])
def test_decode_falls_back_where_not_covered(kind):
    """decode_step returns None for graphs the kernel does not cover; the three-launch path still runs there."""
    if kind == "non_uniform":
        ei, ns, nr = _graph(200, 300, 1200, 3, True), 200, 300
    else:
        ei, ns, nr = _ell_graph(200, 300, 3 if kind == "degree3" else 4, 3), 200, 300
    c = _setup(ei, ns, nr, 2)
    if kind == "halo":  # node-partitioned rollout: the sender rows pass through a halo exchange (dist.partition_model)
        c["net"]._halo = lambda x: x
    got, names = _fused(c)
    assert got is None and names == [], names
    if kind == "halo":
        return
    old_got, old_names = _three_launches(c)
    assert old_names[-1] == "tc_node_out_kernel" and "tc_decode_kernel" not in old_names, old_names
    assert kind != "degree3" or "tc_ell_window_kernel" in old_names, old_names
    want = _oracle(c, "cpu", torch.float64)
    assert (old_got.double().cpu() - want).abs().max().item() <= ABS_TOL


def test_model_step_runs_fused_decoder():
    """A small GraphLAM (H = 64) forecast step: the decoder is tc_decode_kernel, the CUDA-graph replay equals the eager step
    (as in test_models.py), and the rollout stays within the TF32 bound of the fp64 oracle."""
    from test_models import _oracle_graph

    spec = synthetic.make_graph_spec(30, 27, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1, boundary_width=2)
    torch.manual_seed(1)
    m = models.GraphLAM(ds, spec, hidden_dim=64, processor_layers=2)
    fc = models.ARForecaster(m, ds)
    g = _oracle_graph(m, fc)
    cfg = dict(model="graph_lam", hidden_layers=1, processor_layers=2, mesh_aggr="sum")
    G, B, T = m.num_grid_nodes, 3, 2
    gen = torch.Generator().manual_seed(5)
    init, forc, bnd = torch.randn(B, 2, G, 5, generator=gen), torch.randn(B, T, G, 6, generator=gen), torch.randn(B, T, G, 5,
                                                                                                               generator=gen)
    params = {f"predictor.{k}": v.double() for k, v in m.state_dict().items()}
    want = rp.ar_rollout(params, g, cfg, init.double(), forc.double(), bnd.double())
    fc = fc.to(DEV).eval()
    assert m.m2g_gnn._graph(torch.device(DEV, torch.cuda.current_device())).uniform_degree == 4
    with torch.no_grad():
        got, _ = fc(init.to(DEV), forc.to(DEV), bnd.to(DEV))
        with ops.profile_launches() as prof:
            got2, _ = fc(init.to(DEV), forc.to(DEV), bnd.to(DEV))
        graphed = fc.rollout_graphed(init.to(DEV), forc.to(DEV), bnd.to(DEV))
    names = prof.names()
    assert names.count("tc_decode_kernel") == T, names
    assert "tc_ell_window_kernel" not in names and "tc_node_out_kernel" not in names, names
    torch.testing.assert_close(got2, got, rtol=0, atol=0)
    torch.testing.assert_close(graphed, got, rtol=1e-6, atol=1e-6)
    err = (got.cpu().double() - want).abs().max().item()
    print(f"\nGraphLAM 30x27 H=64, {T} steps: max |err| vs fp64 oracle {err:.3e}")
    assert err < 2e-2, err


def test_model_step_falls_back_on_non_uniform_m2g_graph():
    """A GraphLAM whose m2g graph is not uniform (one receiver with 3 of its 4 edges): ``forward_with_boundary`` runs the
    three-launch decoder (tc_ell_window_kernel is not used either: the edge stage takes the general CSR kernels), and the
    captured rollout stays within the TF32 bound of the fp64 oracle."""
    from test_models import _oracle_graph

    spec = dict(synthetic.make_graph_spec(30, 27, hierarchical=False))
    assert torch.equal(spec["m2g_edge_index"][1, :4], torch.zeros(4, dtype=spec["m2g_edge_index"].dtype))
    spec["m2g_edge_index"] = spec["m2g_edge_index"][:, 1:].contiguous()  # receiver 0 keeps 3 edges, the rest 4
    spec["m2g_features"] = spec["m2g_features"][1:].contiguous()
    ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1, boundary_width=2)
    torch.manual_seed(1)
    m = models.GraphLAM(ds, spec, hidden_dim=64, processor_layers=2)
    fc = models.ARForecaster(m, ds)
    g = _oracle_graph(m, fc)
    cfg = dict(model="graph_lam", hidden_layers=1, processor_layers=2, mesh_aggr="sum")
    G, B, T = m.num_grid_nodes, 2, 2
    gen = torch.Generator().manual_seed(6)
    init, forc, bnd = torch.randn(B, 2, G, 5, generator=gen), torch.randn(B, T, G, 6, generator=gen), torch.randn(B, T, G, 5,
                                                                                                               generator=gen)
    want = rp.ar_rollout({f"predictor.{k}": v.double() for k, v in m.state_dict().items()}, g, cfg, init.double(),
                         forc.double(), bnd.double())
    fc = fc.to(DEV).eval()
    assert m.m2g_gnn._graph(torch.device(DEV, torch.cuda.current_device())).uniform_degree == 0
    with torch.no_grad():
        m.static_embeddings()
        with ops.profile_launches() as prof:
            m.forward_with_boundary(init[:, 1].to(DEV), init[:, 0].to(DEV), forc[:, 0].to(DEV), bnd[:, 0].to(DEV),
                                    fc.boundary_mask)
        graphed = fc.rollout_graphed(init.to(DEV), forc.to(DEV), bnd.to(DEV))
    names = prof.names()
    assert "tc_decode_kernel" not in names and "tc_ell_window_kernel" not in names, names
    assert names[-1] == "tc_node_out_kernel", names
    err = (graphed.cpu().double() - want).abs().max().item()
    print(f"\nGraphLAM 30x27, non-uniform m2g: max |err| vs fp64 oracle {err:.3e}; last launches {names[-3:]}")
    assert err < 2e-2, err
