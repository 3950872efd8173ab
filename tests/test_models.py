"""Step-predictor / forecaster parity: GraphLAM and HiLAM forward + AR rollout on the GPU
against the CPU oracle (oracle/reference_port.py restating graph/base.py, graph_lam.py,
hierarchical.py, hi_lam.py, autoregressive.py), plus CPU-side structure checks."""
import pytest
import torch

from neural_lam_b200 import models, synthetic
from oracle import reference_port as rp


def _oracle_graph(model, forecaster=None):
    g = {}
    for k in ("grid_static_features", "g2m_features", "m2g_features", "g2m_edge_index", "m2g_edge_index",
              "diff_std", "diff_mean"):
        g[k] = getattr(model, k).detach().cpu()
    for k in ("m2m_features", "m2m_edge_index", "mesh_static_features", "mesh_up_features", "mesh_up_edge_index",
              "mesh_down_features", "mesh_down_edge_index"):
        if hasattr(model, k):
            v = getattr(model, k)
            g[k] = [t.detach().cpu() for t in v] if isinstance(v, models.BufferList) else v.detach().cpu()
    if forecaster is not None:
        g["boundary_mask"] = forecaster.boundary_mask.detach().cpu()
    return g


def _build(kind, hidden=16, P=2, math="fp32", **kw):
    if kind == "graph_lam":
        spec = synthetic.make_graph_spec(16, 16, hierarchical=False, n_levels=1)
        ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1, boundary_width=1)
        torch.manual_seed(42)
        model = models.GraphLAM(ds, spec, hidden_dim=hidden, processor_layers=P, math=math, **kw)
    elif kind == "graph_lam_multiscale":
        spec = synthetic.make_graph_spec(30, 27, hierarchical=False)
        ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1, boundary_width=2)
        torch.manual_seed(42)
        model = models.GraphLAM(ds, spec, hidden_dim=hidden, processor_layers=P, math=math, **kw)
    else:
        spec = synthetic.make_graph_spec(30, 27, hierarchical=True)
        ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1, boundary_width=2)
        torch.manual_seed(42)
        model = models.HiLAM(ds, spec, hidden_dim=hidden, processor_layers=P, math=math, **kw)
    return spec, ds, model


def test_parameter_names_match_reference_layout():
    _, _, m = _build("graph_lam")
    keys = set(m.state_dict())
    for k in ("grid_embedder.0.weight", "g2m_embedder.2.bias", "m2g_embedder.3.weight", "g2m_gnn.edge_mlp.0.weight",
              "g2m_gnn.aggr_mlp.3.bias", "encoding_grid_mlp.0.weight", "m2g_gnn.aggr_mlp.0.weight",
              "output_map.2.weight", "mesh_embedder.0.weight", "m2m_embedder.0.weight",
              "processor.module_0.edge_mlp.0.weight", "processor.module_1.aggr_mlp.2.bias"):
        assert k in keys, k
    assert not any("edge_index" in k or "features" in k for k in keys)  # graph tensors are non-persistent
    assert m.state_dict()["grid_embedder.0.weight"].shape == (16, 17)  # 2*5 + 1 + 6
    assert m.state_dict()["output_map.2.weight"].shape == (5, 16)
    _, _, h = _build("hi_lam")
    hk = set(h.state_dict())
    for k in ("mesh_embedders.1.0.weight", "mesh_same_embedders.0.0.weight", "mesh_up_embedders.0.0.weight",
              "mesh_down_embedders.0.3.bias", "mesh_init_gnns.0.edge_mlp.0.weight", "mesh_read_gnns.0.aggr_mlp.0.weight",
              "mesh_down_gnns.1.0.edge_mlp.0.weight", "mesh_down_same_gnns.0.1.aggr_mlp.3.weight",
              "mesh_up_gnns.0.0.edge_mlp.2.weight", "mesh_up_same_gnns.1.0.edge_mlp.3.bias"):
        assert k in hk, k
    # 2 + 2(L-1) + P(4L-2) InteractionNets per step (SURVEY.md a13): L=2, P=2 -> 16
    n_gnn = sum(1 for mod in h.modules() if type(mod).__name__ in ("InteractionNet", "PropagationNet"))
    assert n_gnn == 2 + 2 * 1 + 2 * (4 * 2 - 2)


def test_oracle_models_run_on_cpu():
    """The oracle itself (pure CPU) runs both model families and the AR loop."""
    for kind in ("graph_lam", "hi_lam"):
        _, ds, m = _build(kind)
        fc = models.ARForecaster(m, ds)
        g = _oracle_graph(m, fc)
        cfg = dict(model=kind, hidden_layers=1, processor_layers=2, mesh_aggr="sum")
        G = m.num_grid_nodes
        gen = torch.Generator().manual_seed(123)
        init = torch.randn(2, 2, G, 5, generator=gen)
        forc = torch.randn(2, 2, G, 6, generator=gen)
        bnd = torch.randn(2, 2, G, 5, generator=gen)
        out = rp.ar_rollout({f"predictor.{k}": v for k, v in m.state_dict().items()}, g, cfg, init, forc, bnd)
        assert out.shape == (2, 2, G, 5) and torch.isfinite(out).all()
        bm = g["boundary_mask"].bool().squeeze(-1)
        torch.testing.assert_close(out[:, 0][:, bm], bnd[:, 0][:, bm])  # boundary overwritten by truth


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["graph_lam", "graph_lam_multiscale", "hi_lam"])
def test_step_and_rollout_match_oracle_fp32(kind):
    _, ds, m = _build(kind)
    fc = models.ARForecaster(m, ds)
    g = _oracle_graph(m, fc)
    cfg = dict(model="hi_lam" if kind == "hi_lam" else "graph_lam", hidden_layers=1, processor_layers=2, mesh_aggr="sum")
    G = m.num_grid_nodes
    gen = torch.Generator().manual_seed(123)
    B, T = 2, 2
    init = torch.randn(B, 2, G, 5, generator=gen)
    forc = torch.randn(B, T, G, 6, generator=gen)
    bnd = torch.randn(B, T, G, 5, generator=gen)
    params = {f"predictor.{k}": v for k, v in m.state_dict().items()}
    want = rp.ar_rollout(params, g, cfg, init, forc, bnd)
    want64 = rp.ar_rollout({k: v.double() for k, v in params.items()}, g, cfg, init.double(), forc.double(), bnd.double())
    fc = fc.to("cuda")
    with torch.no_grad():
        got, std = fc(init.cuda(), forc.cuda(), bnd.cuda())
        got_graphed = fc.rollout_graphed(init.cuda(), forc.cuda(), bnd.cuda())
    assert std is None
    # tolerance: fp32 kernels vs fp32 oracle after 2 AR steps through up to 16 stacked layers
    torch.testing.assert_close(got.cpu(), want, rtol=2e-4, atol=2e-4)
    torch.testing.assert_close(got_graphed.cpu(), got.cpu(), rtol=1e-6, atol=1e-6)
    # public host-buffer API (pinned in, pinned out, PCIe copies overlapped with the kernels)
    T5 = 5
    forc5, bnd5 = torch.randn(B, T5, G, 6, generator=gen).pin_memory(), torch.randn(B, T5, G, 5, generator=gen).pin_memory()
    with torch.no_grad():
        host = fc.rollout_from_host(init.pin_memory(), forc5, bnd5)
        ref5 = fc.rollout_graphed(init.cuda(), forc5.cuda(), bnd5.cuda())
    assert not host.is_cuda
    torch.testing.assert_close(host, ref5.cpu(), rtol=0, atol=0)
    # slices along T of pinned tensors take the same strided-copy path (one copy per tensor and step, boundary rows only)
    out3 = torch.empty(B, T5, G, 5).pin_memory()
    with torch.no_grad():
        fc.rollout_from_host(init.pin_memory(), forc5[:, 2:], bnd5[:, 2:], out=out3[:, :3])
        ref3 = fc.rollout_graphed(init.cuda(), forc5[:, 2:].cuda(), bnd5[:, 2:].cuda())
    torch.testing.assert_close(out3[:, :3], ref3.cpu(), rtol=0, atol=0)
    err64 = (got.cpu().double() - want64).abs().max().item()
    ref64 = (want.double() - want64).abs().max().item()
    assert err64 < max(10 * ref64, 2e-4), (err64, ref64)


@pytest.mark.gpu
def test_training_step_gradients_match_oracle():
    """Backward through a whole GraphLAM step (recompute-in-backward) vs autograd on the oracle."""
    _, ds, m = _build("graph_lam")
    g = _oracle_graph(m)
    cfg = dict(model="graph_lam", hidden_layers=1, processor_layers=2, mesh_aggr="sum")
    G = m.num_grid_nodes
    gen = torch.Generator().manual_seed(5)
    prev, pprev, forc = torch.randn(2, G, 5, generator=gen), torch.randn(2, G, 5, generator=gen), torch.randn(2, G, 6, generator=gen)
    w = torch.randn(2, G, 5, generator=gen)
    params = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v.clone()) for k, v in m.state_dict().items()}
    out = rp.graph_model_forward(params, g, cfg, prev, pprev, forc)
    (out * w).sum().backward()
    m = m.cuda()
    got, _ = m(prev.cuda(), pprev.cuda(), forc.cuda())
    torch.testing.assert_close(got.detach().cpu(), out.detach(), rtol=1e-4, atol=1e-4)
    (got * w.cuda()).sum().backward()
    for k, p in m.named_parameters():
        assert p.grad is not None, k
        torch.testing.assert_close(p.grad.cpu(), params[k].grad, rtol=2e-3, atol=2e-4, msg=lambda s: f"{k}: {s}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind,hidden", [("hi_lam", 128), ("graph_lam_multiscale", 256)])
def test_wide_hidden_models_run_on_the_generic_tensor_core_path(kind, hidden):
    """BASELINE configs 3-5 use hidden_dim 128 / 256: every per-step launch is the generic wgmma Linear kernel (tc7.cu)
    or an index kernel — no FFMA row-MLP — and the rollout matches the fp64 oracle within the TF32 bound
    (|err| <= max(3 x the reference's TF32 configuration, 1e-2), as in tests/test_real_size.py)."""
    from neural_lam_b200 import ops

    # grid input width 5 + 5 + 6 + 4 = 20 (a multiple of 4, like the MEPS-shaped 56: rows the packed-input path takes)
    spec = synthetic.make_graph_spec(30, 27, hierarchical=(kind == "hi_lam"))
    ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=4, boundary_width=2)
    torch.manual_seed(42)
    m = (models.HiLAM if kind == "hi_lam" else models.GraphLAM)(ds, spec, hidden_dim=hidden, processor_layers=1, math="auto")
    fc = models.ARForecaster(m, ds)
    g = _oracle_graph(m, fc)
    cfg = dict(model="hi_lam" if kind == "hi_lam" else "graph_lam", hidden_layers=1, processor_layers=1, mesh_aggr="sum")
    G = m.num_grid_nodes
    gen = torch.Generator().manual_seed(11)
    B, T = 2, 2
    init, forc, bnd = torch.randn(B, 2, G, 5, generator=gen), torch.randn(B, T, G, 6, generator=gen), torch.randn(B, T, G, 5, generator=gen)
    params = {f"predictor.{k}": v for k, v in m.state_dict().items()}
    with torch.no_grad():
        want64 = rp.ar_rollout({k: v.double() for k, v in params.items()}, g, cfg, init.double(), forc.double(), bnd.double())
        with rp.tf32_matmul():
            ref = rp.ar_rollout(params, g, cfg, init, forc, bnd)
    fc = fc.to("cuda").eval()
    with torch.no_grad():
        got, _ = fc(init.cuda(), forc.cuda(), bnd.cuda())          # first call also fills the static-embedding cache
        with ops.profile_launches() as prof:
            got2, _ = fc(init.cuda(), forc.cuda(), bnd.cuda())
        graphed = fc.rollout_graphed(init.cuda(), forc.cuda(), bnd.cuda())
    names = set(prof.names())
    assert not any("rowmlp_simt" in n for n in names), names
    assert any(n.startswith("tc_linear_kernel") for n in names), names
    torch.testing.assert_close(got2, got, rtol=0, atol=0)
    torch.testing.assert_close(graphed, got, rtol=1e-6, atol=1e-6)
    err = (got.cpu().double() - want64).abs().max().item()
    ref_err = (ref.double() - want64).abs().max().item()
    print(f"{kind} H={hidden}: max |err| vs fp64 oracle {err:.3e} (reference TF32 configuration {ref_err:.3e}); kernels {sorted(names)}")
    assert err <= max(3 * ref_err, 1e-2), (err, ref_err)
