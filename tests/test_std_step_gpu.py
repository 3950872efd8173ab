"""The predicted-std form of the fused forecast-step kernels (``std_out`` of ``ops.decode_step``, ``ops.node_update_step``
and ``ops.rowmlp_step``) and the captured rollouts of models with ``output_std=True`` built on them.

With 2·d outputs y of output_map, outputs c < d take the step epilogue and ``std_out[..., c] = softplus(y[..., d + c])``.
Bounds as in test_decode_gpu.py: against the fp64 oracle max(3 x the reference's TF32 error, 4e-3) and <= 1e-2 for the
kernels; captured against eager 2e-3; the operand rounding ||got - ref_rna|| <= 0.6 ||got - ref_rz||.  The bit identities:
wgmma output columns are independent, so the state columns equal the plain kernel run on the first d rows of the last
Linear, and std_out equals torch's softplus of the plain kernel's raw output of the last d rows.
"""
import pytest
import torch

from neural_lam_b200 import models, ops, synthetic
from neural_lam_b200.networks import make_mlp
from oracle import efm_port
from oracle import reference_port as rp
from model_golden_util import load_model_cases
from test_decode_gpu import DECODER, NS_MULTI, _multi_item_shape, _on_gpu, _setup
from test_models import _oracle_graph
from test_real_size import _check as _check_real_size
from test_tc_kernels import _ell_graph, _graph
from test_tf32_rounding_gpu import RATIO, _p64

pytestmark = pytest.mark.gpu
DEV = "cuda"
ABS_TOL = 1e-2
VS_EAGER_TOL = 2e-3
softplus = torch.nn.functional.softplus


def _std_setup(ei, ns, nr, B, d, big_bias=True, **kw):
    """test_decode_gpu._setup with output_map 64 -> 64 -> 2·d, prev / boundary / diff statistics of d columns; with
    ``big_bias`` the std half of the last bias puts raw outputs above 20 and below -20"""
    c = _setup(ei, ns, nr, B, d_out=2 * d, **kw)
    for k in ("prev", "bnd"):
        if c[k] is not None:
            c[k] = c[k][..., :d].contiguous()
    c["std"], c["mean"], c["d"] = c["std"][:d].contiguous(), c["mean"][:d].contiguous(), d
    if big_bias:
        with torch.no_grad():
            b = c["out_map"][-1].bias
            b[d::3] += 40.0
            b[d + 1::3] -= 40.0
    return c


def _raw_oracle(c, dev, dtype):
    """raw output_map output y (B, nr, 2·d) of the m2g layer through the oracle's op sequence"""
    pn = {k: v.to(dev, dtype) for k, v in _p64(c["net"]).items()}
    po = {k: v.to(dev, dtype) for k, v in _p64(c["out_map"], "m").items()}
    t = {k: c[k].to(dev, dtype) for k in ("send", "rec", "edge")}
    grid = rp.interaction_net(pn, c["ei"].to(dev), t["send"], t["rec"], t["edge"].expand(c["B"], -1, -1), aggr=c["aggr"],
                              update_edges=False)
    return rp.mlp(grid, po, "m", layer_norm=False)


def _oracle(c, dev, dtype):
    """(new state, std) of the std step from the oracle's raw output"""
    y, d = _raw_oracle(c, dev, dtype), c["d"]
    new = c["prev"].to(dev, dtype) + y[..., :d] * c["std"].to(dev, dtype) + c["mean"].to(dev, dtype)
    if c["bnd"] is not None:
        mk = c["mask"].to(dev, dtype)[None, :, None]
        new = mk * c["bnd"].to(dev, dtype) + (1 - mk) * new
    return new, softplus(y[..., d:])


def _run(kind, c, out_map=None, std_out=True, **over):
    """one fused step call of ``kind`` (decode | node | rowmlp) on the inputs of ``c`` (tensors in ``over`` replace
    them) -> (new state, std_out or None, launch names)"""
    net, om, g = _on_gpu(c)
    om = om if out_map is None else out_map.to(DEV)
    g.update({k: (v.to(DEV) if v is not None else None) for k, v in over.items()})
    so = torch.full_like(g["prev"], float("nan")) if std_out else None
    step = (g["prev"], g["bnd"], g["mask"], g["std"], g["mean"])
    with torch.no_grad():
        if kind == "rowmlp":
            grid = net(g["send"], g["rec"], g["edge"].expand(c["B"], -1, -1))
        if kind == "node":
            aggr = net.aggregate_only(g["send"], g["rec"], g["edge"])
        with ops.profile_launches() as prof:
            if kind == "decode":
                got = net.decode_step(g["send"], g["rec"], g["edge"], om, *step, std_out=so)
            elif kind == "node":
                got = ops.node_update_step(net.aggr_mlp, om, g["rec"], aggr, *step, std_out=so)
            else:
                got = ops.rowmlp_step(om, grid, *step, std_out=so)
    return got, so, prof.names()


LAST = {"decode": "tc_decode_kernel", "node": "tc_node_out_kernel", "rowmlp": "tc_rowmlp_kernel"}


def _split_map(out_map, rows):
    """a copy of ``out_map`` whose last Linear keeps output rows ``rows``"""
    m = make_mlp([64, 64, len(range(*rows.indices(out_map[-1].out_features)))], layer_norm=False)
    with torch.no_grad():
        m[0].weight.copy_(out_map[0].weight)
        m[0].bias.copy_(out_map[0].bias)
        m[-1].weight.copy_(out_map[-1].weight[rows])
        m[-1].bias.copy_(out_map[-1].bias[rows])
    return m


def _check(kind, c, name):
    d = c["d"]
    with torch.no_grad():
        want, want_std = _oracle(c, "cpu", torch.float64)
        old = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = True
        try:
            ref, ref_std = _oracle(c, DEV, torch.float32)
        finally:
            torch.backends.cuda.matmul.allow_tf32 = old
    got, got_std, names = _run(kind, c)
    assert got is not None, f"{kind}: the std form is not covered"
    if kind == "decode":
        assert names == DECODER, names
    else:
        assert names[-1] == LAST[kind] and names.count(LAST[kind]) == 1, names
    for what, g_, w, r in (("state", got, want, ref), ("std", got_std, want_std, ref_std)):
        err = (g_.double().cpu() - w).abs().max().item()
        ref_err = (r.double().cpu() - w).abs().max().item()
        print(f"\n{name} {kind} {what}: max |err| vs fp64 oracle {err:.3e} (reference TF32 configuration {ref_err:.3e})")
        assert err <= ABS_TOL, err
        assert err <= max(3 * ref_err, 4e-3), (err, ref_err)
    # the state columns: the plain kernel on the first d output rows, bit for bit
    plain, _, _ = _run(kind, c, out_map=_split_map(c["out_map"], slice(0, d)), std_out=False)
    assert torch.equal(got, plain), (got - plain).abs().max().item()
    # std_out: torch's softplus of the plain kernel's raw output of the last d rows, bit for bit
    zeros = torch.zeros_like(c["prev"])
    raw, _, _ = _run(kind, c, out_map=_split_map(c["out_map"], slice(d, 2 * d)), std_out=False, prev=zeros,
                     std=torch.ones(d), mean=torch.zeros(d), bnd=None, mask=None)
    assert torch.equal(got_std, softplus(raw)), (got_std - softplus(raw)).abs().max().item()
    return raw


DEC_CASES = [
    # name, d, in-degree, B, aggregation, boundary
    ("d1_deg1_sum_bnd", 1, 1, 3, "sum", True),
    ("d17_deg2_mean", 17, 2, 3, "mean", False),
    ("d31_deg4_sum_bnd", 31, 4, 3, "sum", True),
    ("d17_deg8_mean_bnd_b1", 17, 8, 1, "mean", True),
    ("d31_deg8_sum", 31, 8, 3, "sum", False),
    ("d1_deg2_mean_bnd", 1, 2, 3, "mean", True),
]


@pytest.mark.parametrize("case", DEC_CASES, ids=[c[0] for c in DEC_CASES])
def test_decode_std(case):
    name, d, deg, B, aggr, boundary = case
    raw = _check("decode", _std_setup(_ell_graph(300, 1000, deg, 2), 300, 1000, B, d, aggr=aggr, boundary=boundary), name)
    if d > 1:
        assert (raw > 20).any() and (raw < -20).any(), "the softplus threshold is not exercised"


@pytest.mark.parametrize("bcast", [("send",), ("rec",), ("send", "rec")], ids="_".join)
@pytest.mark.parametrize("kind", ["decode", "node", "rowmlp"])
def test_std_batch_broadcast(kind, bcast):
    ei = _ell_graph(300, 777, 4, 6) if kind == "decode" else _graph(300, 777, 3000, 6, True)
    _check(kind, _std_setup(ei, 300, 777, 5, 17, bcast=bcast), f"bcast_{'_'.join(bcast)}")


@pytest.mark.parametrize("B", [5, 32])
@pytest.mark.parametrize("kind", ["decode", "node", "rowmlp"])
def test_std_multi_item(kind, B):
    nr, _, _ = _multi_item_shape(B)
    ei = _ell_graph(NS_MULTI, nr, 4, 4) if kind == "decode" else _graph(NS_MULTI, nr, 4 * nr, 4, True)
    _check(kind, _std_setup(ei, NS_MULTI, nr, B, 17, aggr="mean"), f"multi_item_b{B}")


@pytest.mark.parametrize("d", [1, 17, 31])
@pytest.mark.parametrize("kind", ["node", "rowmlp"])
def test_node_and_rowmlp_std(kind, d):
    """node_update_step after aggregate_only, and rowmlp_step after the whole layer, on a non-uniform graph"""
    _check(kind, _std_setup(_graph(300, 1000, 3500, 3, True), 300, 1000, 3, d, boundary=d != 17), f"d{d}")


@pytest.mark.parametrize("kind", ["decode", "node", "rowmlp"])
def test_d32_is_not_covered(kind):
    ei = _ell_graph(200, 300, 4, 3) if kind == "decode" else _graph(200, 300, 1200, 3, True)
    got, _, names = _run(kind, _std_setup(ei, 200, 300, 2, 32))
    assert got is None and names == [], names


def test_decode_std_rounds_operands_to_nearest():
    c = _std_setup(_ell_graph(100, 1000, 4, 1), 100, 1000, 3, 17, tailed=True, boundary=False, big_bias=False)
    got, got_std, names = _run("decode", c)
    assert names == DECODER, names
    with torch.no_grad():
        with rp.tf32_matmul(mode="rna"):
            rna = torch.cat(_oracle(c, "cpu", torch.float64), -1)
        with rp.tf32_matmul(mode="rz"):
            rz = torch.cat(_oracle(c, "cpu", torch.float64), -1)
    got = torch.cat([got, got_std], -1).double().cpu()
    d_rna, d_rz = (got - rna).norm().item(), (got - rz).norm().item()
    print(f"\ndecode std: ||got - ref_rna|| / ||got - ref_rz|| = {d_rna / d_rz:.3f}")
    assert (got - rna).abs().max().item() <= ABS_TOL
    assert d_rna <= RATIO * d_rz, (d_rna, d_rz)


# ---------------------------------------------------------------------------------------------------------- models
def _spec(kind):
    spec = dict(synthetic.make_graph_spec(30, 27, hierarchical=kind in ("hi_lam", "efm_hi")))
    if kind == "non_uniform":  # receiver 0 keeps 3 of its 4 m2g edges
        spec["m2g_edge_index"] = spec["m2g_edge_index"][:, 1:].contiguous()
        spec["m2g_features"] = spec["m2g_features"][1:].contiguous()
    return spec


EFM_MS = dict(prior_m2m_layers=1, encoder_m2m_layers=1, decoder_m2m_layers=1)
EFM_HI = dict(prior_intra_level_layers=1, encoder_intra_level_layers=1, decoder_intra_level_layers=1)
MODEL_CASES = {
    # name: (model class, kwargs, last launch of the step)
    "uniform": (models.GraphLAM, {}, "tc_decode_kernel"),
    "non_uniform": (models.GraphLAM, {}, "tc_node_out_kernel"),
    "propagation_m2g": (models.GraphLAM, dict(m2g_gnn_type="PropagationNet"), "tc_rowmlp_kernel"),
    "clamped": (models.GraphLAM, dict(output_clamping_lower={"var0": -10.0}, output_clamping_upper={"var2": 10.0}),
                "step_epilogue_clamped_kernel"),
    "hi_lam": (models.HiLAM, {}, None),
}


def _lam(name, output_std=True):
    cls, kw, _ = MODEL_CASES[name]
    spec = _spec(name)
    ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1, boundary_width=2)
    torch.manual_seed(1)
    m = cls(ds, spec, hidden_dim=64, processor_layers=2, output_std=output_std, **kw)
    return m, models.ARForecaster(m, ds), ds


def _inputs_for(m, B, T, seed=5):
    gen = torch.Generator().manual_seed(seed)
    G, d = m.num_grid_nodes, m.num_state_vars
    f = m.grid_input_dim - 2 * d - m.grid_static_features.shape[1]
    return torch.randn(B, 2, G, d, generator=gen), torch.randn(B, T, G, f, generator=gen), torch.randn(B, T, G, d, generator=gen)


@pytest.mark.parametrize("name", list(MODEL_CASES))
def test_model_captured_std_rollout(name):
    m, fc, ds = _lam(name)
    g = _oracle_graph(m, fc)
    cls, kw, last = MODEL_CASES[name]
    cfg = dict(model="hi_lam" if cls is models.HiLAM else "graph_lam", hidden_layers=1, processor_layers=2, mesh_aggr="sum",
               output_std=True, return_std=True, **{k: v for k, v in kw.items() if k.endswith("gnn_type")})
    if name == "clamped":
        cfg["clamp"] = dict(names=list(ds.state_var_names), lower=kw["output_clamping_lower"],
                            upper=kw["output_clamping_upper"], state_mean=ds.state_mean, state_std=ds.state_std)
    B, T = 2, 3
    init, forc, bnd = _inputs_for(m, B, T)
    params = {f"predictor.{k}": v.double() for k, v in m.state_dict().items()}
    want, want_std = rp.ar_rollout(params, g, cfg, init.double(), forc.double(), bnd.double())
    fc = fc.to(DEV).eval()
    x = [t.to(DEV) for t in (init, forc, bnd)]
    with torch.no_grad():
        eager, eager_std = fc(*x)
        so = torch.full((B, T) + tuple(init.shape[2:]), float("nan"), device=DEV)
        graphed = fc.rollout_graphed(*x, std_out=so)
        # the launches of one boundary step: as many as the same model without a std, the last one the fused path's
        m.static_embeddings()
        with ops.profile_launches() as prof:
            m.forward_with_boundary(x[0][:, 1], x[0][:, 0], x[1][:, 0], x[2][:, 0], fc.boundary_mask,
                                    std_out=torch.empty_like(x[0][:, 1]))
        plain, plain_fc, _ = _lam(name, output_std=False)
        plain_fc = plain_fc.to(DEV).eval()
        plain.static_embeddings()
        with ops.profile_launches() as prof_plain:
            plain.forward_with_boundary(x[0][:, 1], x[0][:, 0], x[1][:, 0], x[2][:, 0], plain_fc.boundary_mask)
    names = prof.names()
    if last is not None:
        assert names[-1] == last, names
    assert len(names) == len(prof_plain.names()), (names, prof_plain.names())
    for what, got, e, w in (("pred", graphed, eager, want), ("std", so, eager_std, want_std)):
        vs_eager = (got - e).abs().max().item()
        err = (got.double().cpu() - w).abs().max().item()
        print(f"\n{name} {what}: max |captured - eager| {vs_eager:.3e}, max |err| vs fp64 oracle {err:.3e}")
        assert vs_eager <= VS_EAGER_TOL, vs_eager
        assert err < 2e-2, err
    # the host-buffer API: the same std bit for bit, dense and non-dense host tensors
    with torch.no_grad():
        for dense in (True, False):
            hs = torch.empty(B, T, init.shape[2], init.shape[3] + (0 if dense else 1), pin_memory=True)[..., :init.shape[3]]
            host = fc.rollout_from_host(init.pin_memory(), forc.pin_memory(), bnd.pin_memory(), std_out=hs)
            assert torch.equal(host, graphed.cpu())
            assert torch.equal(hs, so.cpu()), dense


@pytest.mark.parametrize("cls", [models.GraphEFMMultiScale, models.GraphEFM], ids=lambda c: c.__name__)
def test_efm_std_step(cls):
    """Graph-EFM with pinned latent noise: the boundary step's std equals the eager step's and meets the fp64 bound; the
    captured rollout fills std_out."""
    spec = synthetic.make_graph_spec(30, 27, hierarchical=cls is models.GraphEFM)
    ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1, boundary_width=2)
    torch.manual_seed(4)
    m = cls(ds, spec, output_std=True, **(EFM_HI if cls is models.GraphEFM else EFM_MS))
    fc = models.ARForecaster(m, ds)
    params = {k: v.detach().clone() for k, v in m.state_dict().items()}
    m, fc = m.to(DEV).eval(), fc.to(DEV)
    B, G = 2, m.num_grid_nodes
    gen = torch.Generator(device=DEV).manual_seed(1)
    prev, prev_prev = torch.randn(B, G, 5, device=DEV, generator=gen), torch.randn(B, G, 5, device=DEV, generator=gen)
    forcing, bnd = torch.randn(B, G, 6, device=DEV, generator=gen), torch.randn(B, G, 5, device=DEV, generator=gen)
    eps = torch.randn(B, m.latent_spatial_dim, m.latent_dim, device=DEV, generator=gen)
    with torch.no_grad():
        eager, eager_std = m(prev, prev_prev, forcing, latent_noise=eps)
        so = torch.empty_like(prev)
        with ops.profile_launches() as prof:
            new = m.forward_with_boundary(prev, prev_prev, forcing, bnd, fc.boundary_mask, latent_noise=eps, std_out=so)
    assert prof.names()[-1] == "tc_decode_kernel", prof.names()
    mk = fc.boundary_mask.view(1, G, 1)
    assert (new - (mk * bnd + (1 - mk) * eager)).abs().max().item() <= VS_EAGER_TOL
    assert (so - eager_std).abs().max().item() <= VS_EAGER_TOL
    if cls is models.GraphEFMMultiScale:
        g = {k: getattr(m, k).detach() for k in ("grid_static_features", "g2m_features", "m2g_features", "g2m_edge_index",
                                                  "m2g_edge_index", "diff_std", "diff_mean", "m2m_features",
                                                  "m2m_edge_index", "mesh_static_features")}
        cfg = dict(hidden_layers=1, prior_m2m_layers=1, encoder_m2m_layers=1, decoder_m2m_layers=1, output_std=True,
                   num_mesh_nodes=m.num_mesh_nodes, latent_dim=m.latent_dim)
        p64 = {k: v.to(DEV, torch.float64) if v.is_floating_point() else v.to(DEV) for k, v in params.items()}
        want = efm_port.efm_step(p64, g, cfg, prev.double(), prev_prev.double(), forcing.double(), eps.double())
        err = (so.double() - want["pred_std"]).abs().max().item()
        print(f"\n{cls.__name__} std: max |err| vs fp64 oracle {err:.3e}")
        assert err <= ABS_TOL, err
    init, forc, bnds = (torch.randn(B, 2, G, 5, device=DEV), torch.randn(B, 2, G, 6, device=DEV),
                        torch.randn(B, 2, G, 5, device=DEV))
    std_roll = torch.full((B, 2, G, 5), float("nan"), device=DEV)
    fc.rollout_graphed(init, forc, bnds, std_out=std_roll)
    assert torch.isfinite(std_roll).all() and (std_roll > 0).all()


GOLDEN_STD = [c for c in load_model_cases() if c.pred_std is not None]


@pytest.mark.parametrize("case", GOLDEN_STD, ids=[c.name for c in GOLDEN_STD])
def test_reference_golden_std(case):
    """the reference's own std (fp32 on the CPU) from the captured rollout and the host-buffer API (exact fp32 kernels)"""
    _, _, model, fc = case.build(math="fp32")
    fc = fc.to(DEV).eval()
    B, T = case.forcing.shape[:2]
    with torch.no_grad():
        so = torch.empty(case.pred_std.shape, device=DEV)
        pred = fc.rollout_graphed(case.init.to(DEV), case.forcing.to(DEV), case.boundary.to(DEV), std_out=so)
        hs = torch.empty(case.pred_std.shape, pin_memory=True)
        fc.rollout_from_host(case.init.pin_memory(), case.forcing.pin_memory(), case.boundary.pin_memory(), std_out=hs)
    torch.testing.assert_close(pred.cpu(), case.pred, rtol=2e-4, atol=2e-4)
    torch.testing.assert_close(so.cpu(), case.pred_std, rtol=2e-4, atol=2e-4)
    torch.testing.assert_close(hs, case.pred_std, rtol=2e-4, atol=2e-4)


def test_config2_real_size_std_step():
    spec = synthetic.make_graph_spec(268, 238, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=10)
    torch.manual_seed(42)
    model = models.GraphLAM(ds, spec, hidden_dim=64, processor_layers=4, output_std=True)
    fc = models.ARForecaster(model, ds)
    g = _oracle_graph(model, fc)
    cfg = dict(model="graph_lam", hidden_layers=1, processor_layers=4, mesh_aggr="sum", output_std=True, return_std=True)
    init, forc, bnd = _inputs_for(model, 2, 1, seed=123)
    params = {f"predictor.{k}": v for k, v in model.state_dict().items()}
    with torch.no_grad():
        want64 = rp.ar_rollout({k: v.double() for k, v in params.items()}, g, cfg, init.double(), forc.double(), bnd.double())
        with rp.tf32_matmul():
            ref_tf32 = rp.ar_rollout(params, g, cfg, init, forc, bnd)
    fc = fc.to(DEV).eval()
    with torch.no_grad():
        so = torch.empty(bnd.shape, device=DEV)
        got = fc.rollout_graphed(init.to(DEV), forc.to(DEV), bnd.to(DEV), std_out=so).cpu()
    _check_real_size("config 2 GraphLAM output_std, B=2, 1 step: prediction", got, want64[0], ref_tf32[0])
    _check_real_size("config 2 GraphLAM output_std, B=2, 1 step: std", so.cpu(), want64[1], ref_tf32[1])


def test_std_out_errors():
    m, fc, _ = _lam("uniform")
    plain, plain_fc, _ = _lam("uniform", output_std=False)
    m, fc, plain, plain_fc = m.to(DEV), fc.to(DEV), plain.to(DEV), plain_fc.to(DEV)
    init, forc, bnd = (t.to(DEV) for t in _inputs_for(m, 2, 2))
    prev, pp, f0, b0 = init[:, 1], init[:, 0], forc[:, 0], bnd[:, 0]
    with pytest.raises(ValueError, match="std_out"):
        m.forward_with_boundary(prev, pp, f0, b0, fc.boundary_mask)
    with pytest.raises(ValueError, match="does not predict a std"):
        plain.forward_with_boundary(prev, pp, f0, b0, plain_fc.boundary_mask, std_out=torch.empty_like(prev))
    with pytest.raises(ValueError, match="std_out"):
        m.forward_with_boundary(prev, pp, f0, b0, fc.boundary_mask, std_out=torch.empty(2, prev.shape[1], 4, device=DEV))
    with pytest.raises(ValueError, match="std_out"):
        fc.rollout_graphed(init, forc, bnd, std_out=torch.empty(2, 3, *prev.shape[1:], device=DEV))
    with pytest.raises(ValueError, match="std_out"):
        fc.rollout_graphed(init, forc, bnd, std_out=torch.empty(bnd.shape))  # a host tensor
    with pytest.raises(ValueError, match="does not predict a std"):
        plain_fc.rollout_graphed(init, forc, bnd, std_out=torch.empty_like(bnd))
    with pytest.raises(ValueError, match="std_out"):
        fc.rollout_from_host(init.cpu(), forc.cpu(), bnd.cpu(), std_out=torch.empty(2, 2, prev.shape[1], 4))
    with pytest.raises(ValueError, match="does not predict a std"):
        plain_fc.rollout_from_host(init.cpu(), forc.cpu(), bnd.cpu(), std_out=torch.empty(bnd.shape))
    spec = synthetic.make_graph_spec(30, 27, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1, boundary_width=2)
    efm = models.GraphEFMMultiScale(ds, spec, output_std=True, **EFM_MS)
    efc = models.ARForecaster(efm, ds).to(DEV)
    with pytest.raises(ValueError, match="rollout_ensemble"):
        efc.rollout_ensemble(init, forc, bnd, members=2)
