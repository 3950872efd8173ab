"""Hierarchical Graph-EFM oracle pinning on the CPU: the restatement in ``oracle/efm_hi_port`` against golden vectors produced
by the reference's own ``GraphEFM`` + ``models/latent/hi_graph_*.py`` (``oracle/gen_golden_efm_hi.py``), strict loading of
the reference state_dicts into ``models.GraphEFM``, its submodule structure and the graph-type checks."""
import pytest
import torch

from efm_hi_golden_util import load_efm_hi_cases
from neural_lam_b200 import latent, models, synthetic
from neural_lam_b200.gnn_layers import InteractionNet, PropagationNet
from oracle import efm_hi_port

CASES = load_efm_hi_cases()


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_efm_hi_port_matches_reference_golden(case):
    _, ds, model = case.build()
    params, g, cfg = case.oracle_inputs(model, ds)
    with torch.no_grad():
        out = efm_hi_port.efm_hi_step(params, g, cfg, case.prev_state, case.prev_prev_state, case.forcing, case.eps)
        post_mean, post_std = efm_hi_port.efm_hi_posterior(params, g, cfg, case.prev_state, case.prev_prev_state, case.forcing,
                                                        case.target)
    tol = dict(rtol=2e-5, atol=2e-5)
    torch.testing.assert_close(out["prior_mean"], case.prior_mean, **tol)
    torch.testing.assert_close(out["prior_std"], case.prior_std, **tol)
    torch.testing.assert_close(out["pred"], case.pred, **tol)
    if case.pred_std is None:
        assert out["pred_std"] is None
    else:
        torch.testing.assert_close(out["pred_std"], case.pred_std, **tol)
    torch.testing.assert_close(post_mean, case.post_mean, **tol)
    torch.testing.assert_close(post_std, case.post_std, **tol)


def test_efm_hi_port_gradients_match_reference_golden():
    """The port under autograd (fp32) reproduces the reference's parameter gradients of the case with gradients."""
    case = next(c for c in CASES if c.grads)
    _, ds, model = case.build()
    params, g, cfg = case.oracle_inputs(model, ds)
    params = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in params.items()}
    out = efm_hi_port.efm_hi_step(params, g, cfg, case.prev_state, case.prev_prev_state, case.forcing, case.eps)
    pm, ps = efm_hi_port.efm_hi_posterior(params, g, cfg, case.prev_state, case.prev_prev_state, case.forcing, case.target)
    loss = (out["pred"] * case.w_pred).sum() + (pm * case.w_post).sum() + (ps * case.w_post).sum()
    loss.backward()
    assert set(case.grads) == {k for k, p in params.items() if p.grad is not None}
    for k, want in case.grads.items():
        got = params[k].grad
        scale = want.abs().max().item()
        assert (got - want).abs().max().item() <= 1e-4 * scale + 1e-6, k


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_efm_hi_state_dict_matches_reference(case):
    """Parameter and persistent-buffer names and shapes are the reference's (strict load in ``case.build``)."""
    _, _, model = case.build()
    assert set(model.state_dict()) == set(case.params)
    for k, v in model.state_dict().items():
        assert v.shape == case.params[k].shape, k
    assert model.embedd_m2m == any(k.startswith("m2m_embedders.") for k in case.params)


def test_efm_hi_port_runs_in_fp64_and_tf32():
    """The hierarchical oracle runs in fp64 and under ``tf32_matmul()``; both stay close to the fp32 golden."""
    from oracle import reference_port as rp

    case = next(c for c in CASES if c.grads)
    _, ds, model = case.build()
    params, g, cfg = case.oracle_inputs(model, ds)
    p64 = {k: v.double() if v.is_floating_point() else v for k, v in params.items()}
    x = (case.prev_state, case.prev_prev_state, case.forcing)
    with torch.no_grad():
        want = efm_hi_port.efm_hi_step(p64, g, cfg, *[t.double() for t in x], case.eps.double())["pred"]
        with rp.tf32_matmul():
            tf32 = efm_hi_port.efm_hi_step(params, g, cfg, *x, case.eps)["pred"]
    assert want.dtype == torch.float64
    assert (want - case.pred.double()).abs().max().item() <= 1e-4
    assert 0 < (tf32.double() - want).abs().max().item() <= 5e-2


def test_efm_hi_structure():
    spec = synthetic.make_graph_spec(84, 82, hierarchical=True)
    ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1)
    m = models.GraphEFM(ds, spec, hidden_dim=16, prior_intra_level_layers=0, encoder_intra_level_layers=3,
                        decoder_intra_level_layers=2)
    L = len(spec["mesh_static_features"])
    assert L == 3 and m.num_levels == 3
    assert m.latent_spatial_dim == spec["mesh_static_features"][-1].shape[0] == 9
    assert m.num_mesh_nodes == sum(f.shape[0] for f in spec["mesh_static_features"])
    assert len(m.mesh_embedders) == L and len(m.mesh_up_embedders) == len(m.mesh_down_embedders) == L - 1
    assert m.embedd_m2m and len(m.m2m_embedders) == L
    prior, enc, dec = m.prior_model, m.encoder, m.decoder
    assert isinstance(prior, latent.HiGraphLatentEncoder) and prior.intra_level_gnns is None
    assert isinstance(enc, latent.HiGraphLatentEncoder) and enc.output_dist == "diagonal"
    assert len(enc.intra_level_gnns) == L and all(len(s) == 3 for s in enc.intra_level_gnns)
    assert all(type(u) is PropagationNet and not u.update_edges for u in enc.mesh_up_gnns) and len(enc.mesh_up_gnns) == L - 1
    assert isinstance(dec, latent.HiGraphLatentDecoder)
    assert all(type(u) is InteractionNet and not u.update_edges for u in dec.mesh_up_gnns)
    assert all(type(d) is PropagationNet and not d.update_edges for d in dec.mesh_down_gnns)
    assert len(dec.intra_up_gnns) == L and len(dec.intra_down_gnns) == L - 1
    assert not dec.g2m_gnn.update_edges and not dec.m2g_gnn.update_edges
    assert m.encoder.latent_param_map[-1].out_features == 32 and prior.latent_param_map[-1].out_features == 16
    names = {n.split(".")[0] for n, _ in m.named_parameters()}
    assert names == {"grid_prev_embedder", "grid_current_embedder", "g2m_embedder", "m2g_embedder", "prior_model",
                     "mesh_embedders", "mesh_up_embedders", "mesh_down_embedders", "m2m_embedders", "encoder", "decoder"}
    assert "GraphEFM" not in {c.__name__ for c in models.MODELS.values()}
    c = models.GraphEFM(ds, spec, hidden_dim=16, latent_dim=8, learn_prior=False, prior_intra_level_layers=0,
                        encoder_intra_level_layers=0, decoder_intra_level_layers=0)
    assert isinstance(c.prior_model, models.ConstantLatentEncoder) and c.prior_model.num_mesh_nodes == 9
    assert not c.embedd_m2m and not hasattr(c, "m2m_embedders")
    assert c.encoder.intra_level_gnns is None and c.decoder.intra_up_gnns is None and c.decoder.intra_down_gnns is None


def test_efm_hi_graph_type_checks():
    flat = synthetic.make_graph_spec(30, 27, hierarchical=False)
    hi = synthetic.make_graph_spec(30, 27, hierarchical=True)
    ds = synthetic.SyntheticDatastore(flat, d_state=5, d_forcing=6, d_static=1)
    with pytest.raises(ValueError, match="hierarchical mesh"):
        models.GraphEFM(ds, flat, hidden_dim=16)
    with pytest.raises(ValueError, match="flat mesh"):
        models.GraphEFMMultiScale(ds, hi, hidden_dim=16)
    one = models.GraphEFM(ds, hi, hidden_dim=16)
    with pytest.raises(ValueError, match="at least 2 mesh levels"):
        latent.HiGraphLatentEncoder(8, one.g2m_edge_index, one.m2m_edge_index[:1], one.mesh_up_edge_index[:0], 16, 1)
    with pytest.raises(ValueError, match="at least 2 mesh levels"):
        latent.HiGraphLatentDecoder(one.g2m_edge_index, one.m2m_edge_index[:1], one.m2g_edge_index, [], [], 16, 8, 5, 1)


def test_efm_hi_noise_shape_is_top_level():
    spec = synthetic.make_graph_spec(30, 27, hierarchical=True)
    ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1)
    m = models.GraphEFM(ds, spec, hidden_dim=16, latent_dim=8)
    eps = torch.zeros(2, 9, 8)
    assert m._noise(eps, 2, "cpu") is eps
    with pytest.raises(ValueError, match="latent_noise"):
        m._noise(torch.zeros(2, m.num_mesh_nodes, 8), 2, "cpu")
