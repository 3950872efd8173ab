"""Graph-EFM oracle pinning on the CPU: the restatement ``oracle/efm_port`` against golden vectors produced by the
reference's own ``graph_efm.py`` + ``models/latent/*.py`` (``oracle/gen_golden_efm.py``), strict loading of the reference
state_dicts into ``GraphEFMMultiScale``, and the model's host-side checks."""
import pytest
import torch

from efm_golden_util import load_efm_cases
from neural_lam_b200 import models, synthetic
from oracle import efm_port

CASES = load_efm_cases()


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_efm_port_matches_reference_golden(case):
    _, ds, model = case.build()
    params, g, cfg = case.oracle_inputs(model, ds)
    with torch.no_grad():
        out = efm_port.efm_step(params, g, cfg, case.prev_state, case.prev_prev_state, case.forcing, case.eps)
        post_mean, post_std = efm_port.efm_posterior(params, g, cfg, case.prev_state, case.prev_prev_state, case.forcing,
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


def test_efm_port_gradients_match_reference_golden():
    """The port under autograd (fp32) reproduces the reference's parameter gradients of the case with gradients."""
    case = next(c for c in CASES if c.grads)
    _, ds, model = case.build()
    params, g, cfg = case.oracle_inputs(model, ds)
    params = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in params.items()}
    out = efm_port.efm_step(params, g, cfg, case.prev_state, case.prev_prev_state, case.forcing, case.eps)
    pm, ps = efm_port.efm_posterior(params, g, cfg, case.prev_state, case.prev_prev_state, case.forcing, case.target)
    loss = (out["pred"] * case.w_pred).sum() + (pm * case.w_post).sum() + (ps * case.w_post).sum()
    loss.backward()
    assert set(case.grads) == {k for k, p in params.items() if p.grad is not None}
    for k, want in case.grads.items():
        got = params[k].grad
        scale = want.abs().max().item()
        assert (got - want).abs().max().item() <= 1e-4 * scale + 1e-6, k


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_efm_state_dict_matches_reference(case):
    """Parameter and persistent-buffer names and shapes are the reference's (strict load in ``case.build``)."""
    _, _, model = case.build()
    assert set(model.state_dict()) == set(case.params)
    for k, v in model.state_dict().items():
        assert v.shape == case.params[k].shape, k


def test_efm_structure():
    spec = synthetic.make_graph_spec(30, 27, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1)
    m = models.GraphEFMMultiScale(ds, spec, prior_m2m_layers=0, decoder_m2m_layers=0, encoder_m2m_layers=3)
    assert m.prior_model.m2m_gnns is None and m.decoder.m2m_gnns is None and len(m.encoder.m2m_gnns) == 3
    assert m.latent_dim == 64 and m.latent_spatial_dim == m.num_mesh_nodes == spec["mesh_static_features"].shape[0]
    assert m.prior_model.latent_param_map[-1].out_features == 64 and m.encoder.latent_param_map[-1].out_features == 128
    assert "GraphEFMMultiScale" not in {c.__name__ for c in models.MODELS.values()}
    c = models.GraphEFMMultiScale(ds, spec, learn_prior=False, latent_dim=8, prior_dist="diagonal")
    assert isinstance(c.prior_model, models.ConstantLatentEncoder) and not list(c.prior_model.parameters())
    with pytest.raises(ValueError, match="flat mesh"):
        models.GraphEFMMultiScale(ds, synthetic.make_graph_spec(30, 27, hierarchical=True), hidden_dim=16)
    with pytest.raises(ValueError, match="output distribution"):
        models.GraphEFMMultiScale(ds, spec, prior_dist="laplace")
