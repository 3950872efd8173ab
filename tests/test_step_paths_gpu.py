"""The no-grad forecast step takes one encoder path and one decoder path whichever entry runs it (`-m gpu`): the eager
``forward`` and ``forward_with_boundary`` without a boundary (the step a captured rollout replays) launch the same kernels
and compute the same bits, for GraphLAM on a uniform and a non-uniform m2g graph and with clamped outputs, and for
GraphEFMMultiScale and GraphEFM with a learned and a constant prior.  Each case also pins the launch that starts the step
(the fused encoder, where the model has a g2m layer for it) and the one that ends it: tc_decode_kernel (uniform m2g
in-degree), tc_node_out_kernel (non-uniform), the step epilogue kernels (clamped outputs, a predicted std; the model with a
predicted std has no boundary step to compare)."""
import pytest
import torch

from neural_lam_b200 import models, ops, synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda"
D_STATE, D_FORCING, D_STATIC = 17, 18, 4  # 56 input columns: the fused encoder covers them
EFM_MS = dict(prior_m2m_layers=1, encoder_m2m_layers=1, decoder_m2m_layers=1)
EFM_HI = dict(prior_intra_level_layers=1, encoder_intra_level_layers=1, decoder_intra_level_layers=1)
CLAMP = dict(output_clamping_lower={"var0": -10.0, "var1": -10.0}, output_clamping_upper={"var0": 10.0, "var2": 10.0})

# name: (model class, hierarchical graph, uniform m2g in-degree, model kwargs, first launch (None: no fused encoder), last)
CASES = {
    "graph_lam_uniform": (models.GraphLAM, False, True, {}, "tc_encode_kernel", "tc_decode_kernel"),
    "graph_lam_non_uniform": (models.GraphLAM, False, False, {}, "tc_encode_kernel", "tc_node_out_kernel"),
    "graph_lam_clamped": (models.GraphLAM, False, True, CLAMP, "tc_encode_kernel", "step_epilogue_clamped_kernel"),
    "graph_lam_std": (models.GraphLAM, False, True, dict(output_std=True), "tc_encode_kernel", "step_epilogue_kernel"),
    "efm_ms_learned": (models.GraphEFMMultiScale, False, True, EFM_MS, "tc_encode_kernel", "tc_decode_kernel"),
    "efm_ms_constant": (models.GraphEFMMultiScale, False, True, dict(EFM_MS, learn_prior=False), None, "tc_decode_kernel"),
    "efm_hi_learned": (models.GraphEFM, True, True, EFM_HI, "tc_encode2_kernel", "tc_decode_kernel"),
    "efm_hi_constant": (models.GraphEFM, True, True, dict(EFM_HI, learn_prior=False), "tc_encode_kernel", "tc_decode_kernel"),
}


def _model(cls, hierarchical, uniform, kw):
    # 31 x 26: every grid node has a g2m edge, so the fused encoder covers the grid
    spec = dict(synthetic.make_graph_spec(31, 26, hierarchical=hierarchical))
    if not uniform:  # receiver 0 keeps 3 of its 4 m2g edges, the rest 4
        spec["m2g_edge_index"] = spec["m2g_edge_index"][:, 1:].contiguous()
        spec["m2g_features"] = spec["m2g_features"][1:].contiguous()
    ds = synthetic.SyntheticDatastore(spec, d_state=D_STATE, d_forcing=D_FORCING, d_static=D_STATIC, boundary_width=2)
    torch.manual_seed(0)
    m = cls(ds, spec, hidden_dim=64, **kw).to(DEV).eval()
    assert (m.m2g_gnn if hasattr(m, "m2g_gnn") else m.decoder.m2g_gnn)._graph(torch.device(DEV)).uniform_degree == 4 * uniform
    return m


@pytest.mark.parametrize("name", list(CASES))
def test_eager_and_boundary_steps_take_one_path(name):
    cls, hierarchical, uniform, kw, first, last = CASES[name]
    m = _model(cls, hierarchical, uniform, kw)
    B, G = 2, m.num_grid_nodes
    gen = torch.Generator(device=DEV).manual_seed(1)
    prev, prev_prev = torch.randn(B, G, D_STATE, device=DEV, generator=gen), torch.randn(B, G, D_STATE, device=DEV, generator=gen)
    forcing = torch.randn(B, G, D_FORCING, device=DEV, generator=gen)
    noise = {}
    if getattr(m, "samples_latent", False):
        noise["latent_noise"] = torch.randn(B, m.latent_spatial_dim, m.latent_dim, device=DEV, generator=gen)
    with torch.no_grad():
        m.static_embeddings()  # the weight-only embeddings are cached outside the compared steps
        with ops.profile_launches() as prof:
            state, pred_std = m(prev, prev_prev, forcing, **noise)
        names = prof.names()
        assert names[-1] == last, names
        if first:
            assert names[0] == first, names
        else:
            assert not any(n.startswith("tc_encode") for n in names), names
        assert (pred_std is not None) == m.output_std
        if m.output_std:
            return
        with ops.profile_launches() as prof:
            state2 = m.forward_with_boundary(prev, prev_prev, forcing, None, None, **noise)
    assert prof.names() == names, (names, prof.names())
    assert torch.equal(state2, state), (state2 - state).abs().max().item()
