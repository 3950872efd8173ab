"""The ensemble statistics' definitions (DESIGN §4.5) on the CPU: the fp64 oracle ``oracle/ensemble_port.py`` against
independent statements of the same quantities, the derived scores of ``ensemble.EnsembleScores``, and the argument checks
that need no device.

* the pairwise mean pair difference D equals the sorted form 2 Σ (2i - K - 1) x_(i) / (K(K-1)), tied members included;
* crps_ecdf = A - (K-1)/(2K) · D equals the exact integral ∫ (F_K(z) - 1{z >= y})² dz of the members' empirical CDF;
* the fair CRPS A - D/2 of 4 096 draws from N(μ, σ) is within 4 standard errors of the closed form the reference's
  ``crps_gauss`` (metrics.py:371-382) states;
* hand-computed K = 2 values.
"""
import math

import pytest
import torch

from neural_lam_b200 import ensemble, models, synthetic
from oracle import ensemble_port as ep


def _ecdf_crps(x, y):
    """∫ (F_K(z) - 1{z >= y})² dz, exactly: F_K and the step are constant between consecutive points of x ∪ {y}"""
    K = len(x)
    pts = sorted(list(x) + [y])
    total = 0.0
    for a, b in zip(pts[:-1], pts[1:]):
        if b > a:
            F = sum(1 for v in x if v <= a) / K
            H = 1.0 if a >= y else 0.0
            total += (F - H) ** 2 * (b - a)
    return total


def _members(K, G=40, d=3, ties=True, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, K, G, d, generator=g, dtype=torch.float64)
    if ties:  # a few points with tied members: some pairs, and one point with every member equal
        x[:, K // 2] = x[:, 0]
        x[:, :, 0, 0] = 0.25
        x[0, :, 1, 1] = torch.tensor([1.0, -1.0] * (K // 2) + [1.0] * (K % 2), dtype=torch.float64)
    y = torch.randn(2, G, d, generator=g, dtype=torch.float64)
    return x, y


@pytest.mark.parametrize("K", [2, 3, 8, 64])
def test_pair_diff_pairwise_equals_sorted_form(K):
    x, y = _members(K)
    got = ep.point_stats(x, y)["pair_diff"]
    want = ep.pair_diff_sorted(x)
    assert (got - want).abs().max().item() < 1e-12
    assert got[:, 0, 0].abs().max().item() == 0.0  # all members equal


@pytest.mark.parametrize("K", [2, 3, 8, 64])
def test_crps_ecdf_equals_the_empirical_cdf_integral(K):
    x, y = _members(K, G=6, d=2, seed=K)
    s = ep.point_stats(x, y)
    crps = s["abs_err"] - (K - 1) / (2 * K) * s["pair_diff"]
    for b in range(2):
        for g in range(6):
            for v in range(2):
                want = _ecdf_crps(x[b, :, g, v].tolist(), y[b, g, v].item())
                assert abs(crps[b, g, v].item() - want) < 1e-12, (b, g, v)


def test_fair_crps_of_gaussian_draws_matches_closed_form():
    mu, sigma, y, K = 0.3, 1.7, 1.1, 4096
    x = mu + sigma * torch.randn(1, K, 1, 1, generator=torch.Generator().manual_seed(7), dtype=torch.float64)
    s = ep.point_stats(x, torch.full((1, 1, 1), y, dtype=torch.float64))
    fair = (s["abs_err"] - s["pair_diff"] / 2).item()
    # closed form of the reference's crps_gauss (metrics.py:371-382): σ [z (2Φ(z) - 1) + 2 φ(z) - 1/√π], z = (y - μ)/σ
    z = (y - mu) / sigma
    pdf, cdf = math.exp(-z * z / 2) / math.sqrt(2 * math.pi), 0.5 * (1 + math.erf(z / math.sqrt(2)))
    want = sigma * (z * (2 * cdf - 1) + 2 * pdf - 1 / math.sqrt(math.pi))
    # standard error of the U-statistic from its first-order projection h(x_k) = |x_k - y| - E|x_k - X|
    xs = x.reshape(-1)
    h = (xs - y).abs() - (xs[:, None] - xs[None, :]).abs().mean(dim=1)
    se = h.std().item() / math.sqrt(K)
    assert abs(fair - want) < 4 * se, (fair, want, se)


def test_k2_hand_computed():
    x = torch.tensor([[[[1.0, 0.0]], [[3.0, 1.0]]]], dtype=torch.float64)  # (B=1, K=2, G=1, d=2)
    y = torch.tensor([[[2.0, 3.0]]], dtype=torch.float64)
    mean, std, means = ep.ensemble_stats(x, torch.ones(1), y)
    assert mean.tolist() == [[[2.0, 0.5]]]
    assert torch.allclose(std, torch.tensor([[[2.0 ** 0.5, 0.5 ** 0.5]]], dtype=torch.float64))
    # [SE, s², A, D]: v = 0: (0, 2, 1, 2); v = 1: (6.25, 0.5, 2.5, 1)
    assert means.tolist() == [[[0.0, 2.0, 1.0, 2.0], [6.25, 0.5, 2.5, 1.0]]]
    sc = ensemble.EnsembleScores.from_means(means, 2)
    assert sc.crps_fair.tolist() == [[0.0, 2.0]]
    assert sc.crps_ecdf.tolist() == [[0.5, 2.25]]
    for v, yv in enumerate((2.0, 3.0)):
        assert abs(sc.crps_ecdf[0, v].item() - _ecdf_crps(x[0, :, 0, v].tolist(), yv)) < 1e-15
    assert sc.rmse.tolist() == [[0.0, 2.5]]
    assert torch.allclose(sc.ssr[0, 1], torch.tensor(1.5 ** 0.5 * 0.5 ** 0.5 / 2.5, dtype=torch.float64))


def test_interior_mean_and_derived_scores():
    K = 8
    x, y = _members(K, G=50, d=4, ties=False, seed=3)
    mask = torch.zeros(50, dtype=torch.bool)
    mask[7:41] = True
    _, _, means = ep.ensemble_stats(x, mask, y)
    s = ep.point_stats(x, y)
    assert torch.allclose(means[..., 2], s["abs_err"][:, 7:41].mean(dim=1), rtol=1e-14, atol=0)
    sc = ensemble.EnsembleScores.from_means(means, K)
    ref = ep.derived(means, K)
    for name in ("rmse", "spread", "ssr", "crps_fair", "crps_ecdf"):
        assert torch.allclose(getattr(sc, name), ref[name], rtol=1e-14, atol=0), name


def test_argument_checks_without_a_device():
    x = torch.randn(1, 4, 10, 2)
    with pytest.raises(ValueError):
        ensemble.ensemble_stats(torch.randn(1, 1, 10, 2), torch.ones(10))
    with pytest.raises(ValueError):
        ensemble.ensemble_stats(torch.randn(1, 65, 10, 2), torch.ones(10))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ensemble.ensemble_stats(x, torch.ones(10))


def test_rollout_ensemble_argument_checks():
    spec = synthetic.make_graph_spec(12, 10, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=3, d_forcing=2, d_static=1, boundary_width=2)
    G = ds.boundary_mask.numel()
    init, forc, bnd = torch.zeros(1, 2, G, 3), torch.zeros(1, 2, G, 2), torch.zeros(1, 2, G, 3)
    fc = models.ARForecaster(models.GraphLAM(ds, spec, hidden_dim=32, processor_layers=1), ds)
    with pytest.raises(ValueError, match="samples its latent"):
        fc.rollout_ensemble(init, forc, bnd, 4)
    efm = models.ARForecaster(models.GraphEFMMultiScale(ds, spec, hidden_dim=32, prior_m2m_layers=1, decoder_m2m_layers=1), ds)
    for bad in (1, 0, 65, 2.0, True):
        with pytest.raises(ValueError, match="members"):
            efm.rollout_ensemble(init, forc, bnd, bad)
    with pytest.raises(ValueError, match="boundary_states"):
        efm.rollout_ensemble(init, forc, bnd[:, :1], 4)
    with pytest.raises(ValueError, match="init_states"):
        efm.rollout_ensemble(init[:, :1], forc, bnd, 4)
    with pytest.raises(ValueError, match="targets"):
        efm.rollout_ensemble(init, forc, bnd, 4, targets=bnd[..., :2])
