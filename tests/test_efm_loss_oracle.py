"""The fp64 restatement of Graph-EFM's training objective (``oracle/efm_loss_port.py``, DESIGN §4.6) on the CPU.

* the closed-form KL equals ``torch.distributions.kl_divergence`` reduced as defined (sum over the latent dimension, mean
  over the latent nodes) for learned isotropic, learned diagonal and constant priors;
* the restated ``wmse`` / ``nll`` equal the reference's ``neural_lam/metrics.py`` on the stored golden vectors
  (``oracle/gen_golden_efm_loss.py``);
* the closed-form gradient of the ensemble scores (the formulas ``ens_stats_bwd_kernel`` implements) equals fp64 autograd
  through ``ensemble_port.ensemble_stats`` on random data and on ties: duplicated members, members equal to the target,
  all members identical;
* ``efm_loss`` runs on a flat and on a hierarchical golden case, and its terms compose as defined.
"""
import os

import numpy as np
import pytest
import torch
from torch import distributions as tdists

from efm_golden_util import load_efm_cases
from efm_hi_golden_util import load_efm_hi_cases
from oracle import efm_loss_port as lp
from oracle import efm_port
from oracle import ensemble_port as ep

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "efm_loss_metrics.npz")


def _q_and_p(kind, B=3, N=11, L=6, seed=0):
    g = torch.Generator().manual_seed(seed)
    mq, sq = efm_port.mean_std(torch.randn(B, N, 2 * L, generator=g, dtype=torch.float64), "diagonal")
    if kind == "isotropic":
        mp, sp = efm_port.mean_std(torch.randn(B, N, L, generator=g, dtype=torch.float64), "isotropic")
    elif kind == "diagonal":
        mp, sp = efm_port.mean_std(torch.randn(B, N, 2 * L, generator=g, dtype=torch.float64), "diagonal")
    else:  # the constant prior: zero raw parameters
        mp, sp = efm_port.mean_std(torch.zeros(B, N, 2 * L, dtype=torch.float64), "diagonal")
    return mq, sq, mp, sp


@pytest.mark.parametrize("kind", ["isotropic", "diagonal", "constant"])
def test_kl_closed_form_equals_torch_distributions(kind):
    mq, sq, mp, sp = _q_and_p(kind)
    want = tdists.kl_divergence(tdists.Normal(mq, sq), tdists.Normal(mp, sp)).sum(dim=-1).mean(dim=-1)
    got = lp.kl_diag(mq, sq, mp, sp)
    assert got.shape == (3,)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


def test_recon_equals_reference_metrics():
    z = np.load(GOLDEN)
    t = {k: torch.from_numpy(z[k]) for k in z.files}
    torch.testing.assert_close(lp.wmse(t["pred"], t["target"], t["var_std"], mask=t["mask"]), t["wmse"], rtol=1e-12, atol=0)
    torch.testing.assert_close(lp.nll(t["pred"], t["target"], t["std"], mask=t["mask"]), t["nll"], rtol=1e-12, atol=0)


def _autograd_grad(x, mask, y, w):
    x = x.double().clone().requires_grad_()
    _, _, means = ep.ensemble_stats(x, mask, y)
    (means * w).sum().backward()
    return x.grad


def _data(B, K, G, d, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, K, G, d, generator=g, dtype=torch.float64)
    y = torch.randn(B, G, d, generator=g, dtype=torch.float64)
    mask = torch.rand(G, generator=g) > 0.3
    w = torch.randn(B, d, 4, generator=g, dtype=torch.float64)
    return x, y, mask, w


@pytest.mark.parametrize("K", [2, 3, 8])
def test_closed_form_grad_equals_autograd_random(K):
    x, y, mask, w = _data(2, K, 40, 3, seed=K)
    torch.testing.assert_close(lp.ensemble_stats_grad(x, mask, y, w), _autograd_grad(x, mask, y, w), rtol=1e-12, atol=1e-14)


def test_closed_form_grad_equals_autograd_ties():
    B, K, G, d = 2, 6, 40, 3
    x, y, mask, w = _data(B, K, G, d, seed=7)
    x[:, 3:] = x[:, :3]  # every member has a twin
    x[:, 0, :10] = y[:, :10]  # member 0 equals the target on the first nodes
    x[:, :, 20:30] = x[:, :1, 20:30]  # all members identical on these nodes
    torch.testing.assert_close(lp.ensemble_stats_grad(x, mask, y, w), _autograd_grad(x, mask, y, w), rtol=1e-12, atol=1e-14)
    # identical members: the s² and D terms vanish (exactly for D; the s² term up to the rounding of an unshifted mean)
    same = x[:, :1].expand(B, K, G, d).contiguous()
    for q in (1, 3):
        wq = torch.zeros_like(w)
        wq[..., q] = w[..., q]
        for g in (lp.ensemble_stats_grad(same, mask, y, wq), _autograd_grad(same, mask, y, wq)):
            assert g.abs().max().item() <= (1e-15 if q == 1 else 0.0)


def _inputs(G, d, f, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)  # noqa: E731
    return r(B, 2, G, d), r(B, T, G, f), r(B, T, G, d), r(B, T, G, d), 0.5 + torch.rand(d, generator=g, dtype=torch.float64)


@pytest.mark.parametrize("kind", ["flat", "hierarchical"])
def test_efm_loss_port_runs_and_composes(kind):
    case = (load_efm_cases() if kind == "flat" else load_efm_hi_cases())[0]
    _, ds, model = case.build()
    params, g, cfg = case.oracle_inputs(model, ds)
    params = {k: v.double() if v.is_floating_point() else v for k, v in params.items()}
    G, d, B, T, K = model.num_grid_nodes, model.num_state_vars, 2, 2, 3
    f = case.forcing.shape[-1]
    init, forc, bnd, tgt, pvs = _inputs(G, d, f, B, T, seed=1)
    gen = torch.Generator().manual_seed(2)
    lat = (model.latent_spatial_dim, model.latent_dim)
    post_eps = torch.randn(T, B, *lat, generator=gen, dtype=torch.float64)
    prior_eps = torch.randn(T, B * K, *lat, generator=gen, dtype=torch.float64)
    out = lp.efm_loss(params, g, cfg, init, forc, bnd, tgt, pvs, ds.boundary_mask, post_eps, members=K, kl_weight=0.5,
                      crps_weight=0.3, prior_eps=prior_eps, hierarchical=kind == "hierarchical")
    for k in ("recon", "kl", "crps"):
        assert out[k].shape == (T,) and torch.isfinite(out[k]).all(), k
    assert (out["kl"] > 0).all() and (out["crps"] > 0).all()
    torch.testing.assert_close(out["loss"], (out["recon"] + 0.5 * out["kl"] + 0.3 * out["crps"]).mean())
    # the first step's terms from the posterior step and the ensemble port directly
    step = lp.posterior_step(params, g, cfg, init[:, 1], init[:, 0], forc[:, 0], tgt[:, 0], post_eps[0],
                             hierarchical=kind == "hierarchical")
    interior = (1 - ds.boundary_mask.double()).reshape(-1).bool()
    new = ds.boundary_mask.double() * bnd[:, 0] + (1 - ds.boundary_mask.double()) * step["pred"]
    torch.testing.assert_close(out["recon"][0], lp.wmse(new, tgt[:, 0], pvs, mask=interior).mean())
    torch.testing.assert_close(out["kl"][0], step["kl"].mean())
    # without the ensemble term: no crps, the same recon and kl
    out0 = lp.efm_loss(params, g, cfg, init, forc, bnd, tgt, pvs, ds.boundary_mask, post_eps, members=K, kl_weight=0.5,
                       hierarchical=kind == "hierarchical")
    assert out0["crps"] is None
    torch.testing.assert_close(out0["recon"], out["recon"])
    torch.testing.assert_close(out0["kl"], out["kl"])
