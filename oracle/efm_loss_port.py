"""fp64 restatement of Graph-EFM's training objective (``models.BaseGraphEFM.forward_posterior`` and
``models.ARForecaster.efm_loss``, DESIGN §4.6), test infrastructure only.

The reference defines no Graph-EFM loss; the definitions restated here are the library's (Oskarsson et al. 2024's
KL-weighted ELBO plus a CRPS of members sampled from the prior):

* posterior step: q = the variational encoder on the grid embedding with the target, p = the prior, z = μ_q + ε σ_q,
  decoder and (clamped) update as in the prior step; kl = Σ_latent [log(σ_p/σ_q) + (σ_q² + (μ_q - μ_p)²)/(2σ_p²) - ½],
  averaged over the latent nodes -> (B,);
* per AR step t: recon[t] = mean_b wmse(pred, target, per_var_std, interior) (or nll with the predicted std), kl[t] =
  mean_b kl, crps[t] = mean_b Σ_v crps_fair[b, v] / per_var_std[v] of the prior members (``ensemble_port``); loss = mean_t
  (recon + λ_KL kl + λ_CRPS crps).

The step modules are ``efm_port`` / ``efm_hi_port``.  ``wmse`` / ``nll`` restate the reference's ``neural_lam/metrics.py``
(:87-137, :283-329) because the GPU tests run without the reference tree; ``load_reference_metrics`` loads that file
unmodified, ``gen_golden_efm_loss.py`` stores its outputs under ``tests/golden/`` and the CPU tests pin the restatement to
them.  Any object with the reference's ``wmse`` / ``nll`` may be passed as ``metrics``.
"""
import math
import sys

import torch

from . import efm_hi_port, efm_port, ensemble_port
from .reference_port import clamped_new_state


def load_reference_metrics():
    """The reference's ``neural_lam/metrics.py``, loaded unmodified (it imports only torch)."""
    from .load_reference import _PKG, _load_file, _synthetic_package, available

    if not available():
        raise FileNotFoundError("reference source not found")
    _synthetic_package("")
    return _load_file("metrics", "neural_lam/metrics.py")


def _reduce(entry, mask):
    """metrics.py ``mask_and_reduce_metric(..., average_grid=True, sum_vars=True)``"""
    if mask is not None:
        entry = entry[..., mask, :]
    return entry.mean(dim=-2).sum(dim=-1)


def wmse(pred, target, pred_std, mask=None):
    return _reduce((pred - target) ** 2 / pred_std ** 2, mask)


def nll(pred, target, pred_std, mask=None):
    return _reduce(torch.log(pred_std) + 0.5 * math.log(2 * math.pi) + (target - pred) ** 2 / (2 * pred_std ** 2), mask)


def kl_diag(mean_q, std_q, mean_p, std_p):
    """closed-form KL(N(μ_q, σ_q) ‖ N(μ_p, σ_p)), summed over the latent dimension, averaged over the latent nodes -> (B,)"""
    kl = torch.log(std_p / std_q) + (std_q ** 2 + (mean_q - mean_p) ** 2) / (2 * std_p ** 2) - 0.5
    return kl.sum(dim=-1).mean(dim=-1)


def ensemble_stats_grad(members, interior_mask, target, grad_means):
    """Closed-form gradient of ``ensemble_port.ensemble_stats``' interior means with respect to the members, fp64 (DESIGN
    §4.5): grad_means (B, d, 4) upstream of [SE, s², A, D] -> (B, K, G, d).  One member at a time, so it needs no K² G d
    floats (autograd through ``ensemble_port`` keeps every pair difference)."""
    x, y = members.double(), target.double()
    K = x.shape[1]
    keep = interior_mask.reshape(-1).bool()
    w = grad_means.double()[:, None, None] / keep.sum()  # (B, 1, 1, d, 4), the 1/N of the interior means
    m = x.mean(dim=1, keepdim=True)
    pairs = torch.zeros_like(x)
    for l in range(K):
        pairs += torch.sign(x - x[:, l:l + 1])
    g = (w[..., 0] * 2 * (m - y.unsqueeze(1)) / K + w[..., 1] * 2 * (x - m) / (K - 1)
         + w[..., 2] * torch.sign(x - y.unsqueeze(1)) / K + w[..., 3] * 2 * pairs / (K * (K - 1)))
    return g * keep.view(1, 1, -1, 1)


def _update(g, cfg, mean_delta, prev_state):
    delta = mean_delta * g["diff_std"] + g["diff_mean"]
    clamp = cfg.get("clamp")
    if clamp:
        dt = prev_state.dtype
        return clamped_new_state(delta, prev_state, clamp["names"], clamp["lower"], clamp["upper"], clamp["state_mean"].to(dt),
                                 clamp["state_std"].to(dt))
    return prev_state + delta


def posterior_step(params, graph, cfg, prev_state, prev_prev_state, forcing, target, eps, hierarchical=False):
    """One ``forward_posterior`` -> dict(pred, pred_std, kl, post_mean, post_std, prior_mean, prior_std)."""
    dt = prev_state.dtype
    if hierarchical:
        g = efm_hi_port._cast_hi(graph, dt)
        st = efm_hi_port.hi_static_embeddings(params, g, cfg)
        post, prior_fn, dec = efm_hi_port.efm_hi_posterior, efm_hi_port.hi_prior, efm_hi_port.hi_decoder
    else:
        g = efm_port._cast(graph, dt)
        st = efm_port.static_embeddings(params, g, cfg)
        post, prior_fn, dec = efm_port.efm_posterior, efm_port.prior, efm_port.decoder
    grid_emb = efm_port.grid_embedding(params, g, cfg, prev_state, prev_prev_state, forcing)
    mq, sq = post(params, graph, cfg, prev_state, prev_prev_state, forcing, target)
    mp, sp = prior_fn(params, g, cfg, grid_emb, st)
    mean_delta, pred_std = dec(params, g, cfg, grid_emb, mq + eps.to(dt) * sq, st)
    return dict(pred=_update(g, cfg, mean_delta, prev_state), pred_std=pred_std, kl=kl_diag(mq, sq, mp, sp), post_mean=mq,
                post_std=sq, prior_mean=mp, prior_std=sp)


def efm_loss(params, graph, cfg, init_states, forcing, boundary, target, per_var_std, boundary_mask, post_eps, members=2,
             kl_weight=1.0, crps_weight=0.0, prior_eps=None, hierarchical=False, metrics=None):
    """``ARForecaster.efm_loss`` with explicit noise (post_eps (T, B, N_lat, L), prior_eps (T, B·members, N_lat, L)) ->
    dict(loss, recon (T,), kl (T,), crps (T,) or None).  ``boundary_mask`` (G, 1) as the forecaster holds it."""
    metrics = metrics or sys.modules[__name__]
    step = efm_hi_port.efm_hi_step if hierarchical else efm_port.efm_step
    B, T, G, d = target.shape
    K = members
    bm = boundary_mask.to(init_states.dtype)
    interior_mask = 1 - bm
    interior = interior_mask.reshape(-1).bool()
    ex = lambda x: x.unsqueeze(1).expand(B, K, *x.shape[1:]).reshape(B * K, *x.shape[1:])  # noqa: E731
    prev_prev, prev = init_states[:, 0], init_states[:, 1]
    ens_prev_prev, ens_prev = ex(prev_prev), ex(prev)
    recon, kl, crps = [], [], []
    for t in range(T):
        out = posterior_step(params, graph, cfg, prev, prev_prev, forcing[:, t], target[:, t], post_eps[t], hierarchical)
        new = bm * boundary[:, t] + interior_mask * out["pred"]
        if out["pred_std"] is None:
            recon.append(metrics.wmse(new, target[:, t], per_var_std, mask=interior).mean())
        else:
            recon.append(metrics.nll(new, target[:, t], out["pred_std"], mask=interior).mean())
        kl.append(out["kl"].mean())
        prev_prev, prev = prev, new
        if crps_weight > 0:
            pred = step(params, graph, cfg, ens_prev, ens_prev_prev, ex(forcing[:, t]), prior_eps[t])["pred"]
            ens = bm * ex(boundary[:, t]) + interior_mask * pred
            _, _, means = ensemble_port.ensemble_stats(ens.view(B, K, G, d), interior, target[:, t])
            fair = ensemble_port.derived(means, K)["crps_fair"]
            crps.append((fair / per_var_std).sum(dim=-1).mean())
            ens_prev_prev, ens_prev = ens_prev, ens
    recon, kl = torch.stack(recon), torch.stack(kl)
    total = recon + kl_weight * kl
    crps = torch.stack(crps) if crps else None
    if crps is not None:
        total = total + crps_weight * crps
    return dict(loss=total.mean(), recon=recon, kl=kl, crps=crps)
