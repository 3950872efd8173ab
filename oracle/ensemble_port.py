"""fp64 restatement of the ensemble statistics of ``neural_lam_b200.ensemble`` (DESIGN §4.5), test infrastructure only.

Per initial condition b, grid node g and variable v, with x_1 .. x_K the members and y the target:
  m = (1/K) Σ_k x_k,  s² = (1/(K-1)) Σ_k (x_k - m)²,  SE = (m - y)²,  A = (1/K) Σ_k |x_k - y|,
  D = (1/(K(K-1))) Σ_{k≠l} |x_k - x_l|   (summed over the pairs, as written)
SE, s², A and D are averaged over the interior grid nodes (the reference's ``interior_mask_bool`` with
``mask_and_reduce_metric(..., average_grid=True, sum_vars=False)``, metrics.py:37-84).  The reference itself has no
ensemble scores (its metrics.py has the closed-form ``crps_gauss`` only).
"""
import torch


def point_stats(members, target=None):
    """members (B, K, G, d), target (B, G, d) or None -> dict of fp64 (B, G, d) tensors: mean, var, and with a target
    se, abs_err, pair_diff."""
    x = members.double()
    K = x.shape[1]
    m = x.mean(dim=1)
    out = {"mean": m, "var": ((x - m.unsqueeze(1)) ** 2).sum(dim=1) / (K - 1)}
    if target is not None:
        y = target.double()
        out["se"] = (m - y) ** 2
        out["abs_err"] = (x - y.unsqueeze(1)).abs().mean(dim=1)
        pairs = torch.zeros_like(m)
        for k in range(K):  # Σ_{k≠l}, one member at a time: K² G d floats never exist at once
            pairs += (x[:, k:k + 1] - x).abs().sum(dim=1)
        out["pair_diff"] = pairs / (K * (K - 1))
    return out


def pair_diff_sorted(members):
    """D by the sorted form Σ_{k≠l} |x_k - x_l| = 2 Σ_i (2i - K - 1) x_(i) (i = 1..K), over dim 1."""
    x = members.double().sort(dim=1).values
    K = x.shape[1]
    w = (2 * torch.arange(1, K + 1, dtype=torch.float64) - K - 1).view(1, K, *([1] * (x.dim() - 2)))
    return 2 * (w * x).sum(dim=1) / (K * (K - 1))


def ensemble_stats(members, interior_mask, target=None):
    """-> (mean (B, G, d), std (B, G, d), means (B, d, 4) of [SE, s², A, D] over the interior nodes, or None), fp64"""
    s = point_stats(members, target)
    std = s["var"].sqrt()
    if target is None:
        return s["mean"], std, None
    keep = interior_mask.reshape(-1).bool()
    means = torch.stack([s[q][:, keep].mean(dim=1) for q in ("se", "var", "abs_err", "pair_diff")], dim=-1)
    return s["mean"], std, means


def derived(means, K):
    """means (..., 4) of [SE, s², A, D] -> dict of rmse, spread, ssr, crps_fair, crps_ecdf"""
    se, var, a, d = means.unbind(-1)
    rmse, spread = se.sqrt(), var.sqrt()
    return {"rmse": rmse, "spread": spread, "ssr": ((K + 1) / K) ** 0.5 * spread / rmse, "crps_fair": a - d / 2,
            "crps_ecdf": a - (K - 1) / (2 * K) * d}
