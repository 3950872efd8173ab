"""Ensemble statistics and scores of K forecast members on the device (``nlam_ensemble_stats``, DESIGN §4.5).

Per initial condition b, grid node g and variable v, with x_1 .. x_K the members and y the target:

=============================  ==============================================
ensemble mean                  m = (1/K) Σ_k x_k
ensemble variance              s² = (1/(K-1)) Σ_k (x_k - m)²   (torch.var)
squared error of the mean      SE = (m - y)²
mean absolute error term       A = (1/K) Σ_k |x_k - y|
mean pair difference           D = (1/(K(K-1))) Σ_{k≠l} |x_k - x_l|
=============================  ==============================================

SE, s², A and D are averaged over the interior grid nodes (the reference's ``interior_mask_bool`` and
``mask_and_reduce_metric(..., average_grid=True, sum_vars=False)``, metrics.py:37-84).  The scores derived from those
means are ``EnsembleScores``' properties: rmse = sqrt(mean SE), spread = sqrt(mean s²), the spread-skill ratio
ssr = sqrt((K+1)/K) · spread / rmse, the fair CRPS A - D/2 and the CRPS of the members' empirical distribution
A - (K-1)/(2K) · D (both linear in A and D, so they can be formed after the grid average).

There is no CPU or eager fallback: CPU tensors, tensors that are not float32 and K outside 2 .. 64 raise.
"""
from dataclasses import dataclass

import torch

from . import _lib
from .ops import _require_cuda, _stream_ptr

MAX_MEMBERS = 64


@dataclass(frozen=True)
class EnsembleScores:
    """Interior-grid means of one ensemble's per-point scores, one value per (..., variable): ``se`` = mean SE,
    ``var`` = mean s², ``abs_err`` = mean A, ``pair_diff`` = mean D, for ``members`` = K members."""
    se: torch.Tensor
    var: torch.Tensor
    abs_err: torch.Tensor
    pair_diff: torch.Tensor
    members: int

    @classmethod
    def from_means(cls, means, members):
        """``means`` (..., d, 4): [SE, s², A, D] in the last dimension (the layout of ``nlam_ensemble_stats``)."""
        return cls(means[..., 0], means[..., 1], means[..., 2], means[..., 3], members)

    @property
    def rmse(self):
        return self.se.sqrt()

    @property
    def spread(self):
        return self.var.sqrt()

    @property
    def ssr(self):
        K = self.members
        return ((K + 1) / K) ** 0.5 * self.spread / self.rmse

    @property
    def crps_fair(self):
        return self.abs_err - 0.5 * self.pair_diff

    @property
    def crps_ecdf(self):
        K = self.members
        return self.abs_err - (K - 1) / (2 * K) * self.pair_diff


def _member_blocks(members):
    """(B, K, G, d) with dense (G, d) blocks (any strides over B and K), else a contiguous copy"""
    if members.dim() != 4:
        raise ValueError(f"members: expected (B, K, G, d), got shape {tuple(members.shape)}")
    _, _, G, d = members.shape
    if (d > 1 and members.stride(3) != 1) or (G > 1 and members.stride(2) != d):
        members = members.contiguous()
    return members


def _check_members(K):
    if not 2 <= K <= MAX_MEMBERS:
        raise ValueError(f"ensemble statistics need 2 <= K <= {MAX_MEMBERS} members, got K = {K}")


def workspace_bytes(B, G, d):
    """Device workspace ``launch`` needs for the scores of B ensembles of (G, d) states."""
    return int(_lib.lib().nlam_ensemble_stats_workspace_bytes(B, G, d))


def launch(members, interior, mean, std, target=None, scores=None, workspace=None):
    """Low-level call into preallocated tensors (no allocation: legal inside a CUDA-graph capture).  ``members``
    (B, K, G, d) with dense (G, d) blocks, ``interior`` (G) float32 (nonzero = interior node), ``mean`` / ``std``
    (B, G, d) contiguous; with ``scores`` (B, d, 4) contiguous also ``target`` (B, G, d) with dense (G, d) blocks and a
    uint8 ``workspace`` of ``workspace_bytes(B, G, d)`` bytes."""
    B, K, G, d = members.shape
    _check_members(K)
    _require_cuda(members, interior, mean, std, target, scores)
    for t, shape in ((mean, (B, G, d)), (std, (B, G, d))):
        if tuple(t.shape) != shape or not t.is_contiguous():
            raise ValueError(f"ensemble statistics: expected a contiguous output of shape {shape}, got {tuple(t.shape)}")
    tp = ip = sp = wp = None
    tbs, ws_bytes = 0, 0
    if scores is not None:
        if target is None or workspace is None:
            raise ValueError("ensemble statistics: scores need a target and a workspace")
        if tuple(target.shape) != (B, G, d) or (d > 1 and target.stride(2) != 1) or (G > 1 and target.stride(1) != d):
            raise ValueError(f"target: expected (B, G, d) = {(B, G, d)} with dense rows, got {tuple(target.shape)}")
        if tuple(scores.shape) != (B, d, 4) or not scores.is_contiguous():
            raise ValueError(f"scores: expected a contiguous ({B}, {d}, 4) tensor, got {tuple(scores.shape)}")
        if interior.numel() != G or not interior.is_contiguous():
            raise ValueError(f"interior mask: expected {G} contiguous values, got {interior.numel()}")
        tp, tbs, ip, sp = target.data_ptr(), target.stride(0), interior.data_ptr(), scores.data_ptr()
        wp, ws_bytes = workspace.data_ptr(), workspace.numel() * workspace.element_size()
    with torch.cuda.device(members.device):
        _lib.check(_lib.lib().nlam_ensemble_stats(
            members.data_ptr(), members.stride(0), members.stride(1), B, K, G, d, tp, tbs, ip, mean.data_ptr(),
            std.data_ptr(), sp, wp, ws_bytes, _stream_ptr(members.device)))


def ensemble_stats(members, interior_mask, target=None):
    """Ensemble mean, spread and (with ``target``) scores of stored members.

    ``members`` (B, K, G, d) float32 on the device; any strides over B and K (rows b·K + k of a forecast batch viewed as
    (B, K, G, d), or a time slice ``x[:, :, t]`` of a (B, K, T, G, d) ensemble, are read without a copy).
    ``interior_mask`` (G) or (G, 1): nonzero / True on the interior grid nodes the scores average over (the forecaster's
    ``interior_mask``).  ``target`` (B, G, d).  Returns ``(mean, std, scores)``: mean m and std s = sqrt(s²) as (B, G, d)
    and an ``EnsembleScores`` of (B, d) tensors, or None without a target."""
    members = _member_blocks(members)
    B, K, G, d = members.shape
    _check_members(K)
    interior = interior_mask.reshape(-1)
    if interior.dtype == torch.bool:
        interior = interior.float()
    _require_cuda(members, interior, target)
    interior = interior.contiguous()
    mean = torch.empty(B, G, d, device=members.device)
    std = torch.empty_like(mean)
    scores = ws = None
    if target is not None:
        if target.dim() != 3:
            raise ValueError(f"target: expected (B, G, d), got shape {tuple(target.shape)}")
        if (d > 1 and target.stride(2) != 1) or (G > 1 and target.stride(1) != d):
            target = target.contiguous()
        scores = torch.empty(B, d, 4, device=members.device)
        ws = torch.empty(workspace_bytes(B, G, d), dtype=torch.uint8, device=members.device)
    launch(members, interior, mean, std, target=target, scores=scores, workspace=ws)
    return mean, std, (EnsembleScores.from_means(scores, K) if scores is not None else None)
