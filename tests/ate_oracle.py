"""Float64 oracle of the trajectory metric: misc/ate.py:7-25 compute_ate, i.e. scipy.spatial.procrustes
followed by the reference's ATE, restated in torch (dtype-generic, batched over leading dimensions).
TEST INFRASTRUCTURE ONLY: flowmap_b200 never imports it."""
from __future__ import annotations

import torch
from torch import Tensor


def trajectory_ate(gt: Tensor, pred: Tensor):
    """scipy.spatial.procrustes + the reference's ATE on (..., F, 3) trajectories, in their dtype.

    Centre both sets, scale each to unit Frobenius norm, R = U V^T from the SVD of gt^T pred (no
    determinant fix: reflections are allowed), s = sum of the singular values, aligned_pred =
    s * pred R^T, ate = sqrt(mean((aligned_gt - aligned_pred)^2)) summed term by term.  Returns
    (ate, aligned_gt, aligned_pred, degenerate) where `degenerate` marks scipy's ValueError (a set
    is one point after centring: norm exactly 0); ate is NaN there."""
    a = gt - gt.mean(dim=-2, keepdim=True)
    b = pred - pred.mean(dim=-2, keepdim=True)
    na = a.square().sum(dim=(-2, -1)).sqrt()
    nb = b.square().sum(dim=(-2, -1)).sqrt()
    degenerate = (na == 0) | (nb == 0)
    a = a / torch.where(degenerate, torch.ones_like(na), na)[..., None, None]
    b = b / torch.where(degenerate, torch.ones_like(nb), nb)[..., None, None]
    u, sig, vt = torch.linalg.svd(a.transpose(-1, -2) @ b)
    r = u @ vt
    aligned = sig.sum(-1)[..., None, None] * (b @ r.transpose(-1, -2))
    ate = (a - aligned).square().mean(dim=(-2, -1)).sqrt()
    ate = torch.where(degenerate, torch.full_like(ate, float("nan")), ate)
    return ate, a, aligned, degenerate
