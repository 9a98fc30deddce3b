"""Absolute trajectory error (flowmap/misc/ate.py:7-25) on the fm_trajectory_ate kernel.

The reference aligns the two trajectories with ``scipy.spatial.procrustes`` on the host; the kernel
follows scipy step for step in float64 (centre, scale to unit norm, R = U V^T with reflections
allowed, scale by the sum of the singular values) and sums the squared residuals on the device.
"""
from __future__ import annotations

import torch
from torch import Tensor

from ._lib import check, lib


def trajectory_ate(gt: Tensor, pred: Tensor):
    """Batched ATE without host synchronisation.  gt, pred: (T, F, 3) or (F, 3) CUDA tensors.

    Returns (ate (T,), aligned_gt, aligned_pred (T, F, 3) float32, status (T,) int32), leading dimension
    dropped for (F, 3) inputs.  status is 1 where scipy would raise "Input matrices must contain >1
    unique points" (ate is NaN there).  In rank-deficient cases (F = 2, collinear points, an exactly
    planar ground truth) the ATE and aligned_gt are unique, aligned_pred only up to a mirror along the
    null direction of aligned_gt."""
    if gt.shape != pred.shape or gt.dim() not in (2, 3) or gt.shape[-1] != 3:
        raise ValueError(f"flowmap_b200: trajectory_ate takes two (T, F, 3) or (F, 3) tensors, got "
                         f"{tuple(gt.shape)} and {tuple(pred.shape)}")
    if not gt.is_cuda or gt.device != pred.device:
        raise ValueError("flowmap_b200: trajectory_ate needs both trajectories on one CUDA device "
                         "(no CPU path exists)")
    single = gt.dim() == 2
    g = gt.detach().reshape(-1, *gt.shape[-2:]).float().contiguous()
    p = pred.detach().reshape(-1, *pred.shape[-2:]).float().contiguous()
    T, F = g.shape[:2]
    if F < 1:
        raise ValueError("flowmap_b200: trajectory_ate needs at least one point")
    ate = torch.empty(T, dtype=torch.float32, device=g.device)
    al_gt, al_pred = torch.empty_like(g), torch.empty_like(p)
    status = torch.empty(T, dtype=torch.int32, device=g.device)
    with torch.cuda.device(g.device):
        check(lib().fm_trajectory_ate(g.data_ptr(), p.data_ptr(), T, F, ate.data_ptr(), al_gt.data_ptr(),
                                      al_pred.data_ptr(), status.data_ptr(),
                                      torch.cuda.current_stream().cuda_stream), "fm_trajectory_ate")
    if single:
        return ate[0], al_gt[0], al_pred[0], status[0]
    return ate, al_gt, al_pred, status


def compute_ate(gt: Tensor, predicted: Tensor):
    """flowmap.misc.ate.compute_ate: (ate (0-d float32), aligned_gt, aligned_predicted) for two
    (point, 3) trajectories, each result on its input's device.  CPU inputs are evaluated on the
    current CUDA device.  Raises scipy.spatial.procrustes' ValueErrors; the degenerate-input check
    reads the kernel's status on the host (the reference synchronises here as well)."""
    if gt.dim() != 2 or predicted.dim() != 2:
        raise ValueError("Input matrices must be two-dimensional")
    if gt.shape != predicted.shape:
        raise ValueError("Input matrices must be of same shape")
    if gt.numel() == 0:
        raise ValueError("Input matrices must be >0 rows and >0 cols")
    if gt.shape[1] != 3:
        raise ValueError("flowmap_b200: compute_ate takes (point, 3) trajectories")
    if gt.is_cuda:
        dev = gt.device
    elif predicted.is_cuda:
        dev = predicted.device
    elif torch.cuda.is_available():
        dev = torch.device("cuda", torch.cuda.current_device())
    else:
        raise ValueError("flowmap_b200: compute_ate runs on a CUDA device (no CPU path exists)")
    ate, al_gt, al_pred, status = trajectory_ate(gt.detach().to(dev), predicted.detach().to(dev))
    if int(status) != 0:
        raise ValueError("Input matrices must contain >1 unique points")
    return ate.to(gt.device), al_gt.to(gt.device), al_pred.to(predicted.device)
