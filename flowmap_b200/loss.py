"""Loss side of the hot path.  Mirrors flowmap/loss/loss.py:24-58, loss_flow.py:26-70 and
the mapping registry of flowmap/loss/mapping/__init__.py (same names / cfg fields)."""
from __future__ import annotations

import weakref
from dataclasses import dataclass
from typing import Literal

import torch
from torch import Tensor, nn

from . import ops
from .types import Flows


@dataclass
class MappingHuberCfg:
    name: Literal["huber"]
    delta: float


@dataclass
class MappingL1Cfg:
    name: Literal["l1"]


@dataclass
class MappingL2Cfg:
    name: Literal["l2"]


@dataclass
class LossCfgCommon:
    enable_after: int
    weight: float


@dataclass
class LossFlowCfg(LossCfgCommon):
    name: Literal["flow"]
    mapping: object


@dataclass
class LossTrackingCfg(LossCfgCommon):
    name: Literal["tracking"]
    mapping: object


class Loss(nn.Module):
    """loss.py:24-58: gate on enable_after, scale by weight."""

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg

    def forward(self, batch, flows, tracks, model_output, global_step) -> Tensor:
        if global_step < self.cfg.enable_after:  # loss.py:40-41
            return torch.tensor(0, dtype=torch.float32, device=batch.videos.device)
        return self.compute_weighted_loss(batch, flows, tracks, model_output, global_step)


def _relative_from_extrinsics(extrinsics: Tensor) -> Tensor:
    """inv(P_i) P_{i+1} for callers that hand in extrinsics without the Procrustes output
    (projection.py:176); rigid inverse [R^T | -R^T t]."""
    r, t = extrinsics[:, :-1, :3, :3], extrinsics[:, :-1, :3, 3:]
    rn, tn = extrinsics[:, 1:, :3, :3], extrinsics[:, 1:, :3, 3:]
    rt_ = r.transpose(-1, -2)
    return torch.cat((rt_ @ rn, rt_ @ (tn - t)), dim=-1)


class LossFlow(Loss):
    """loss_flow.py:26-70.  The weight (loss.py:46) and the 1/mask-sum normalisation are
    folded into the kernel so that it emits final gradients in the same pass."""

    def __init__(self, cfg: LossFlowCfg):
        super().__init__(cfg)
        self._mask_key = None
        self._mask_sum = None

    def _mask_total(self, flows: Flows) -> Tensor:
        # The denominator depends on the (constant) masks only: recompute when the mask
        # tensors change identity or are written to.
        fm, bm = flows.forward_mask, flows.backward_mask
        key = self._mask_key
        hit = (key is not None and key[0]() is fm and key[1]() is bm and
               key[2] == (fm._version, bm._version))
        if not hit:
            self._mask_sum = ops.mask_sum(fm, bm)
            self._mask_key = (weakref.ref(fm), weakref.ref(bm), (fm._version, bm._version))
        return self._mask_sum

    def compute_weighted_loss(self, batch, flows, tracks, model_output, global_step):
        out = model_output
        fused = out.__dict__.get("_fused")  # the output of a fused step (flowmap_b200.fused)
        if fused is not None:
            value = fused.flow_loss(self, tracks)
            if value is not None:
                return value
        k4 = getattr(out, "k4", None)
        if k4 is None:
            k4 = ops.intrinsics_to_k4(out.intrinsics)
        rt = getattr(out, "relative", None)
        if rt is None:
            rt = _relative_from_extrinsics(out.extrinsics)
        m = self.cfg.mapping
        return ops.flow_loss(out.depths, rt, k4, flows.forward, flows.backward,
                             flows.forward_mask, flows.backward_mask, self._mask_total(flows),
                             m.name, getattr(m, "delta", 0.0), self.cfg.weight,
                             getattr(out, "k_mode", "full"))


class LossTracking(Loss):
    """loss_tracking.py:23-61: all-pairs track reprojection loss over every segment."""

    def __init__(self, cfg: LossTrackingCfg):
        super().__init__(cfg)
        self._packed = None
        self._packed_key = None

    def _pack(self, tracks, device):
        key = tuple(id(t) for t in tracks)
        if key != self._packed_key or self._packed is None:
            self._packed = ops.PackedTracks(tracks, device)  # tracks are constant across steps
            self._packed_key = key
            self._keepalive = list(tracks)
        return self._packed

    def compute_weighted_loss(self, batch, flows, tracks, model_output, global_step):
        assert tracks is not None  # loss_tracking.py:37
        out = model_output
        fused = out.__dict__.get("_fused")
        if fused is not None:
            value = fused.track_loss(self, tracks)
            if value is not None:
                return value
        k4 = getattr(out, "k4", None)
        if k4 is None:
            k4 = ops.intrinsics_to_k4(out.intrinsics)
        m = self.cfg.mapping
        # one focal length behind all frames (or constant K): autograd sums d/dk4 over the frames
        # anyway, so the kernel may book the intrinsics terms on any frame
        shared_k = getattr(out, "k_mode", "full") in ("shared_focal", "const")
        return ops.track_loss(out.depths, out.extrinsics, k4, self._pack(tracks, out.depths.device),
                              m.name, getattr(m, "delta", 0.0), self.cfg.weight, shared_k)


LOSSES = {"flow": LossFlow, "tracking": LossTracking}


def get_losses(cfgs):
    return [LOSSES[c.name](c) for c in cfgs]
