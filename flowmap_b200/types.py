"""Data containers of the hot path, field-for-field with the reference's dataclasses so
that either side's objects can be passed to the other.

Batch: flowmap/dataset/types.py:12-19; Flows: flowmap/flow/flow_predictor.py:17-21;
Tracks: flowmap/tracking/track_predictor.py:14-20; BackboneOutput:
flowmap/model/backbone/backbone.py:15-17; ModelOutput/ModelExports:
flowmap/model/model.py:24-38.
"""
from __future__ import annotations

from dataclasses import dataclass, fields, replace
from typing import Optional

from torch import Tensor


class _Movable:
    def to(self, device):
        """Shallow copy with every tensor field moved (misc/manipulable.py:25-38)."""
        changes = {f.name: getattr(self, f.name).to(device) for f in fields(self)
                   if isinstance(getattr(self, f.name), Tensor)}
        return replace(self, **changes)


@dataclass
class Batch(_Movable):
    videos: Tensor  # (batch, frame, 3, height, width)
    indices: Tensor  # (batch, frame) int64
    scenes: list
    datasets: list
    extrinsics: Optional[Tensor] = None  # (batch, frame, 4, 4)
    intrinsics: Optional[Tensor] = None  # (batch, frame, 3, 3)


@dataclass
class Flows(_Movable):
    forward: Tensor  # (batch, pair, height, width, 2)
    backward: Tensor  # (batch, pair, height, width, 2)
    forward_mask: Tensor  # (batch, pair, height, width)
    backward_mask: Tensor  # (batch, pair, height, width)


@dataclass
class Tracks(_Movable):
    xy: Tensor  # (batch, frame, point, 2)
    visibility: Tensor  # (batch, frame, point) bool
    start_frame: int


@dataclass
class BackboneOutput:
    depths: Tensor  # (batch, frame, height, width)
    weights: Tensor  # (batch, frame-1, height, width)


class ModelOutput:
    """Same attributes as the reference's ModelOutput.  ``surfaces`` (b f h w 3, 415 MB at
    150x360x640) is never needed by the fused kernels, so it is materialised on first
    access only (by the unprojection kernel, differentiable)."""

    def __init__(self, depths, surfaces, intrinsics, extrinsics, backward_correspondence_weights, *,
                 relative=None, k4=None, k_mode="full"):
        # positional order = the reference's dataclass (model.py:24-30); `surfaces` may be None
        # (materialised on first access); the extra fields are keyword-only
        self.depths = depths
        self.intrinsics = intrinsics
        self.extrinsics = extrinsics
        self.backward_correspondence_weights = backward_correspondence_weights
        self._surfaces = surfaces
        self.relative = relative  # (b, f-1, 3, 4) Procrustes [R|t], frame i+1 -> frame i
        self.k4 = k4  # (b, f, 4) = (fx, fy, cx, cy)
        self.k_mode = k_mode  # how the intrinsics were produced (see ops.flow_loss)

    @property
    def surfaces(self) -> Tensor:
        if "_fused" in self.__dict__:  # the output of a fused step (flowmap_b200.fused): the step's own surfaces
            from .fused import materialize
            return materialize(self).surfaces
        if self._surfaces is None:
            from . import ops
            k4 = self.k4 if self.k4 is not None else ops.intrinsics_to_k4(self.intrinsics)
            self._surfaces = ops.unproject_depth(self.depths, k4)
        return self._surfaces

    def __getattr__(self, name):
        # only reached for attributes that are not set: those a fused step (flowmap_b200.fused) computes when they
        # are read
        if "_fused" not in self.__dict__ or name.startswith("__"):
            raise AttributeError(name)
        from .fused import materialize
        return getattr(materialize(self), name)


@dataclass
class ModelExports:
    extrinsics: Tensor
    intrinsics: Tensor
    colors: Tensor
    depths: Tensor
