"""Model side of the hot path: backbone -> intrinsics -> Procrustes poses.

Mirrors flowmap/model/model.py:41-110 and the registries of flowmap/model/{backbone,
intrinsics,extrinsics}/__init__.py with the same class names, cfg dataclasses and
forward signatures; the bodies call the sm_90a kernels through flowmap_b200.ops.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Literal, Optional

import torch
from torch import Tensor, nn

from . import ops
from .types import BackboneOutput, Batch, Flows, ModelExports, ModelOutput


# --------------------------------------------------------------------------- backbones
@dataclass
class BackboneExplicitDepthCfg:
    """config/model/backbone/explicit_depth.yaml"""
    name: Literal["explicit_depth"]
    initial_depth: float
    weight_sensitivity: float


class BackboneExplicitDepth(nn.Module):
    """flowmap/model/backbone/backbone_explicit_depth.py:19-41: free depth and
    correspondence-weight tensors; parameter names kept (`depth`, `weights`) so reference
    checkpoints load."""

    def __init__(self, cfg, num_frames, image_shape):
        super().__init__()
        self.cfg, self.num_frames, self.image_shape = cfg, num_frames, image_shape
        self.depth = nn.Parameter(torch.full((num_frames, *image_shape), cfg.initial_depth,
                                             dtype=torch.float32))
        self.weights = nn.Parameter(torch.zeros((num_frames - 1, *image_shape),
                                                dtype=torch.float32))

    def forward(self, batch: Batch, flows: Flows) -> BackboneOutput:
        assert batch.videos.shape[0] == 1  # backbone_explicit_depth.py:35-36
        return BackboneOutput(self.depth[None],
                              (self.cfg.weight_sensitivity * self.weights).sigmoid()[None])


BACKBONES = {"explicit_depth": BackboneExplicitDepth}


def get_backbone(cfg, num_frames, image_shape):
    if cfg.name not in BACKBONES:
        raise NotImplementedError(
            f"backbone '{cfg.name}' is outside the hot path (SURVEY 2, row 6): construct the "
            "reference's backbone and pass its BackboneOutput to the kernels instead")
    return BACKBONES[cfg.name](cfg, num_frames, image_shape)


# --------------------------------------------------------------------------- intrinsics
def focal_lengths_to_intrinsics(focal_lengths: Tensor, image_shape) -> Tensor:
    """flowmap/model/intrinsics/common.py:6-20."""
    h, w = image_shape
    scaled = focal_lengths * (h * w) ** 0.5
    k = torch.zeros((*focal_lengths.shape, 3, 3), dtype=torch.float32, device=focal_lengths.device)
    k[..., 0, 2] = 0.5
    k[..., 1, 2] = 0.5
    k[..., 2, 2] = 1.0
    sel = torch.zeros((2, 3, 3), dtype=torch.float32, device=focal_lengths.device)
    sel[0, 0, 0] = 1.0
    sel[1, 1, 1] = 1.0
    return k + (scaled / w)[..., None, None] * sel[0] + (scaled / h)[..., None, None] * sel[1]


@dataclass
class IntrinsicsRegressedCfg:
    name: Literal["regressed"]
    initial_focal_length: float


class IntrinsicsRegressed(nn.Module):
    """flowmap/model/intrinsics/intrinsics_regressed.py:22-41."""

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        self.focal_length = nn.Parameter(torch.tensor(cfg.initial_focal_length,
                                                      dtype=torch.float32))

    def forward(self, batch, flows, backbone_output, global_step) -> Tensor:
        b, f, _, h, w = batch.videos.shape
        return focal_lengths_to_intrinsics(self.focal_length, (h, w)).expand(b, f, 3, 3)


@dataclass
class IntrinsicsGroundTruthCfg:
    name: Literal["ground_truth"]


class IntrinsicsGroundTruth(nn.Module):
    """flowmap/model/intrinsics/intrinsics_ground_truth.py:18-27."""

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg

    def forward(self, batch, flows, backbone_output, global_step) -> Tensor:
        return batch.intrinsics


@dataclass
class RegressionCfg:
    after_step: int
    window: int


@dataclass
class IntrinsicsSoftminCfg:
    name: Literal["softmin"]
    num_procrustes_points: int
    min_focal_length: float
    max_focal_length: float
    num_candidates: int
    regression: Optional[RegressionCfg]


class IntrinsicsSoftmin(nn.Module):
    """flowmap/model/intrinsics/intrinsics_softmin.py:40-141.  First stage: candidate sweep on
    the first frame pair -> softmin-weighted focal length (the weighted sum of candidate
    matrices equals K(sum softmin_n f_n), SURVEY A.10); after `regression.after_step` steps a
    regressed focal length seeded with the mean of the last `window` estimates."""

    def __init__(self, cfg: IntrinsicsSoftminCfg):
        super().__init__()
        self.cfg = cfg
        self.register_buffer("focal_length_candidates",
                             torch.linspace(cfg.min_focal_length, cfg.max_focal_length,
                                            cfg.num_candidates), persistent=False)
        if cfg.regression is not None:
            self.intrinsics_regressed = IntrinsicsRegressed(IntrinsicsRegressedCfg("regressed", 0.0))
            self.window = []
        self.injected_indices = None  # tests: same point set as the oracle (SURVEY A.8 item 1)

    def forward(self, batch, flows, backbone_output, global_step) -> Tensor:
        b, f, _, h, w = batch.videos.shape
        c = self.cfg
        if c.regression is not None and global_step >= c.regression.after_step:
            if global_step == c.regression.after_step:
                self.intrinsics_regressed.focal_length.data = torch.stack(self.window).mean()
            return self.intrinsics_regressed(batch, flows, backbone_output, global_step)
        device = backbone_output.depths.device
        indices = self.injected_indices
        if indices is None:
            indices = ops.random_subset(h * w, min(c.num_procrustes_points, h * w), device)
        err = ops.softmin_errors(backbone_output.depths, backbone_output.weights, flows.backward,
                                 indices, self.focal_length_candidates)
        weights = torch.softmax(-(err - err.min(dim=1, keepdim=True).values) * 10, dim=1)
        focal = (weights * self.focal_length_candidates).sum(dim=1)  # (b,)
        if c.regression is not None:
            start = c.regression.after_step - c.regression.window
            if global_step >= start and self.training:
                self.window.append(focal.sum().detach())
        return focal_lengths_to_intrinsics(focal, (h, w))[:, None].expand(b, f, 3, 3)


INTRINSICS = {"ground_truth": IntrinsicsGroundTruth, "regressed": IntrinsicsRegressed,
              "softmin": IntrinsicsSoftmin}


def get_intrinsics(cfg):
    return INTRINSICS[cfg.name](cfg)


# --------------------------------------------------------------------------- extrinsics
@dataclass
class ExtrinsicsProcrustesCfg:
    name: Literal["procrustes"]
    num_points: Optional[int]
    randomize_points: bool


class ExtrinsicsProcrustes(nn.Module):
    """flowmap/model/extrinsics/extrinsics_procrustes.py:23-59.  The reference receives
    the materialised surfaces; here the point cloud is formed inside the moment kernel, so
    ``forward`` takes depths + k4 and returns (extrinsics, relative poses)."""

    def __init__(self, cfg, num_frames):
        super().__init__()
        self.cfg, self.num_frames = cfg, num_frames

    def select_indices(self, h: int, w: int, device) -> Optional[Tensor]:
        c = self.cfg
        if c.num_points is None:
            return None  # all pixels; the kernel's dense path
        if c.randomize_points:
            return torch.randint(0, h * w, (c.num_points,), dtype=torch.int64, device=device)
        return torch.linspace(0, h * w - 1, c.num_points, dtype=torch.int64, device=device)

    def forward(self, batch, flows, backbone_output, k4, indices=None):
        _, _, h, w = backbone_output.depths.shape
        if indices is None:
            indices = self.select_indices(h, w, backbone_output.depths.device)
        rt = ops.procrustes_poses(backbone_output.depths, backbone_output.weights, k4,
                                  flows.backward, indices)
        return ops.pose_chain(rt), rt


@dataclass
class ExtrinsicsRegressedCfg:
    name: Literal["regressed"]


class ExtrinsicsRegressed(nn.Module):
    """flowmap/model/extrinsics/extrinsics_regressed.py:47-83, the free-pose ablation (no Procrustes:
    nothing for the moment kernels to do).  Per-pair translations and quaternions (parameter names
    and the scipy (i, j, k, r) order kept so that reference checkpoints load); plain ATen arithmetic
    for the 3 x 3 matrices, the chain on the scan kernel.  The flow / tracking kernels take its
    relative poses like the Procrustes ones."""

    def __init__(self, cfg, num_frames):
        super().__init__()
        assert num_frames >= 2
        self.cfg, self.num_frames = cfg, num_frames
        self.translations = nn.Parameter(torch.zeros((num_frames - 1, 3), dtype=torch.float32))
        rotations = torch.zeros((num_frames - 1, 4), dtype=torch.float32)
        rotations[:, -1] = 1
        self.rotations = nn.Parameter(rotations)

    @staticmethod
    def quaternion_to_matrix(q: Tensor, eps: float = 1e-8) -> Tensor:
        i, j, k, r = q.unbind(-1)
        s = 2 / ((q * q).sum(-1) + eps)
        rows = (1 - s * (j * j + k * k), s * (i * j - k * r), s * (i * k + j * r),
                s * (i * j + k * r), 1 - s * (i * i + k * k), s * (j * k - i * r),
                s * (i * k - j * r), s * (j * k + i * r), 1 - s * (i * i + j * j))
        return torch.stack(rows, -1).reshape(*q.shape[:-1], 3, 3)

    def forward(self, batch, flows, backbone_output, k4=None, indices=None):
        assert backbone_output.depths.shape[0] == 1  # extrinsics_regressed.py:75-76
        rt = torch.cat((self.quaternion_to_matrix(self.rotations), self.translations[..., None]), dim=-1)[None]
        return ops.pose_chain(rt.contiguous()), rt


EXTRINSICS = {"procrustes": ExtrinsicsProcrustes, "regressed": ExtrinsicsRegressed}


def get_extrinsics(cfg, num_frames):
    return EXTRINSICS[cfg.name](cfg, num_frames)


# --------------------------------------------------------------------------- model
@dataclass
class ModelCfg:
    backbone: object
    intrinsics: object
    extrinsics: object
    use_correspondence_weights: bool


class Model(nn.Module):
    """flowmap/model/model.py:41-110."""

    def __init__(self, cfg: ModelCfg, num_frames=None, image_shape=None):
        super().__init__()
        self.cfg = cfg
        self.backbone = get_backbone(cfg.backbone, num_frames, image_shape)
        self.intrinsics = get_intrinsics(cfg.intrinsics)
        self.extrinsics = get_extrinsics(cfg.extrinsics, num_frames)

    # ---- fused evaluation (flowmap_b200.fused): Model.forward launches nothing but a network backbone,
    # the losses run the two halves of the fused step
    fused_enabled = True  # class-wide switch (tests compare the two evaluation orders)

    def _fusable(self, batch: Batch, flows: Flows, backbone_out: Optional[BackboneOutput] = None) -> bool:
        """Whether the losses of this step can run on the fused halves.  A network backbone (any backbone
        but BackboneExplicitDepth, e.g. the reference's BackboneMidas) is judged on the BackboneOutput of
        the step: CUDA depths (B, F, H, W) and weights (B, F-1, H, W).  B > 1 (pretraining) takes one focal
        length per video: softmin intrinsics without a regression stage (the regressed focal length, and the
        window of a regression stage, are one value for the whole batch in the reference), or ground-truth K.
        Ground-truth K must come as a floating (B, F, 3, 3) `batch.intrinsics` on the flows' device."""
        b, f, _, h, w = batch.videos.shape
        gt = isinstance(self.intrinsics, IntrinsicsGroundTruth)
        if not (self.fused_enabled and torch.is_grad_enabled() and self.training and
                isinstance(self.extrinsics, ExtrinsicsProcrustes) and
                isinstance(self.intrinsics, (IntrinsicsRegressed, IntrinsicsSoftmin, IntrinsicsGroundTruth)) and
                flows.forward.is_cuda):
            return False
        if gt:
            k = batch.intrinsics
            if not (isinstance(k, Tensor) and k.is_floating_point() and k.device == flows.forward.device and
                    tuple(k.shape) == (b, f, 3, 3)):
                return False
        if isinstance(self.backbone, BackboneExplicitDepth):
            return b == 1 and self.backbone.depth.is_cuda
        if backbone_out is None:
            return False
        if b > 1 and not (gt or isinstance(self.intrinsics, IntrinsicsSoftmin) and self.intrinsics.cfg.regression is None):
            return False
        d, wt = backbone_out.depths, backbone_out.weights
        return (isinstance(d, Tensor) and isinstance(wt, Tensor) and d.is_floating_point() and
                wt.is_floating_point() and d.device == wt.device == flows.forward.device and
                tuple(d.shape) == (b, f, h, w) and tuple(wt.shape) == (b, f - 1, h, w))

    def _fused_params(self, global_step: int, inputs=None):
        """Tensors that receive a gradient from the fused step, in the order of FusedStep's buffers:
        the explicit-depth parameters, or a network backbone's float32 `inputs` (depths [, weights]) of
        this step, then the focal length that is being learned (none for ground-truth K)."""
        if inputs is not None:
            params = list(inputs)
        else:
            params = [self.backbone.depth]
            if self.cfg.use_correspondence_weights:
                params.append(self.backbone.weights)
        intr = self.intrinsics
        if isinstance(intr, IntrinsicsRegressed):
            params.append(intr.focal_length)
        elif (isinstance(intr, IntrinsicsSoftmin) and intr.cfg.regression is not None and
              global_step >= intr.cfg.regression.after_step):
            params.append(intr.intrinsics_regressed.focal_length)
        return params

    def _overfit_fields(self) -> dict:
        """The fields of an OverfitCfg that this model's configuration sets (a network backbone's BackboneOutput
        holds the weights themselves: sensitivity 0 to the kernels)."""
        mc, bc, ic, ec = self.cfg, self.cfg.backbone, self.cfg.intrinsics, self.cfg.extrinsics
        explicit = isinstance(self.backbone, BackboneExplicitDepth)
        soft = isinstance(self.intrinsics, IntrinsicsSoftmin)
        reg = ic.regression if soft else None
        intrinsics = ("ground_truth" if isinstance(self.intrinsics, IntrinsicsGroundTruth) else
                      "softmin" if soft else "regressed")
        return dict(
            initial_depth=bc.initial_depth if explicit else 0.0,
            weight_sensitivity=bc.weight_sensitivity if explicit else 0.0,
            use_correspondence_weights=mc.use_correspondence_weights, procrustes_points=ec.num_points,
            procrustes_randomize=ec.randomize_points, intrinsics=intrinsics,
            softmin_points=ic.num_procrustes_points if soft else 8192,
            softmin_min=ic.min_focal_length if soft else 0.5, softmin_max=ic.max_focal_length if soft else 2.0,
            softmin_candidates=ic.num_candidates if soft else 60,
            regression_after=reg.after_step if reg is not None else None,
            regression_window=reg.window if reg is not None else 100)

    def _fused_engine(self, batch: Batch, flows: Flows, tracks, flow_loss):
        """The FusedOverfitter bound to this model's parameters for (flows, tracks); built on first
        use, re-pointed when the Flows tensors change, None if the configuration is not covered.  A batch of
        several videos with tracks is not (loss_tracking.py serves one video): the whole step then runs per-op,
        as the flow loss must not run fused while the tracking loss reads a detached snapshot."""
        if batch.videos.shape[0] > 1 and tracks is not None:
            return None
        from .overfit import FusedOverfitter, OverfitCfg
        lm = flow_loss.cfg.mapping
        key = (tuple(batch.videos.shape), None if tracks is None else tuple(id(t) for t in tracks),
               lm.name, getattr(lm, "delta", 0.01))
        eng = getattr(self, "_engine", None)
        if eng is None or self._engine_key != key:
            explicit = isinstance(self.backbone, BackboneExplicitDepth)
            cfg = OverfitCfg(
                **self._overfit_fields(),
                flow_weight=flow_loss.cfg.weight, flow_enable_after=flow_loss.cfg.enable_after,
                use_tracking=tracks is not None, tracking_enable_after=0, mapping=lm.name,
                delta=getattr(lm, "delta", 0.01))
            dev = self.backbone.depth.device if explicit else flows.forward.device
            eng = FusedOverfitter(cfg, batch, flows, tracks, device=dev, model=self)
            object.__setattr__(self, "_engine", eng)
            object.__setattr__(self, "_engine_key", key)
            object.__setattr__(self, "_engine_flows", None)
        cur = (flows.forward, flows.backward, flows.forward_mask, flows.backward_mask)
        # the step reads contiguous Flows tensors themselves, and contiguous copies of the others: a copy is
        # taken again every step, as a loader may have rewritten the tensor behind the same view
        if (self._engine_flows is None or any(a is not b for a, b in zip(cur, self._engine_flows)) or
                not all(t.is_contiguous() for t in cur)):
            eng.set_flows(flows, mask_sum=flow_loss._mask_total(flows))
            object.__setattr__(self, "_engine_flows", cur)
        return eng

    def forward(self, batch: Batch, flows: Flows, global_step: int) -> ModelOutput:
        from .fused import fused_output
        if isinstance(self.backbone, BackboneExplicitDepth):
            if self._fusable(batch, flows):
                return fused_output(self, batch, flows, global_step)
            return self._forward_materialized(batch, flows, global_step)
        # a network backbone runs once per step, under autograd as usual; the fused halves take its output
        backbone_out = self.backbone.forward(batch, flows)
        if self._fusable(batch, flows, backbone_out):
            return fused_output(self, batch, flows, global_step, backbone_out)
        return self._forward_materialized(batch, flows, global_step, backbone_out)

    def _forward_materialized(self, batch: Batch, flows: Flows, global_step: int,
                              backbone_out: Optional[BackboneOutput] = None) -> ModelOutput:
        """The per-op evaluation; `backbone_out` is this step's output of the backbone when it already ran."""
        if backbone_out is None:
            backbone_out = self.backbone.forward(batch, flows)
        if not self.cfg.use_correspondence_weights:  # model.py:67-68
            backbone_out = BackboneOutput(backbone_out.depths, torch.ones_like(backbone_out.weights))
        intrinsics = self.intrinsics.forward(batch, flows, backbone_out, global_step)
        k4 = ops.intrinsics_to_k4(intrinsics)
        extrinsics, rt = self.extrinsics.forward(batch, flows, backbone_out, k4)
        k_mode = {IntrinsicsRegressed: "shared_focal", IntrinsicsSoftmin: "shared_focal",
                  IntrinsicsGroundTruth: "const"}.get(type(self.intrinsics), "full")
        return ModelOutput(backbone_out.depths, None, intrinsics, extrinsics, backbone_out.weights,
                           relative=rt, k4=k4, k_mode=k_mode)

    @torch.no_grad()
    def export(self, batch: Batch, flows: Flows, global_step: int) -> ModelExports:
        assert batch.videos.shape[0] == 1  # model.py:100-101
        out = self._forward_materialized(batch, flows, global_step)
        return ModelExports(out.extrinsics, out.intrinsics, batch.videos, out.depths)
