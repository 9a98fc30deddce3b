"""The optimisation loop around the hot path: what flowmap/overfit.py:76-112 builds and
flowmap/model/model_wrapper_overfit.py:51-73,104-105 runs every step (Model.forward ->
sum of losses -> backward -> Adam), without the Lightning/Hydra shell.
"""
from __future__ import annotations

from dataclasses import dataclass, fields, replace
from typing import Optional

import torch
from torch import Tensor

from . import checkpoint, ops
from .loss import (LossFlowCfg, LossTrackingCfg, MappingHuberCfg, MappingL1Cfg, MappingL2Cfg,
                   get_losses)
from .model import (BackboneExplicitDepth, BackboneExplicitDepthCfg, ExtrinsicsProcrustesCfg, IntrinsicsGroundTruth,
                    IntrinsicsGroundTruthCfg, IntrinsicsRegressedCfg, IntrinsicsSoftminCfg, Model, ModelCfg,
                    RegressionCfg)
from .ops import _ptr
from .types import Batch, Flows


@dataclass
class OverfitCfg:
    """The values of config/overfit.yaml + config/{model,loss}/** that the step reads."""
    initial_depth: float = 0.1
    weight_sensitivity: float = 100.0
    use_correspondence_weights: bool = True
    procrustes_points: Optional[int] = None  # experiment/ablation_explicit_depth.yaml:11-12
    procrustes_randomize: bool = False
    intrinsics: str = "regressed"
    initial_focal: float = 0.85
    softmin_points: int = 8192
    softmin_min: float = 0.5
    softmin_max: float = 2.0
    softmin_candidates: int = 60
    regression_after: Optional[int] = 1000
    regression_window: int = 100
    flow_weight: float = 1000.0
    flow_enable_after: int = 0
    tracking_weight: float = 100.0
    tracking_enable_after: int = 50
    use_tracking: bool = False
    mapping: str = "huber"
    delta: float = 0.01
    lr: float = 3e-5


def _mapping_cfg(name: str, delta: float):
    return {"huber": MappingHuberCfg("huber", delta), "l1": MappingL1Cfg("l1"),
            "l2": MappingL2Cfg("l2")}[name]


def build_model_and_losses(cfg: OverfitCfg, num_frames: int, image_shape):
    if cfg.intrinsics == "regressed":
        icfg = IntrinsicsRegressedCfg("regressed", cfg.initial_focal)
    elif cfg.intrinsics == "ground_truth":  # intrinsics_ground_truth.py: K comes with the batch
        icfg = IntrinsicsGroundTruthCfg("ground_truth")
    else:
        reg = None if cfg.regression_after is None else RegressionCfg(cfg.regression_after,
                                                                      cfg.regression_window)
        icfg = IntrinsicsSoftminCfg("softmin", cfg.softmin_points, cfg.softmin_min,
                                    cfg.softmin_max, cfg.softmin_candidates, reg)
    mcfg = ModelCfg(BackboneExplicitDepthCfg("explicit_depth", cfg.initial_depth,
                                             cfg.weight_sensitivity), icfg,
                    ExtrinsicsProcrustesCfg("procrustes", cfg.procrustes_points,
                                            cfg.procrustes_randomize),
                    cfg.use_correspondence_weights)
    model = Model(mcfg, num_frames, image_shape)
    lcfgs = [LossFlowCfg(cfg.flow_enable_after, cfg.flow_weight, "flow",
                         _mapping_cfg(cfg.mapping, cfg.delta))]
    if cfg.use_tracking:
        lcfgs.append(LossTrackingCfg(cfg.tracking_enable_after, cfg.tracking_weight, "tracking",
                                     _mapping_cfg(cfg.mapping, cfg.delta)))
    return model, get_losses(lcfgs)


class FusedAdam:
    """torch.optim.Adam(params, lr) semantics (model_wrapper_overfit.py:104-105) on the
    fm_adam_step kernel: one launch per parameter tensor, no foreach temporaries."""

    def __init__(self, params, lr: float, betas=(0.9, 0.999), eps: float = 1e-8):
        self.params = [p for p in params]
        self.lr, self.betas, self.eps = lr, betas, eps
        self.steps = [0 for _ in self.params]  # torch keeps one step counter per parameter
        self.state = [(torch.zeros_like(p), torch.zeros_like(p)) for p in self.params]

    def zero_grad(self):
        for p in self.params:
            p.grad = None

    @torch.no_grad()
    def step(self):
        for i, (p, (m, v)) in enumerate(zip(self.params, self.state)):
            if p.grad is None:  # torch.optim skips parameters that did not receive a gradient
                continue
            self.steps[i] += 1
            ops.adam_step(p.data, p.grad.contiguous(), m, v, self.steps[i], self.lr, self.betas,
                          self.eps)


class Overfitter:
    """Holds the constant batch/flows/tracks and runs optimisation steps
    (model_wrapper_overfit.py:24-73)."""

    def __init__(self, cfg: OverfitCfg, batch: Batch, flows: Flows, tracks=None,
                 device="cuda", model=None):
        self.cfg = cfg
        self.batch, self.flows = batch.to(device), flows.to(device)
        self.tracks = None if tracks is None else [t.to(device) for t in tracks]
        _, f, _, h, w = batch.videos.shape
        if model is None:
            self.model, self.losses = build_model_and_losses(cfg, f, (h, w))
            self.model.to(device)
            self.optimizer = FusedAdam(self.model.parameters(), cfg.lr)
        else:  # bound to a caller's Model (the autograd drop-in surface, flowmap_b200.fused)
            self.model, self.losses, self.optimizer = model, None, None
        self.global_step = 0
        # torch.optim.Adam counts the updates each parameter has received, not the trainer's
        # global_step (they differ when a run starts at global_step > 0 with a fresh optimiser, and
        # for the focal length, which sees its first gradient at the softmin -> regressed hand-over)
        self.optimizer_steps = 0
        self.focal_steps = 0

    def training_step(self):
        """Returns (total loss tensor (device), ModelOutput); no host sync."""
        self.optimizer.zero_grad()
        out = self.model(self.batch, self.flows, self.global_step)
        total = 0
        for loss_fn in self.losses:
            total = total + loss_fn.forward(self.batch, self.flows, self.tracks, out,
                                            self.global_step)
        total.backward()
        self.optimizer.step()
        self.global_step += 1
        return total.detach(), out


_FLOW_NAMES = ("forward", "backward", "forward_mask", "backward_mask")


def video_tables(frames, device):
    """The device tables of an fm_video_layout for videos of `frames` frames packed along the frame axis:
    the frame offsets (B + 1,), the video of every frame (T,) and of every pair (T - B,), int32."""
    B, fr = len(frames), torch.tensor(frames)
    fo = torch.tensor([sum(frames[:i]) for i in range(B + 1)], dtype=torch.int32)
    return (fo.to(device), torch.repeat_interleave(torch.arange(B, dtype=torch.int32), fr).to(device),
            torch.repeat_interleave(torch.arange(B, dtype=torch.int32), fr - 1).to(device))


def _video(x, i: int):
    """Video i of a Batch or Flows of several videos, as a one-video instance of the same type (views)."""
    return replace(x, **{f.name: getattr(x, f.name)[i:i + 1] for f in fields(x) if getattr(x, f.name) is not None})


class FusedOverfitter:
    """Same optimisation as :class:`Overfitter` (explicit-depth backbone, Procrustes poses,
    regressed focal length, flow [+ tracking] loss, Adam) but each step is ONE C-ABI call,
    fm_overfit_step: no autograd graph, no intermediate tensors, the sigmoid of the weight
    logits and its chain rule evaluated inside the kernels, gradients accumulated into a
    single buffer per parameter.

    The constructor reads its inputs as B videos, each with its Batch, Flows, track segments and frame count
    F_b, all of one H x W.  They come in one of three forms:

    - one video: `batch.videos` (1, F, 3, H, W), Flows (1, F-1, ...), `tracks` a list of segments.  The
      step is fm_overfit_step, whose buffers are the Model's own parameters, and which also serves the
      split-step surface and pair sharding.
    - a tensor batch: `batch.videos` (B, F, 3, H, W) with B > 1, Flows (B, F-1, ...): videos of one length.
    - a list of B one-video Batches with a list of their Flows (1, F_b - 1, ...): videos of different lengths.

    Several videos run B INDEPENDENT overfits in one step (fm_overfit_step_videos).  Video b gets what a
    one-video FusedOverfitter on video b with the same cfg and step clock seed gets: its flow loss is
    normalised by its own mask sum, its tracking loss by its own valid count, and its gradients, Adam
    moments, focal length, softmin window and poses are its own.  This differs on purpose from the
    reference's LossFlow at b > 1 (pretraining), which normalises a batch by ONE pooled mask sum.  Shared by
    the batch: the Procrustes point subset and the softmin point sample of each step.  The parameters live
    in buffers packed along the frame axis, video b owning frames [fo_b, fo_b + F_b) and pairs
    [fo_b - b, fo_b - b + F_b - 1); `models[b]` is video b's Model, whose parameters are views into them.
    `tracks` is a list of B segment lists.  Several videos do not serve pair sharding or the split-step
    surface (but for a network Model's batch, below).

    Whatever takes or hands out one value per video follows the form: the buffer of one video, a
    (B, F [- 1], ...) tensor for a tensor batch, a list for a list of Batches.  That holds for the totals
    and poses of training_step(), extrinsics(), intrinsics_k4(), gradients(), set_flows, set_intrinsics
    and the metrics log, whose rows are (steps,) for one video and (steps, B) for several.  `batches` holds
    the videos' Batches in every form.

    Bound to a Model whose backbone is a network (any backbone but BackboneExplicitDepth, the drop-in
    surface of flowmap_b200.fused), the optimiser owns no depth or weight buffers and no Adam state for
    them: every step's depths and weights come from the network, through forward_phase, and only the
    split phases run (cfg.weight_sensitivity 0: the weights themselves, their gradient d loss / d weight).
    Such a Model also takes a tensor batch (the reference's pretraining step: softmin intrinsics without a
    regression stage, or ground-truth K, no tracks), whose rows are the network's depths and weights and
    the caller's Flows, which set_flows re-points to rather than copies.  Its mask_sum holds the pooled
    normaliser of LossFlow at b > 1 in every video's slot, so that the (B,) losses sum to the batch's loss,
    and backward_phase takes one flow_scale for the whole batch.

    cfg.intrinsics "ground_truth" (intrinsics_ground_truth.py, calibrated data) takes K as given: from
    each video's `batch.intrinsics`, normalised as in the reference and possibly different for every frame.
    There is no focal parameter and the step computes no intrinsics gradient (fm_overfit_step with focal =
    g_k4 = track_g_k4 = NULL, and the split forward's tracking sweep fm_track_loss_fwd_const_k);
    set_intrinsics swaps K in place.  Pair sharding does not serve it."""

    def __init__(self, cfg: OverfitCfg, batch: Batch, flows: Flows, tracks=None, device="cuda", model=None):
        from ._lib import VideoLayout, lib
        import ctypes
        listed = isinstance(batch, (list, tuple))
        B = len(batch) if listed else batch.videos.shape[0]
        # a list of B network Models: B overfits in one packed split step (flowmap_b200.fused.network_videos_step)
        self._net_videos = isinstance(model, (list, tuple))
        one = not listed and B == 1 and not self._net_videos
        tensor_batch = not listed and not one
        self.cfg, self._gt, self._tensor_batch = cfg, cfg.intrinsics == "ground_truth", tensor_batch
        # bound to a caller's Model (the autograd drop-in surface, flowmap_b200.fused)
        self._bound = model is not None
        if self._net_videos:
            self._check_network_models(cfg, list(model), B)
            self._network = True
        else:
            self._network = isinstance(model, Model) and not isinstance(model.backbone, BackboneExplicitDepth)
        # a network Model's tensor batch: the pretraining step, one pooled flow-loss normaliser
        self._pooled = self._network and not self._net_videos and tensor_batch

        # ---- the videos: one (Batch, Flows) each, validated before anything reaches the device
        if self._net_videos:
            pass
        elif model is not None and (listed or tensor_batch and not self._network):
            raise ValueError("flowmap_b200: a bound Model holds one video (batch size 1)")
        if self._pooled:
            if tracks is not None or cfg.use_tracking:
                raise ValueError("flowmap_b200: a network backbone's batch of several videos takes no tracks")
            if (self._gt != isinstance(model.intrinsics, IntrinsicsGroundTruth) or
                    not self._gt and (cfg.intrinsics != "softmin" or cfg.regression_after is not None)):
                raise ValueError("flowmap_b200: a network backbone's batch of several videos needs softmin intrinsics "
                                 "without a regression stage (one focal length per video), or ground-truth intrinsics, "
                                 f"in both cfg.intrinsics ({cfg.intrinsics!r}) and the bound model "
                                 f"({type(model.intrinsics).__name__})")
        elif model is not None and not self._net_videos and isinstance(model.intrinsics, IntrinsicsGroundTruth) != self._gt:
            raise ValueError(f"flowmap_b200: the bound model's intrinsics ({type(model.intrinsics).__name__}) do not "
                             f"match cfg.intrinsics = {cfg.intrinsics!r}")
        if listed and (not batch or not isinstance(flows, (list, tuple)) or len(flows) != B):
            raise ValueError("flowmap_b200: videos of different lengths need one Flows per Batch")
        if not one and (cfg.use_tracking or tracks is not None) and (tracks is None or len(tracks) != B):
            raise ValueError(f"flowmap_b200: tracks must hold one segment list per video ({B})")
        if tensor_batch:
            for name in _FLOW_NAMES:
                if tuple(getattr(flows, name).shape[:2]) != (B, batch.videos.shape[1] - 1):
                    raise ValueError(f"flowmap_b200: flows.{name} must hold (B, F-1) = ({B}, "
                                     f"{batch.videos.shape[1] - 1}) pairs")
        videos = list(zip(batch, flows)) if listed else \
            [(_video(batch, i), _video(flows, i)) for i in range(B)] if tensor_batch else [(batch, flows)]
        h, w = videos[0][0].videos.shape[-2:]
        for i, (bt, fl) in enumerate(videos):
            nb, f = bt.videos.shape[:2]
            if nb != 1:
                raise ValueError(f"flowmap_b200: video {i} must be a one-video Batch")
            if tuple(bt.videos.shape[-2:]) != (h, w):
                raise ValueError("flowmap_b200: the videos of one step need the same H x W")
            if f < 2:
                raise ValueError(f"flowmap_b200: video {i} has {f} frame(s), a pair needs 2")
            for name in _FLOW_NAMES:
                if tuple(getattr(fl, name).shape[:4]) != (1, f - 1, h, w):
                    raise ValueError(f"flowmap_b200: flows[{i}].{name} must hold (1, F_b-1, H, W) = "
                                     f"(1, {f - 1}, {h}, {w})")

        # ---- one body for every form
        if listed:
            self.batches = [bt.to(device) for bt in batch]
            self.batch = self.batches[0]
        else:
            self.batch = batch.to(device)
            self.batches = [_video(self.batch, i) for i in range(B)] if tensor_batch else [self.batch]
        frames = [bt.videos.shape[1] for bt in self.batches]
        self.B, self.frames, self.T, self._hw = B, frames, sum(frames), (h, w)
        self._first = [sum(frames[:i]) for i in range(B)]
        T = self.T
        # the kernels read raw pointers: canonical (contiguous float32) tensors, kept alive here
        # (FlowPredictor.rescale_flow returns a permuted view, flow_predictor.py:40-49)
        if one or self._pooled:  # the tensors given, or copies of those that are not contiguous
            self.flows = self._canonical_flows(flows.to(device))
        else:  # copies packed along the pair axis: the pairs of video b follow those of video b - 1
            self.flows = Flows(*(torch.cat([ops._canon(getattr(fl, n).to(device), n)[0] for _, fl in videos])
                                 .contiguous() for n in _FLOW_NAMES))
        dev = self.flows.forward.device
        if one:  # the Uniform entry points, on the Model's own parameters
            self._layout, self._track_frames = None, None
            self._lead = ((1, T), (1, T - 1), ())  # leading dims of the per-frame, per-pair and per-video buffers
            self.tracks = None if tracks is None else [t.to(device) for t in tracks]
            self._ws = ops.workspace(1, T, h, w, dev)
        else:  # the _videos entry points, on buffers packed along the frame axis
            self._tables = video_tables(frames, dev)
            self._layout = VideoLayout(B, T, *(t.data_ptr() for t in self._tables))
            self._layout_ref = ctypes.byref(self._layout)
            self._lead, self._track_frames = ((T,), (T - B,), (B,)), frames
            self.tracks = None if tracks is None else [[t.to(device) for t in v] for v in tracks]
            self._ws = torch.empty(lib().fm_workspace_bytes_videos(B, T), dtype=torch.uint8, device=dev)

        if model is None:
            built = [build_model_and_losses(cfg, f, (h, w)) for f in frames]
            self.models, self.losses = [m.to(device) for m, _ in built], built[0][1]
        elif self._net_videos:
            self.models, self.losses = list(model), None
        else:
            self.models, self.losses = [model], None
        self.model = self.models[0]

        def gather(params, stack: bool):
            """One buffer for the videos' `params`: the Model's own tensor for one video, else the videos' tensors
            stacked or concatenated, which the parameters become views of."""
            if one:
                return params[0].data
            buf = (torch.stack if stack else torch.cat)([p.data for p in params]).contiguous()
            for p, part in zip(params, buf.unbind() if stack else buf.split([p.shape[0] for p in params])):
                p.data = part
            return buf
        if self._network:  # the step's depths / weights arrive with forward_phase
            self._depth = self._wlog = None
        else:  # a tensor batch's are (B, F [- 1], H, W)
            self._depth = gather([m.backbone.depth for m in self.models], tensor_batch)
            self._wlog = gather([m.backbone.weights for m in self.models], tensor_batch)
        if self._gt:
            self._focal = None
        elif cfg.intrinsics != "softmin":
            self._focal = gather([m.intrinsics.focal_length for m in self.models], True)
        elif cfg.regression_after is not None:
            self._focal = gather([m.intrinsics.intrinsics_regressed.focal_length for m in self.models], True)
        else:
            self._focal = torch.zeros(self._lead[2], device=dev)
        if self._pooled:  # LossFlow's pooled normaliser at b > 1, in every video's slot
            pooled = ops.mask_sum(self.flows.forward_mask, self.flows.backward_mask)
            self._msum = pooled.expand(self._lead[2]).contiguous()
        else:
            self._msum = self._video_mask_sums(self.flows)
        self.global_step = 0
        # torch.optim.Adam counts the updates each parameter has received, not the trainer's
        # global_step (they differ when a run starts at global_step > 0 with a fresh optimiser, and
        # for the focal length, which sees its first gradient at the softmin -> regressed hand-over)
        self.optimizer_steps = self.focal_steps = 0
        self._init_step(cfg)
        if self._gt:
            k = [bt.intrinsics for bt in self.batches] if listed else self.batch.intrinsics
            # a Model-bound optimiser serves the autograd surface, which rewrites K before every step and, like
            # the reference, does not check its values
            if self._bound:
                self._write_k4(k)
            else:
                self.set_intrinsics(k)

    @staticmethod
    def _check_network_models(cfg: "OverfitCfg", models, B: int):
        """The Models of B networks' overfits: one per video, each with a network backbone, all of one
        configuration that `cfg` describes (the step runs one OverfitCfg and one step clock for all of them)."""
        if len(models) != B:
            raise ValueError(f"flowmap_b200: {len(models)} Models for {B} videos: one network Model per video")
        for i, m in enumerate(models):
            if not isinstance(m, Model) or isinstance(m.backbone, BackboneExplicitDepth):
                raise ValueError(f"flowmap_b200: model {i} is not a Model with a network backbone (an explicit-depth "
                                 "Model optimises its own depth: several of them go to a FusedOverfitter of their own)")
            if m.cfg != models[0].cfg:
                raise ValueError(f"flowmap_b200: model {i}'s cfg differs from model 0's: the videos of one step share "
                                 "one configuration")
        want = models[0]._overfit_fields()
        diff = {k: (getattr(cfg, k), v) for k, v in want.items() if getattr(cfg, k) != v}
        if diff:
            raise ValueError(f"flowmap_b200: cfg does not describe the Models (cfg value, model value): {diff}")

    def _canonical_flows(self, flows: Flows, device=None) -> Flows:
        """Flows of this optimiser's (B, F-1, H, W, ...) shape on `device` (default: that of flows.forward), as
        the contiguous float32 tensors the step reads: the tensors themselves, or copies of those that are not
        contiguous."""
        want = (self.B, self.frames[0] - 1, *self._hw)
        canon = []
        for name in _FLOW_NAMES:
            t = ops._canon(getattr(flows, name), name)
            device = device or t.device
            shape = want + (2,) if name in ("forward", "backward") else want
            if tuple(t.shape) != shape or t.device != device:
                raise ValueError(f"flowmap_b200: flows.{name} must be a {shape} tensor on {device}")
            canon.append(t)
        return Flows(*canon)

    def _init_step(self, cfg):
        """What one video and packed videos wire alike: the softmin buffers, the Adam state, the gradient
        and output buffers, the args struct, the step clock and the tracking buffers."""
        from ._lib import OverfitStepArgs, PackedTracksC, lib
        import ctypes
        (h, w), B, T = self._hw, self.B, self.T
        frame_dims, pair_dims, video_dims = self._lead
        dev = self.flows.forward.device
        self._softmin = cfg.intrinsics == "softmin"
        if self._softmin:
            n = cfg.softmin_candidates
            self._cand_f = self.model.intrinsics.focal_length_candidates.float().contiguous()
            self._cand_k4 = ops.candidate_k4(self._cand_f, h, w, B)
            self._sw_err, self._sw_sm, self._sw_gerr = (torch.empty(B, n, device=dev) for _ in range(3))
            self._sw_rt = torch.empty(B * n, 3, 4, device=dev)
            self._sw_focal = torch.zeros(B, device=dev)
            self._sw_ws = torch.empty(lib().fm_softmin_workspace_bytes(B, n), dtype=torch.uint8, device=dev)
            # candidate 0's intrinsics for every frame: what the early moment pass of a sweep step uses
            self._k4_base = self._cand_k4.reshape(-1, 4)[0].expand(T, 4).contiguous()
            self.window = []
            self.injected_indices = None
        z = lambda t: None if t is None else torch.zeros_like(t)  # noqa: E731
        # the moments of the (T, H, W) depth and (T - B, H, W) logit rows: none for a network's depths and weights
        rows = lambda n: None if self._network else torch.zeros(n, h, w, device=dev)  # noqa: E731
        self._state = [rows(T), rows(T), rows(T - B), rows(T - B), z(self._focal), z(self._focal)]
        self._g_depth, self._g_w = torch.empty(T, h, w, device=dev), torch.empty(T - B, h, w, device=dev)
        # ground-truth K: no focal parameter, and no intrinsics gradient buffers (the constant-intrinsics step)
        self._g_focal = z(self._focal)
        self._k4, self._g_k4 = torch.empty(T, 4, device=dev), None if self._gt else torch.empty(T, 4, device=dev)
        self.rt = torch.empty(*pair_dims, 3, 4, device=dev)
        self._loss = torch.zeros(video_dims, device=dev)
        self._track_loss = torch.zeros_like(self._loss)
        self._indices = self.model.extrinsics.select_indices(h, w, dev) if not cfg.procrustes_randomize else None
        a = OverfitStepArgs()
        a.F, a.H, a.W = T if self._layout is None else 0, h, w  # F: ignored by fm_overfit_step_videos
        a.depth = _ptr(self._depth)
        a.weight_logits = _ptr(self._wlog) if cfg.use_correspondence_weights else None
        a.weight_sensitivity = cfg.weight_sensitivity
        a.focal, a.k4 = _ptr(self._focal), _ptr(self._k4)  # a sweep step's calls pass the sweep's estimate
        a.fflow, a.bflow = _ptr(self.flows.forward), _ptr(self.flows.backward)
        a.fmask, a.bmask = _ptr(self.flows.forward_mask), _ptr(self.flows.backward_mask)
        a.mask_sum = _ptr(self._msum)
        a.mapping, a.delta, a.flow_weight = ops.MAPPINGS[cfg.mapping], cfg.delta, cfg.flow_weight
        (a.m_depth, a.v_depth, a.m_weights, a.v_weights, a.m_focal, a.v_focal) = [_ptr(t) for t in self._state]
        a.beta1, a.beta2, a.eps = 0.9, 0.999, 1e-8
        a.g_depth, a.g_weights = _ptr(self._g_depth), _ptr(self._g_w)
        a.g_focal, a.g_k4 = _ptr(self._g_focal), _ptr(self._g_k4)
        a.rt, a.loss, a.ws = _ptr(self.rt), _ptr(self._loss), _ptr(self._ws)
        # step-dependent scalars live in device memory: every step is the same launch sequence
        self._clock = ops.StepClock(dev, cfg.lr)
        self._side_stream = torch.cuda.Stream(device=dev)  # parallel branch of the step (see _step_softmin)
        a.clock = self._clock.ptr
        a.video_grad_scales = int(self._net_videos)  # backward_phase's scales: one per video
        self._total = torch.zeros_like(self._loss)
        self._idx_buf = torch.empty(min(cfg.softmin_points, h * w), dtype=torch.int64, device=dev) \
            if self._softmin else None
        self.use_cuda_graph = False  # opt-in: replay the update step as ONE CUDA graph launch
        self._graphs, self._eager_runs = {}, {}
        self._packed = None
        if cfg.use_tracking:
            assert self.tracks is not None
            pk = ops.PackedTracks(self.tracks, dev, self._track_frames)
            self._packed = pk
            self._pk_c = PackedTracksC(_ptr(pk.seg), _ptr(pk.xy), _ptr(pk.vis), pk.num_segments, pk.max_rows,
                                       pk.max_points, pk.total)
            self._ext = torch.empty(*frame_dims, 4, 4, device=dev)
            self._g_ext = torch.empty(*frame_dims, 4, 4, device=dev)
            self._g_rt = torch.empty(*pair_dims, 3, 4, device=dev)
            self._tg_k4 = None if self._gt else torch.empty(T, 4, device=dev)
            self._tws = torch.empty(lib().fm_track_workspace_bytes(T, pk.total), dtype=torch.uint8, device=dev)
            a.track_weight = cfg.tracking_weight
            a.extrinsics, a.g_extrinsics, a.g_rt = _ptr(self._ext), _ptr(self._g_ext), _ptr(self._g_rt)
            a.track_g_k4, a.track_loss, a.track_ws = _ptr(self._tg_k4), _ptr(self._track_loss), _ptr(self._tws)
        self._args, self._ctypes = a, ctypes
        self._lib = lib()
        self._mlog = None  # per-step metrics ring (enable_metrics_log)

    def _per_video(self, t: Tensor, pairs: bool = False):
        """Each video's rows of a (T, ...) frame buffer, or with `pairs` a (T - B, ...) pair buffer: the buffer
        itself for one video, a (B, F [- 1], ...) view for a tensor batch, a list of views for a list of Batches."""
        if self._layout is None:
            return t
        if self._tensor_batch:
            return t.view(self.B, -1, *t.shape[1:])
        return [t[f0 - pairs * i:f0 - pairs * i + f - pairs] for i, (f0, f) in enumerate(zip(self._first, self.frames))]

    def _call_step(self, what: str = "fm_overfit_step", **fields):
        """Run the step on a copy of _args with this call's `fields` (phase, tracks, step, defer_adam, focal, ...)
        set: _args holds what every call shares, and no call leaves a field behind for the next one."""
        from ._lib import OverfitStepArgs, check
        args = OverfitStepArgs.from_buffer_copy(self._args)
        for name, value in fields.items():
            setattr(args, name, value)
        st = torch.cuda.current_stream().cuda_stream
        a = self._ctypes.byref(args)
        if self._layout is not None:
            check(self._lib.fm_overfit_step_videos(a, self._layout_ref, st), what)
        else:
            check(self._lib.fm_overfit_step(a, st), what)

    def set_flows(self, flows: Flows, mask_sum: Optional[Tensor] = None):
        """Point the step at another device-resident Flows of the same shape (the next batch of a
        prefetching loader) without rebuilding parameters or optimiser state.  `mask_sum` is the
        flow-loss normaliser (loss_flow.py:70) if the caller already has it.  Several videos: the new
        flows are copied into the packed buffers, from one (B, F-1, ...) Flows for a tensor batch, else
        from a list of one Flows per video.  One video, or a network backbone's batch of several: the step
        reads the new Flows themselves, and `mask_sum` (default: the pooled sum of all their masks) goes to
        every video."""
        if self._layout is not None and not self._pooled:
            if self._tensor_batch and isinstance(flows, Flows):
                flows = [_video(flows, i) for i in range(flows.forward.shape[0])]
            if not isinstance(flows, (list, tuple)) or len(flows) != self.B:
                raise ValueError(f"flowmap_b200: set_flows needs one Flows per video ({self.B})")
            for name in _FLOW_NAMES:
                dst = self._per_video(getattr(self.flows, name), pairs=True)
                for i, fl in enumerate(flows):
                    t = ops._canon(getattr(fl, name), name)
                    if t.shape != (1, *dst[i].shape) or t.device != dst[i].device:
                        raise ValueError(f"flowmap_b200: flows[{i}].{name} does not match the optimiser's shapes / device")
                    dst[i].copy_(t[0])
            self._msum.copy_(self._video_mask_sums(self.flows) if mask_sum is None else mask_sum)
            return
        flows = self._canonical_flows(flows, self.flows.forward.device)
        self.flows = flows  # the canonical tensors stay referenced while the kernels hold their pointers
        a = self._args
        a.fflow, a.bflow = flows.forward.data_ptr(), flows.backward.data_ptr()
        a.fmask, a.bmask = flows.forward_mask.data_ptr(), flows.backward_mask.data_ptr()
        self._msum.copy_(self._mask_sum(flows) if mask_sum is None else mask_sum)
        self._graphs.clear()  # captured launches hold the old pointers
        self._eager_runs.clear()

    def _mask_sum(self, flows: Flows) -> Tensor:
        return ops.mask_sum(flows.forward_mask, flows.backward_mask)

    def _video_mask_sums(self, flows: Flows) -> Tensor:
        """Each video's own flow-loss normaliser, float64: a scalar for one video, else (B,)."""
        fm, bm = self._per_video(flows.forward_mask, pairs=True), self._per_video(flows.backward_mask, pairs=True)
        return torch.stack([ops.mask_sum(fm[i], bm[i]) for i in range(self.B)]).reshape(self._lead[2])

    def _adam_frames(self, i: int, lo: int, hi: int):
        """Adam (step clock) on frames lo <= f < hi of parameter i (0 depth, 1 weight logits); several videos:
        on the frames (pairs) lo <= r < min(hi, F_b (- 1)) of every video."""
        p, g = ((self._depth, self._g_depth), (self._wlog, self._g_w))[i]
        m, v = self._state[2 * i], self._state[2 * i + 1]
        if self._layout is None:
            ops.adam_step_clock(p[lo:hi], g[lo:hi], m[lo:hi], v[lo:hi], self._clock)
            return
        from ._lib import check
        with torch.cuda.device(p.device):
            check(self._lib.fm_adam_step_clock_frames_videos(
                p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), g[0].numel(), self._layout_ref, i, lo, hi,
                self._clock.ptr, 0, self._clock.betas[0], self._clock.betas[1], 1e-8,
                torch.cuda.current_stream().cuda_stream), "fm_adam_step_clock_frames_videos")

    def _softmin_stage(self) -> bool:
        c = self.cfg
        return self._softmin and not (c.regression_after is not None and
                                      self.global_step >= c.regression_after)

    def _begin_step(self):
        """The step's Procrustes point subset, redrawn every step under procrustes_randomize, and its flow
        weight, 0 before flow_enable_after (loss.py:40-41)."""
        c, a = self.cfg, self._args
        if c.procrustes_randomize:
            self._indices = self.model.extrinsics.select_indices(*self._hw, self.rt.device)
        a.indices = _ptr(self._indices)
        a.num_indices = 0 if self._indices is None else self._indices.numel()
        a.flow_weight = c.flow_weight if self.global_step >= c.flow_enable_after else 0.0

    def _sweep_indices(self, clocked: bool = False, split: bool = False) -> Tensor:
        """The sweep's point sample (intrinsics_softmin.py:90): injected_indices when set -- on the split
        step also the model's own -- else a random subset, seeded by the step clock when `clocked` (the
        update steps of training_step, which a CUDA graph may replay)."""
        idx = self.injected_indices
        if idx is None and split:
            idx = getattr(self.model.intrinsics, "injected_indices", None)
        if idx is None:
            hw = self._hw[0] * self._hw[1]
            if clocked:
                idx = ops.random_subset_clock(self._clock, hw, self._idx_buf)
            else:
                idx = ops.random_subset(hw, min(self.cfg.softmin_points, hw), self.rt.device)
        return idx.contiguous()

    def _weight_args(self):
        """(pointer, sensitivity) of the correspondence weights that the sweep and the moment pass read."""
        if not self.cfg.use_correspondence_weights:
            return None, 0.0
        return _ptr(self._wlog), self.cfg.weight_sensitivity

    def _sweep_forward(self, idx: Tensor, stream):
        """Candidate sweep on the first pair of every video at the points `idx`, and its softmin focal
        estimate into _sw_focal (intrinsics_softmin.py:84-131), on the CUDA stream handle `stream`."""
        from ._lib import check
        L, n, (h, w) = self._lib, self.cfg.softmin_candidates, self._hw
        wl, sens = self._weight_args()
        head = (_ptr(self._depth), wl, sens, _ptr(self.flows.backward), _ptr(idx), idx.numel(), _ptr(self._cand_k4),
                n, _ptr(self._sw_err), _ptr(self._sw_rt), _ptr(self._sw_ws))
        if self._layout is not None:
            check(L.fm_softmin_sweep_fwd_videos(*head, self._layout_ref, h, w, stream), "fm_softmin_sweep_fwd_videos")
        else:
            check(L.fm_softmin_sweep_fwd(*head, 1, self.T, h, w, stream), "fm_softmin_sweep_fwd")
        check(L.fm_softmin_focal(_ptr(self._sw_err), _ptr(self._cand_f), n, self.B, _ptr(self._sw_sm),
                                 _ptr(self._sw_focal), stream), "fm_softmin_focal")

    def _sweep_backward(self, idx: Tensor, stream):
        """The sweep's backward from d loss / d focal in _g_focal: adds to the gradients of frames 0 / 1 and
        pair 0 of every video."""
        from ._lib import check
        L, n, (h, w) = self._lib, self.cfg.softmin_candidates, self._hw
        wl, sens = self._weight_args()
        check(L.fm_softmin_focal_bwd(_ptr(self._sw_sm), _ptr(self._cand_f), _ptr(self._sw_focal),
                                     _ptr(self._g_focal), n, self.B, _ptr(self._sw_gerr), stream),
              "fm_softmin_focal_bwd")
        head = (_ptr(self._depth), wl, sens, _ptr(self.flows.backward), _ptr(idx), idx.numel(), _ptr(self._cand_k4),
                n, _ptr(self._sw_rt), _ptr(self._sw_gerr), _ptr(self._g_depth), _ptr(self._g_w) if wl else None,
                _ptr(self._sw_ws))
        if self._layout is not None:
            check(L.fm_softmin_sweep_bwd_videos(*head, self._layout_ref, h, w, stream), "fm_softmin_sweep_bwd_videos")
        else:
            check(L.fm_softmin_sweep_bwd(*head, 1, self.T, h, w, stream), "fm_softmin_sweep_bwd")

    def _early_moments(self, stream):
        """The step's Procrustes moment pass on the candidate-0 intrinsics (see _step_softmin), on the CUDA
        stream handle `stream`."""
        from ._lib import check
        L, (h, w) = self._lib, self._hw
        wl, sens = self._weight_args()
        head = (_ptr(self._depth), _ptr(self._k4_base), _ptr(self.flows.backward), wl, sens, _ptr(self._ws))
        if self._layout is not None:
            check(L.fm_procrustes_moments_videos(*head, self._layout_ref, h, w, stream), "fm_procrustes_moments_videos")
        else:
            check(L.fm_procrustes_moments(*head, self.T, h, w, stream), "fm_procrustes_moments")

    def _window(self, split: bool = False):
        """The hand-over window of the softmin stage (intrinsics_softmin.py:133-139): on the split step
        of a bound model that has one, the model's own list (drop-in surface), else this optimiser's."""
        intr = self.model.intrinsics
        return intr.window if split and hasattr(intr, "window") and self._bound else self.window

    def _window_open(self) -> bool:
        """Whether this step's sweep estimate joins the hand-over window."""
        c = self.cfg
        return (self._softmin_stage() and c.regression_after is not None and
                self.global_step >= c.regression_after - c.regression_window)

    def _append_window(self, split: bool = False):
        """Append the sweep's focal estimate to the open window: a scalar, or (B,) for several videos; B
        networks' Models each keep their own video's scalars."""
        if self._window_open() and self._net_videos:
            for m, f in zip(self.models, self._sw_focal.clone().unbind()):
                m.intrinsics.window.append(f)
        elif self._window_open():
            self._window(split).append(self._sw_focal[0].clone() if self._layout is None else self._sw_focal.clone())

    def _hand_over(self, split: bool = False):
        """At global_step == regression_after, seed the regressed focal length (each video's) with the
        window's mean; the stacked window is (n,) for one video, (n, B) for several."""
        if self._softmin and self.global_step == self.cfg.regression_after and self._net_videos:
            for b, m in enumerate(self.models):
                self._focal[b].copy_(torch.stack(m.intrinsics.window).mean())
        elif self._softmin and self.global_step == self.cfg.regression_after:
            self._focal.copy_(torch.stack(self._window(split)).mean(0))

    def _step_softmin(self, update: bool, **fields):
        """Sweep stage (intrinsics_softmin.py:84-141): focal estimate from the candidate sweep,
        the step itself with that focal length, the sweep's backward, then Adam.  `fields`: the step's
        tracks and metrics_log."""
        c = self.cfg
        f, w = max(self.frames), self._hw[1]
        st = torch.cuda.current_stream().cuda_stream
        # All-pixel Procrustes: the moment pass of the step does not have to wait for the focal length
        # the sweep is about to produce -- the sums for one K follow exactly from the sums for another
        # (fm_overfit_step_args.moments_k4) -- so it runs beside the sweep, on the candidate-0 intrinsics.
        early_moments = update and self._indices is None
        cur = torch.cuda.current_stream()
        with torch.cuda.device(self.rt.device):
            if early_moments:
                self._side_stream.wait_stream(cur)
                self._early_moments(st)
            with torch.cuda.stream(self._side_stream if early_moments else cur):
                idx = self._sweep_indices(clocked=update)
                self._sweep_forward(idx, torch.cuda.current_stream().cuda_stream)
            if early_moments:
                cur.wait_stream(self._side_stream)
            # all-pixel dense path: the logits of pairs >= 1 are updated inside the step (their
            # gradient is final there); depth and pair 0 wait for the sweep's backward
            # (one video only: the fused update defers pair 0 of the batch, not pair 0 of every video)
            fuse = (update and c.use_correspondence_weights and self._indices is None and w % 4 == 0 and
                    self._layout is None)
            self._call_step(focal=_ptr(self._sw_focal), step=int(fuse), defer_adam=int(fuse),
                            moments_k4=_ptr(self._k4_base) if early_moments else None, **fields)
            # The sweep's backward only touches the gradients of frames 0 / 1 (the candidate Procrustes
            # runs on the first pair): the depth update of every other frame runs beside it on a second
            # stream (a parallel branch of the captured step), frames 0 / 1 follow the sweep.
            side, cur = None, torch.cuda.current_stream()
            if update and f > 2:
                side = self._side_stream
                side.wait_stream(cur)
                with torch.cuda.stream(side):
                    self._adam_frames(0, 2, f)
            self._sweep_backward(idx, st)
        if update:
            self._adam_frames(0, 0, 2)
            if c.use_correspondence_weights:
                self._adam_frames(1, 0, 1 if fuse else f - 1)  # pair 0 only when the rest was fused
            if side is not None:
                cur.wait_stream(side)

    # ---- split step: the two halves of one iteration WITHOUT the parameter update, for callers that
    # need the loss values before they decide on the backward (torch.autograd: flowmap_b200.fused)
    def forward_phase(self, global_step: int, training: bool = True, depth: Optional[Tensor] = None,
                      weights: Optional[Tensor] = None, tracking: bool = False):
        """Poses + flow loss with its direct gradients (fm_overfit_step, FM_STEP_FORWARD; the
        candidate sweep first in the softmin stage).  Returns the weighted flow loss (device scalar,
        a buffer that the next call overwrites; (B,) per-video losses for a network's batch of B videos).
        Bound to a network backbone, `depth` (B, F, H, W) and, with correspondence weights, `weights`
        (B, F-1, H, W) are the step's contiguous float32 inputs (B = 1 but for a network's batch); they stay
        referenced until the next call (backward_phase reads them).  B networks' videos (a list of Models):
        `depth` (T, H, W) and `weights` (T - B, H, W) packed along the frame axis, and `tracking` adds the chained
        poses and every video's tracking loss (track_losses()) to this half."""
        if not self._network:
            self._refuse_videos("the split-step surface")
        f, (h, w) = self.frames[0], self._hw
        if self._network:
            self._bind_inputs(depth, weights, f, h, w)
        elif depth is not None or weights is not None:
            raise ValueError("flowmap_b200: an explicit-depth optimiser reads its own depth and weights")
        st = torch.cuda.current_stream().cuda_stream
        self.global_step = global_step
        self._begin_step()
        tracks = None
        if tracking:
            if not self._net_videos or self._packed is None:
                raise ValueError("flowmap_b200: forward_phase(tracking=True) serves B networks' videos with tracks")
            tracks = self._ctypes.pointer(self._pk_c)
        self._sweep_idx = None
        with torch.cuda.device(self.rt.device):
            if self._softmin_stage():
                self._sweep_idx = self._sweep_indices(split=True)
                self._sweep_forward(self._sweep_idx, st)
                focal = self._sw_focal
                if training:
                    self._append_window(split=True)
            else:
                if training:
                    self._hand_over(split=True)
                focal = self._focal
            self._call_step("fm_overfit_step (forward)", phase=1, tracks=tracks, focal=_ptr(focal))  # FM_STEP_FORWARD
        return self._loss

    def track_losses(self) -> Tensor:
        """The (B,) weighted tracking losses of the last forward_phase(tracking=True) (a buffer that the next
        call overwrites)."""
        return self._track_loss

    def _bind_inputs(self, depth, weights, f, h, w):
        """Point the step at a network backbone's depths / weights of this step."""
        use_w, b = self.cfg.use_correspondence_weights, self.B
        shapes = ((self.T, h, w), (self.T - b, h, w)) if self._net_videos else ((b, f, h, w), (b, f - 1, h, w))
        for name, t, shape in (("depth", depth, shapes[0]), ("weights", weights if use_w else None, shapes[1])):
            if t is None and (name == "depth" or use_w):
                raise ValueError(f"flowmap_b200: a network backbone's step needs its `{name}`")
            if t is not None and (tuple(t.shape) != shape or t.dtype != torch.float32 or not t.is_contiguous()
                                  or t.device != self.rt.device):
                raise ValueError(f"flowmap_b200: `{name}` must be a contiguous float32 {shape} tensor on {self.rt.device}")
        self._depth, self._wlog = depth, weights if use_w else None
        self._args.depth = depth.data_ptr()
        self._args.weight_logits = weights.data_ptr() if use_w else None

    def tracking_forward_phase(self):
        """Chained poses + tracking loss of the step begun by forward_phase (loss_tracking.py:28-61).
        Returns the weighted tracking loss (device scalar buffer)."""
        from ._lib import check
        self._refuse_videos("the split-step surface")
        c, L, pk = self.cfg, self._lib, self._packed
        _, f, _, h, w = self.batch.videos.shape
        st = torch.cuda.current_stream().cuda_stream
        head = (_ptr(self._depth), _ptr(self._k4), _ptr(self._ext), _ptr(pk.seg), pk.num_segments, pk.max_rows,
                pk.max_points, _ptr(pk.xy), _ptr(pk.vis), pk.total, ops.MAPPINGS[c.mapping], c.delta,
                c.tracking_weight, _ptr(self._track_loss), _ptr(self._tws), f, h, w, 0, 0, f)
        with torch.cuda.device(self.rt.device):
            check(L.fm_pose_chain(_ptr(self.rt), _ptr(self._ext), 1, f, st), "fm_pose_chain")
            if self._gt:  # constant K: the sweep without intrinsics terms, as the backward half reads it
                check(L.fm_track_loss_fwd_const_k(*head, st), "fm_track_loss_fwd_const_k")
            else:
                check(L.fm_track_loss_fwd_sharded(*head, 1, st), "fm_track_loss_fwd")
        return self._track_loss

    def backward_phase(self, flow_scale=None, track_scale=None, with_tracking: bool = False):
        """Second half: [tracking backward,] Procrustes backward, focal gradient[, the sweep's
        backward].  flow_scale / track_scale: device float scalars d total / d loss (None = 1); a network's
        batch of videos takes one flow_scale for all of them, B networks' videos (B,) float32 tensors, one
        d total / d loss_b per video.  Leaves the gradients in gradients()."""
        if not self._network:
            self._refuse_videos("the split-step surface")
        st = torch.cuda.current_stream().cuda_stream
        # Without tracks this phase adds g_rt / track_g_k4 as a caller's pose / intrinsics gradient: a step
        # whose tracking loss is not enabled yet (loss.py:40-41) has none, whatever those buffers hold.
        tracking = (dict(tracks=self._ctypes.pointer(self._pk_c)) if with_tracking else
                    dict(g_rt=None, track_g_k4=None))
        with torch.cuda.device(self.rt.device):
            self._call_step("fm_overfit_step (backward)", phase=2,  # FM_STEP_BACKWARD
                            flow_grad_scale=_ptr(flow_scale), track_grad_scale=_ptr(track_scale), **tracking)
            if self._sweep_idx is not None:
                self._sweep_backward(self._sweep_idx, st)

    def _refuse_videos(self, what: str):
        if self._layout is not None:
            raise ValueError(f"flowmap_b200: {what} serves one video, not several")

    def _step_body(self, update: bool, track_on: bool, sweep: bool):
        """One step as a fixed launch sequence (no host-side step numbers: see ops.StepClock)."""
        if update:
            self._clock.tick(tick_focal=not sweep and not self._gt)
        fields = dict(tracks=self._ctypes.pointer(self._pk_c) if track_on else None,
                      # the metrics row is indexed by the step clock, which only update steps advance
                      metrics_log=self._mlog.data_ptr() if (update and self._mlog is not None) else None)
        if sweep:
            self._step_softmin(update, **fields)
        else:
            with torch.cuda.device(self.rt.device):
                self._call_step(step=int(update), **fields)
        if track_on:
            torch.add(self._loss, self._track_loss, out=self._total)
        else:
            self._total.copy_(self._loss)

    def _run_body(self, key, graphable: bool, body, ticks_focal: bool):
        """Run one step body: eagerly, or -- from its third run on -- as a replay of its CUDA graph
        (the body must tick the step clock first and be a fixed launch sequence)."""
        if graphable and self._eager_runs.get(key, 0) >= 2:
            g = self._graphs.get(key)
            if g is None:  # capture records the launches without running them: replayed right below
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, capture_error_mode="thread_local"):
                    body()
                self._graphs[key] = g
                self._clock.steps -= 1  # the capture's host-side tick was not executed
                self._clock.focal_steps -= int(ticks_focal)
            g.replay()
            self._clock.steps += 1
            self._clock.focal_steps += int(ticks_focal)
        else:
            body()
            if graphable:
                self._eager_runs[key] = self._eager_runs.get(key, 0) + 1

    def training_step(self, update: bool = True):
        """Returns (total loss (device tensor: a scalar, or the (B,) per-video totals), relative poses
        rt (B, F-1, 3, 4), or a list of (F_b - 1, 3, 4) for videos of different lengths)."""
        c = self.cfg
        if self._network:
            raise ValueError("flowmap_b200: a network backbone's step runs through the model's losses "
                             "(forward_phase / backward_phase), not training_step")
        self._begin_step()
        track_on = c.use_tracking and self.global_step >= c.tracking_enable_after
        sweep = self._softmin_stage()
        if update:
            self._clock.set(self.optimizer_steps, self.focal_steps)
            self._hand_over()
        window_on = self._window_open()
        key = (track_on, sweep, self.global_step >= c.flow_enable_after)
        graphable = (update and self.use_cuda_graph and not c.procrustes_randomize and not window_on and
                     getattr(self, "injected_indices", None) is None)
        ticks_focal = not sweep and not self._gt
        self._run_body(key, graphable, lambda upd=update: self._step_body(upd, track_on, sweep), ticks_focal)
        if update:
            self._append_window()
            self.global_step += 1
            self.optimizer_steps += 1
            self.focal_steps += int(ticks_focal)
        return self._total.clone(), self._per_video(self.rt, pairs=True)

    def extrinsics(self) -> Tensor:
        """Camera-to-world poses of the last step (projection.py:187-210): (B, F, 4, 4), or a list of
        (F_b, 4, 4) for videos of different lengths."""
        rt = self._per_video(self.rt, pairs=True)
        return ops.pose_chain(rt) if isinstance(rt, Tensor) else [ops.pose_chain(r[None])[0] for r in rt]

    def gradients(self):
        """d loss / d depth, weights and focal length of the last step; "focal" is None with ground-truth K."""
        depth, g_focal = self._per_video(self._g_depth), self._g_focal
        return {"depth": depth, "weights": self._per_video(self._g_w, pairs=True),
                "focal": g_focal if g_focal is None or isinstance(depth, Tensor) else list(g_focal.unbind())}

    def set_intrinsics(self, intrinsics):
        """Ground-truth intrinsics for the following steps, copied into the step's k4 buffer (captured CUDA
        graphs stay valid): (1, F, 3, 3) for one video, (B, F, 3, 3) for a tensor batch, a list of the videos'
        (1, F_b, 3, 3) for a list of Batches; normalised as in the reference.  ValueError on a missing, wrongly
        shaped or non-finite K (the finiteness check synchronises with the host)."""
        per = self._check_intrinsics(intrinsics)
        finite = torch.isfinite(per.flatten(1)).all(1) if isinstance(per, Tensor) else \
            torch.stack([torch.isfinite(k).all() for k in per])
        bad = (~finite).nonzero()
        if bad.numel():
            raise ValueError(f"flowmap_b200: the intrinsics of video {int(bad[0, 0])} are not finite")
        self._write_k4(intrinsics)

    def _check_intrinsics(self, intrinsics):
        """The shape checks of a ground-truth K (host only): the (B, F, 3, 3) tensor of one video or a tensor
        batch, or the list of a list of Batches."""
        if not self._gt:
            raise ValueError("flowmap_b200: set_intrinsics needs cfg.intrinsics = 'ground_truth'")
        if intrinsics is None:
            raise ValueError("flowmap_b200: ground-truth intrinsics need batch.intrinsics")
        if isinstance(intrinsics, (list, tuple)):
            if self._layout is None or self._tensor_batch:
                raise ValueError("flowmap_b200: one intrinsics tensor for this optimiser, not a list")
            per = list(intrinsics)
        else:
            if self._layout is not None and not self._tensor_batch:
                raise ValueError(f"flowmap_b200: videos of different lengths need a list of {self.B} intrinsics")
            if intrinsics.dim() != 4:
                raise ValueError(f"flowmap_b200: intrinsics must be (B, F, 3, 3), got {tuple(intrinsics.shape)}")
            # a tensor holds videos of one length: video 0's shape stands for all of them
            per = [intrinsics[:1]] * intrinsics.shape[0]
        if len(per) != self.B:
            raise ValueError(f"flowmap_b200: intrinsics for {len(per)} videos, the optimiser holds {self.B}")
        for i, (k, f) in enumerate(zip(per, self.frames)):
            if k is None:
                raise ValueError(f"flowmap_b200: video {i} carries no intrinsics (batch.intrinsics)")
            if tuple(k.shape) != (1, f, 3, 3):
                raise ValueError(f"flowmap_b200: the intrinsics of video {i} must be (1, {f}, 3, 3), got "
                                 f"{tuple(k.shape)}")
        return intrinsics if isinstance(intrinsics, Tensor) else per

    def _write_k4(self, intrinsics):
        """Copy a ground-truth K into the step's k4 buffer without synchronising the host: the shape checks of
        set_intrinsics, no finiteness check (a non-finite K gives a non-finite loss, as in the reference).  A
        tensor converts as one batched op."""
        k = self._check_intrinsics(intrinsics)
        k = k.reshape(-1, 3, 3) if isinstance(k, Tensor) else torch.cat([t[0].to(self._k4.device) for t in k])
        self._k4.copy_(ops.intrinsics_to_k4(k))

    def intrinsics_k4(self) -> Tensor:
        """(F, 4) = (fx, fy, cx, cy) used by the last step; (B, F, 4) for a (B, F) tensor batch; a list of
        (F_b, 4) for videos of different lengths."""
        return self._per_video(self._k4)

    METRIC_NAMES = ("train/loss/flow", "train/loss/tracking", "train/intrinsics/fx_error",
                    "train/intrinsics/fy_error", "metrics/ate")

    def enable_metrics_log(self, capacity: int):
        """Log, from inside every update step, what the reference logs for it: the weighted flow and
        tracking losses (loss.py:40: 0 before the tracking loss is enabled), the focal-length errors
        (model_wrapper_overfit.py:63-71) against the frame means of `batch.intrinsics`, and the ATE of
        the step's camera centres against `batch.extrinsics[0, :, :3, 3]` (metrics/ate of
        VisualizerTrajectory, scipy.spatial.procrustes semantics, fm_trajectory_ate).  Columns without
        ground truth are NaN.  The rows live in a device ring of `capacity` steps, written without host
        synchronisation; read them with metrics_log().

        Row k describes update k (0-based, global_step = k when it ran): the poses and intrinsics that
        update evaluated, before its Adam step -- the values the reference's training_step logs at
        global_step k.  The reference's validation after update k (experiment/dump_ate.yaml's
        val_check_interval: 1) evaluates the updated parameters: that is row k + 1."""
        if self._net_videos:
            raise ValueError("flowmap_b200: B networks' overfits run the split step, which writes no metrics log")
        if capacity < 1:
            raise ValueError("flowmap_b200: the metrics log needs a capacity >= 1")
        dev, nan = self.rt.device, float("nan")
        gts, fxfy = [], []  # each video's ground truth
        for bt in self.batches:
            gts.append(None if bt.extrinsics is None else
                       bt.extrinsics[0, :, :3, 3].to(device=dev, dtype=torch.float32))
            k = None if bt.intrinsics is None else bt.intrinsics[0].double()
            fxfy.append(torch.tensor([nan, nan], dtype=torch.float64) if k is None else
                        torch.stack((k[:, 0, 0].mean(), k[:, 1, 1].mean())).cpu())
        # the camera centres packed like the frames, NaN for a video without them; none at all: no ATE
        self._mlog_gt = None if all(g is None for g in gts) else torch.cat(
            [torch.full((f, 3), nan, device=dev) if g is None else g for g, f in zip(gts, self.frames)]).contiguous()
        fxfy = torch.stack(fxfy)
        self._mlog_fxfy = fxfy.to(device=dev, dtype=torch.float32).contiguous()
        if getattr(self, "_ext", None) is None:  # flow-only steps chain the poses for the log
            self._ext = torch.empty(*self._lead[0], 4, 4, device=dev)
        self._mlog = torch.full((capacity, *self._lead[2], 5), nan, device=dev)
        self._mlog_first = self.optimizer_steps
        a = self._args
        a.extrinsics = self._ext.data_ptr()
        a.gt_positions = None if self._mlog_gt is None else self._mlog_gt.data_ptr()
        # the one-video step reads its video's fx / fy as scalars, packed videos the (B, 2) rows
        (a.gt_fx, a.gt_fy), a.gt_fxfy, a.metrics_capacity = fxfy[0].tolist(), self._mlog_fxfy.data_ptr(), capacity
        self._graphs.clear()  # captured steps were recorded without the log
        self._eager_runs.clear()

    def metrics_log(self) -> dict:
        """The logged rows of the update steps run since enable_metrics_log (the last `capacity` of
        them), in step order, as CPU float32 tensors keyed by the reference's log names: (steps,), or
        (steps, B) with B videos.  One host synchronisation."""
        if self._mlog is None:
            raise ValueError("flowmap_b200: the metrics log is off (enable_metrics_log)")
        cap = self._mlog.shape[0]
        steps = torch.arange(max(self._mlog_first, self.optimizer_steps - cap), self.optimizer_steps)
        rows = self._mlog[(steps % cap).to(self._mlog.device)].cpu()
        return {name: rows[..., i] for i, name in enumerate(self.METRIC_NAMES)}

    # ---- checkpoints: the format and the interchange with torch.optim.Adam live in flowmap_b200.checkpoint
    def _refuse_checkpoint(self):
        if self._bound:
            raise ValueError("flowmap_b200: an optimiser bound to a caller's Model (model=) keeps no Adam state: "
                             "checkpoint the Model and the caller's torch optimiser")

    def _adam_slots(self, b: int):
        """Video b's Adam state as torch.optim.Adam holds it for models[b].parameters(): per parameter its
        (exp_avg, exp_avg_sq) views of the packed moments and its update count."""
        s, f0, f = self._state, self._first[b], self.frames[b]
        rows = lambda t, p: t if self._layout is None else t[f0 - p * b:f0 - p * b + f - p]  # noqa: E731
        moments = [(rows(s[0], 0), rows(s[1], 0)), (rows(s[2], 1), rows(s[3], 1))]
        if s[4] is not None:  # softmin without a regression stage has a buffer here but no focal parameter
            moments.append((s[4], s[5]) if self._layout is None else (s[4][b], s[5][b]))
        steps = checkpoint.adam_steps(self.cfg, self.optimizer_steps, self.focal_steps)
        return [(m, v, n) for (m, v), n in zip(moments, steps)]

    def state_dict(self) -> dict:
        """The run's state (flowmap_b200.checkpoint): each video's Model.state_dict() and torch.optim.Adam
        state, the step counters, the softmin hand-over window and the step clock's seed; not the settings
        use_cuda_graph and injected_indices, nor the metrics log.  No host synchronisation: the tensors are
        clones on the optimiser's device, made on the current stream (Adam's `step` entries are CPU scalars,
        as in torch).  A run under cfg.procrustes_randomize draws its point sets from torch's RNG, which is
        not saved: its resumed point sets differ from those of the uninterrupted run."""
        self._refuse_checkpoint()
        videos = [checkpoint.video_entry(f, {k: t.clone() for k, t in m.state_dict().items()}, self._adam_slots(b),
                                         self.cfg.lr) for b, (m, f) in enumerate(zip(self.models, self.frames))]
        window = torch.stack(self.window) if self._softmin and self.window else None
        return checkpoint.new_state(self.cfg, self.global_step, self.optimizer_steps, self.focal_steps,
                                    self._clock.base_seed, window, videos)

    def load_state_dict(self, state: dict) -> None:
        """Continue the run of `state` on this optimiser, built on the same inputs: parameters and moments
        are copied into the packed buffers in place (captured CUDA graphs stay valid), the counters, window
        and seed replace this optimiser's.  ValueError naming the field when the format, cfg, number of
        videos, frames per video, H x W or intrinsics mode differ; the Flows, tracks and ground-truth K are
        inputs, not state."""
        self._refuse_checkpoint()
        checkpoint.check(state, self.cfg, self.frames, self._hw)
        with torch.no_grad():
            for b, (m, v) in enumerate(zip(self.models, state["videos"])):
                m.load_state_dict(v["model"])  # copy_ into the parameters: views of the packed buffers
                checkpoint.load_moments(v["optimizer"], self._adam_slots(b))
        self.global_step, self.optimizer_steps, self.focal_steps = (
            int(state[k]) for k in ("global_step", "optimizer_steps", "focal_steps"))
        if self._softmin:
            w = state["window"]
            self.window = [] if w is None else list(w.to(self.rt.device).clone().unbind(0))
        seed = int(state["base_seed"])
        if seed != self._clock.base_seed:  # a captured step holds the seed as a launch argument of its tick
            self._clock.base_seed = seed
            self._graphs.clear()
            self._eager_runs.clear()
        self._clock.set(self.optimizer_steps, self.focal_steps)


class ShardedFusedOverfitter(FusedOverfitter):
    """Pair-sharded :class:`FusedOverfitter` (flowmap_b200.parallel, SURVEY 8(e)).

    Every rank holds the frames / pairs of its ShardPlan and runs fm_overfit_step on them
    without the Adam part; ONE all-reduce carries the loss, the focal-length gradient and the
    boundary depth-gradient frames, then each rank applies Adam to its parameters (replicas of
    a boundary frame see identical gradients).

    Tracking loss (not pair-local: a track segment spans up to 41 frames): the step is split
    (FM_STEP_FORWARD / FM_STEP_BACKWARD).  In between, the relative poses are gathered (149 x 12
    floats), every rank chains them, evaluates the tracking loss for the SOURCE frames it owns
    against all target frames, the loss sum / valid count / per-frame pose and intrinsics sums
    (F x 10 doubles) are all-reduced, and every rank backpropagates the (now global) pose
    gradient through the chain to its own pairs.  `tracks` are the global segments.

    Softmin intrinsics: the candidate sweep lives on the rank that owns pair 0; its focal
    estimate is broadcast before the step and its backward runs after the step's all-reduce
    (the summed d loss / d focal), so the sweep adds two one-float collectives."""

    def __init__(self, cfg: OverfitCfg, batch: Batch, flows: Flows, plan, tracks=None, device="cuda",
                 group=None):
        from . import parallel
        from ._lib import lib
        if isinstance(batch, (list, tuple)) or batch.videos.shape[0] != 1:
            raise ValueError("flowmap_b200: pair sharding optimises one video (batch size 1)")
        if cfg.intrinsics == "ground_truth":
            raise ValueError("flowmap_b200: pair sharding does not serve ground-truth intrinsics")
        super().__init__(replace(cfg, use_tracking=False), batch, flows, None, device)
        self.cfg = cfg
        self.plan, self.group = plan, group
        _, f_local, _, h, w = batch.videos.shape
        if f_local != plan.num_local_frames:
            raise ValueError("flowmap_b200: batch does not match the shard plan")
        dev = self.rt.device
        self.reducer = parallel.StepReducer(plan, (h, w), dev, 2, group)
        self._msum.copy_(parallel.global_mask_sum(self._msum, group))  # in place: args hold its address
        if self._softmin and plan.world > 1 and plan.pair_range[1] - plan.pair_range[0] < 2 and plan.rank == 0:
            raise ValueError("flowmap_b200: the rank owning pair 0 needs >= 2 pairs in the softmin stage")
        if cfg.use_tracking:
            if tracks is None:
                raise ValueError("flowmap_b200: use_tracking needs the (global) track segments")
            F = plan.num_pairs_total + 1
            pk = ops.PackedTracks([t.to(dev) for t in tracks], dev)
            self._packed, self._F = pk, F
            z = lambda *shape: torch.zeros(*shape, device=dev)  # noqa: E731
            self._rt_all, self._g_rt_all = z(1, F - 1, 3, 4), z(1, F - 1, 3, 4)
            self._ext_all, self._g_ext_all = z(1, F, 4, 4), z(1, F, 4, 4)
            self._tg_k4_all = z(F, 4)
            self._g_rt_local = z(1, f_local - 1, 3, 4)
            self._tws = torch.empty(lib().fm_track_workspace_bytes(F, pk.total), dtype=torch.uint8, device=dev)
            self._treduce = self._tws[:lib().fm_track_reduce_bytes(F)].view(torch.float64)
            self._src_range = parallel.source_frame_range(plan)

    def enable_metrics_log(self, capacity: int):
        raise ValueError("flowmap_b200: the per-step metrics log covers the single-GPU FusedOverfitter; a "
                         "pair-sharded rank holds only part of the trajectory")

    def _refuse_checkpoint(self):
        raise ValueError("flowmap_b200: checkpoints cover the single-GPU FusedOverfitter; a pair-sharded rank "
                         "holds only part of the video's state")

    def _mask_sum(self, flows: Flows) -> Tensor:
        from . import parallel
        return parallel.global_mask_sum(ops.mask_sum(flows.forward_mask, flows.backward_mask), self.group)

    def sync_boundary_depth(self):
        """Make the replicas of every shared boundary frame identical (owner = left rank)."""
        import torch.distributed as dist
        p = self.plan
        if p.world == 1:
            return
        buf = torch.zeros(p.world - 1, *self._depth.shape[1:], device=self._depth.device)
        if p.has_right:
            buf[p.rank].copy_(self._depth[-1])
        dist.all_reduce(buf, group=self.group)
        if p.has_left:
            self._depth[0].copy_(buf[p.rank - 1])

    def _first_rank(self) -> int:
        import torch.distributed as dist
        return 0 if self.group is None else dist.get_global_rank(self.group, 0)

    def _tracking_exchange(self, h: int, w: int):
        """Between the two halves of a split step; returns tracking's d loss / d focal (global)."""
        import torch.distributed as dist
        from . import parallel
        from ._lib import check
        c, L, pk, F = self.cfg, self._lib, self._packed, self._F
        a0, b0 = self.plan.pair_range
        st = torch.cuda.current_stream().cuda_stream
        parallel.gather_pairs(self.plan, self.rt, self._rt_all, self.group)
        k4_all = self._k4[0].expand(F, 4).contiguous()  # one shared focal length
        args = (_ptr(k4_all), _ptr(self._ext_all), _ptr(pk.seg), pk.num_segments, pk.max_rows, pk.max_points,
                _ptr(pk.xy), _ptr(pk.vis), pk.total, ops.MAPPINGS[c.mapping], c.delta, c.tracking_weight)
        tail = (F, h, w, a0, self._src_range[0], self._src_range[1])
        with torch.cuda.device(self.rt.device):
            check(L.fm_pose_chain(_ptr(self._rt_all), _ptr(self._ext_all), 1, F, st), "fm_pose_chain")
            check(L.fm_track_loss_fwd_sharded(_ptr(self._depth), *args, None, _ptr(self._tws), *tail, 1, st),
                  "fm_track_loss_fwd_sharded")  # shared focal: only the summed K gradient is used
            if self.plan.world > 1:
                dist.all_reduce(self._treduce, group=self.group)
            check(L.fm_track_loss_value(_ptr(self._tws), c.tracking_weight, _ptr(self._track_loss), st),
                  "fm_track_loss_value")
            check(L.fm_track_loss_bwd_sharded(_ptr(self._depth), *args, None, _ptr(self._g_depth),
                                              _ptr(self._g_ext_all), _ptr(self._tg_k4_all), _ptr(self._tws), *tail, st),
                  "fm_track_loss_bwd_sharded")
            check(L.fm_pose_chain_bwd(_ptr(self._rt_all), _ptr(self._ext_all), _ptr(self._g_ext_all),
                                      _ptr(self._g_rt_all), 1, F, st), "fm_pose_chain_bwd")
        self._g_rt_local.copy_(self._g_rt_all[:, a0:b0])
        scale = (h * w) ** 0.5
        return (self._tg_k4_all[:, 0].double().sum() * (scale / w) +
                self._tg_k4_all[:, 1].double().sum() * (scale / h)).float()

    def _flow_only_body(self):
        """Flow loss with a regressed focal length, update step, as a fixed launch sequence: the step
        (weight-logit Adam fused in), the exchange started, Adam on the interior depth frames WHILE the
        boundary frames and the two scalars travel, then the boundary frames and the focal length."""
        p, r = self.plan, self.reducer
        clk = self._clock
        clk.tick(tick_focal=True)
        with torch.cuda.device(self.rt.device):
            # the step writes its two scalars (loss, d focal) straight into the all-reduce buffer
            self._call_step(step=1, defer_adam=2, loss=r.scal[0:1].data_ptr(), g_focal=r.scal[1:2].data_ptr())
        reqs = r.start(self._g_depth)
        stt, n = self._state, self._depth.shape[0]
        lo, hi = int(p.has_left and p.world > 1), n - int(p.has_right and p.world > 1)
        if hi > lo:
            ops.adam_step_clock(self._depth[lo:hi], self._g_depth[lo:hi], stt[0][lo:hi], stt[1][lo:hi], clk)
        red = r.finish(reqs, self._g_depth)
        if lo > 0:
            ops.adam_step_clock(self._depth[:1], self._g_depth[:1], stt[0][:1], stt[1][:1], clk)
        if hi < n:
            ops.adam_step_clock(self._depth[n - 1:], self._g_depth[n - 1:], stt[0][n - 1:], stt[1][n - 1:], clk)
        ops.adam_step_clock(self._focal.reshape(1), red[1:2], stt[4].reshape(1), stt[5].reshape(1), clk,
                            focal_clock=True)
        self._total.copy_(red[0])

    def training_step(self, update: bool = True):
        import torch.distributed as dist
        c, p = self.cfg, self.plan
        _, _, _, h, w = self.batch.videos.shape
        self._begin_step()
        if (update and not self._softmin and not c.procrustes_randomize and self._indices is None and
                c.use_correspondence_weights and w % 4 == 0 and
                not (c.use_tracking and self.global_step >= c.tracking_enable_after)):
            self._clock.set(self.optimizer_steps, self.focal_steps)
            self._run_body(("flow", self.global_step >= c.flow_enable_after), self.use_cuda_graph,
                           self._flow_only_body, True)
            self.global_step += 1
            self.optimizer_steps += 1
            self.focal_steps += 1
            return self._total.clone(), self.rt
        st = torch.cuda.current_stream().cuda_stream
        dev = self.rt.device
        track_on = c.use_tracking and self.global_step >= c.tracking_enable_after
        sweep = self._softmin_stage()
        own_sweep = sweep and p.rank == 0
        # the weight logits' gradient is rank-local and final inside the step: update them there
        # (all pairs, or pairs >= 1 on the rank whose sweep still touches pair 0); depth and the
        # focal length wait for the exchange below
        fuse_w = update and c.use_correspondence_weights and self._indices is None and w % 4 == 0
        if update:
            self._clock.set(self.optimizer_steps, self.focal_steps)
            self._clock.tick(tick_focal=not sweep)
        fields = dict(step=int(fuse_w), defer_adam=(1 if own_sweep else 2) if fuse_w else 0)
        if sweep:
            if own_sweep:
                idx = self._sweep_indices()
                with torch.cuda.device(dev):
                    self._sweep_forward(idx, st)
            if p.world > 1:
                dist.broadcast(self._sw_focal, src=self._first_rank(), group=self.group)
            fields["focal"] = _ptr(self._sw_focal)
        elif update:
            self._hand_over()  # identical on all ranks
        extra_focal = None
        with torch.cuda.device(dev):
            if track_on:
                self._call_step("fm_overfit_step (forward)", phase=1, **fields)  # FM_STEP_FORWARD
                extra_focal = self._tracking_exchange(h, w)
                self._call_step("fm_overfit_step (backward)", phase=2, g_rt=_ptr(self._g_rt_local),  # FM_STEP_BACKWARD
                                track_g_k4=None, **fields)
            else:
                self._call_step(**fields)
        g_focal = self._g_focal.reshape(())
        if extra_focal is not None and p.rank == 0:  # global value, counted once
            g_focal = g_focal + extra_focal
        red = self.reducer.reduce(torch.stack((self._loss.reshape(()), g_focal)), self._g_depth)
        self._g_focal.copy_(red[1])
        if own_sweep:  # backward of the sweep with the summed focal gradient: frames 0/1, pair 0
            with torch.cuda.device(dev):
                self._sweep_backward(idx, st)
        if update:
            stt, clk = self._state, self._clock
            ops.adam_step_clock(self._depth, self._g_depth, stt[0], stt[1], clk)
            if c.use_correspondence_weights and (not fuse_w or own_sweep):
                k = 1 if fuse_w else self._wlog.shape[0]  # pair 0 only when the rest was fused
                ops.adam_step_clock(self._wlog[:k], self._g_w[:k], stt[2][:k], stt[3][:k], clk)
            self._append_window()
            if not sweep:
                self.focal_steps += 1
                ops.adam_step_clock(self._focal.reshape(1), self._g_focal.reshape(1), stt[4].reshape(1),
                                    stt[5].reshape(1), clk, focal_clock=True)
            self.global_step += 1
            self.optimizer_steps += 1
        total = red[0] + self._track_loss if track_on else red[0]
        return total, self.rt

