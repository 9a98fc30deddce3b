"""Fused evaluation behind the reference-shaped API.

`Model.forward` -> `LossFlow.forward` / `LossTracking.forward` -> `total.backward()` is the surface
flowmap/model/model_wrapper_overfit.py:51-73 drives.  Evaluated op by op it costs one C-ABI call
and several ATen launches per module; here the same surface runs on the two halves of the fused
step (fm_overfit_step, FM_STEP_FORWARD / FM_STEP_BACKWARD):

  * `Model.forward` launches nothing and returns a `LazyModelOutput` (with ground-truth intrinsics an
    ordinary ModelOutput that holds the batch's K: `fused_output`);
  * the first `LossFlow.forward` of the step runs the forward half (candidate sweep in the softmin
    stage, Procrustes poses, flow loss with its direct gradients) and returns the loss value as the
    output of an autograd node; `LossTracking.forward` adds the tracking sweep;
  * all loss nodes hang off ONE root node whose inputs are the model's parameters; autograd calls
    its backward once, after every loss has reported its grad_output, and that call runs the
    backward half and hands the finished parameter gradients to autograd (no intermediate tensors,
    no per-op ATen glue).

A network backbone (any backbone but BackboneExplicitDepth, e.g. the reference's BackboneMidas: a CNN
for the depths, a per-pixel MLP or sigmoid(s * weights) for the correspondence weights) stays in
torch.  `Model.forward` runs it once, under autograd, and the step's output keeps its BackboneOutput.
The root's inputs are then that step's depths and weights, converted to contiguous float32 inside the
graph; the halves read them with weight sensitivity 0 (the weights themselves, not logits), and the
root's backward hands d loss / d depths and d loss / d weights to autograd, which carries them on into
the network.  Outputs read before or after the losses reuse the stored BackboneOutput: the backbone
never runs twice in one step.

A network backbone's batch of several videos (the pretraining step, pretrain.py) runs on the packed layout
of fm_overfit_step_videos when its intrinsics are softmin without a regression stage, or ground truth, and no
tracks come with it: one candidate sweep and one focal length per video (or each video's own per-frame K), and
LossFlow's one pooled mask sum for the whole batch (loss_flow.py:31-70), written into every video's slot, so
that the step's (B,) losses sum to the loss autograd sees and one grad_output scales them all.

Ground-truth intrinsics (intrinsics_ground_truth.py) run the constant-intrinsics step for explicit depth, a
network on one video and a network's batch alike, when `batch.intrinsics` is a floating (B, F, 3, 3) tensor on
the flows' device: it is read into the step's k4 buffer before every forward half (a loader's new K, or the same
tensor rewritten in place), without a host synchronisation or a check of its values, as in the reference; no
focal length is learned and the snapshot reports k_mode "const".

Anything the fused step does not cover (a consumer that reads `model_output.extrinsics` under
autograd, several explicit-depth videos, a batch of several videos with a regressed focal length, a
regression stage or tracks, ground-truth intrinsics without a CUDA `batch.intrinsics`, eval mode, different
mappings for the two losses) makes the step's output materialise itself through the per-op autograd
Functions of flowmap_b200.ops: same results, the former speed.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor

from . import ops
from .types import BackboneOutput, Batch, Flows, ModelOutput


class _StepRoot(torch.autograd.Function):
    """Root of one fused step: token = f(parameters, or a network backbone's depths / weights).  Its
    backward runs the backward half."""

    @staticmethod
    def forward(ctx, step, *params):
        ctx.step = step
        return torch.empty((), dtype=torch.float32, device=params[0].device)

    @staticmethod
    def backward(ctx, _g_token):
        grads = ctx.step.run_backward()
        return (None, *(g if need else None for g, need in zip(grads, ctx.needs_input_grad[1:])))


class _LossNode(torch.autograd.Function):
    """One loss of the step (a scalar, or B networks' (B,) losses): value computed by the forward half, gradient
    deferred to the root."""

    @staticmethod
    def forward(ctx, token, step, which, value):
        ctx.step, ctx.which = step, which
        return value.clone()  # the engine's buffer is overwritten by the next step

    @staticmethod
    def backward(ctx, g):
        # one scalar, or (network_videos_step) one grad_output per video
        ctx.step.scales[ctx.which] = g.to(torch.float32).contiguous()
        return g, None, None, None


class FusedStep:
    """State of one optimisation step evaluated through the fused halves."""

    def __init__(self, model, batch: Batch, flows: Flows, global_step: int,
                 backbone_out: Optional[BackboneOutput] = None):
        self.model, self.batch, self.flows, self.global_step = model, batch, flows, global_step
        self.backbone_out = backbone_out  # a network backbone's output of this step, else None
        self.engine = None
        self.token: Optional[Tensor] = None
        self.scales = {}
        self.flow_done = self.track_done = False
        self.dead = False  # the output was materialised through the per-op path instead

    # ---- forward half
    def flow_loss(self, loss_mod, tracks) -> Optional[Tensor]:
        if self.dead or self.flow_done:
            return None
        eng = self.model._fused_engine(self.batch, self.flows, tracks, loss_mod)
        if eng is None:
            return None
        self.engine = eng
        eng.cfg.flow_weight, eng.cfg.flow_enable_after = loss_mod.cfg.weight, loss_mod.cfg.enable_after
        eng._msum.copy_(loss_mod._mask_total(self.flows))
        if eng._gt:  # this step's K: a loader brings a new one with every batch, or rewrites it in place
            eng._write_k4(self.batch.intrinsics)
        inputs = None
        if self.backbone_out is not None:  # the kernels read float32 rows; the casts stay in the graph
            bo = self.backbone_out
            inputs = [bo.depths.to(torch.float32).contiguous()]
            if eng.cfg.use_correspondence_weights:
                inputs.append(bo.weights.to(torch.float32).contiguous())
        params = self.model._fused_params(self.global_step, inputs)
        for p, buf in zip(params, self._grad_buffers(params)):
            if p.is_leaf and p.grad is not None and buf is not None and p.grad.data_ptr() == buf.data_ptr():
                p.grad = p.grad.clone()  # a kept gradient must not alias the buffer about to be rewritten
        self._params = params
        value = eng.forward_phase(self.global_step, training=self.model.training,
                                  depth=None if inputs is None else inputs[0].detach(),
                                  weights=inputs[1].detach() if inputs is not None and len(inputs) > 1 else None)
        self.token = _StepRoot.apply(self, *params)
        self.flow_done = True
        if value.dim():  # a batch of videos: each normalised by the pooled mask sum, their sum is LossFlow's value
            value = value.sum()
        return _LossNode.apply(self.token, self, "flow", value)

    def track_loss(self, loss_mod, tracks) -> Optional[Tensor]:
        eng = self.engine
        if self.dead or not self.flow_done or self.track_done or eng is None or eng._packed is None:
            return None
        fm = eng.cfg
        lm = loss_mod.cfg.mapping
        if lm.name != fm.mapping or getattr(lm, "delta", fm.delta) != fm.delta:
            return None  # the fused step evaluates both losses with one mapping
        fm.tracking_weight = loss_mod.cfg.weight
        eng._args.track_weight = loss_mod.cfg.weight
        value = eng.tracking_forward_phase()
        self.track_done = True
        return _LossNode.apply(self.token, self, "tracking", value)

    # ---- backward half
    def _grad_buffers(self, params):
        eng = self.engine
        g = eng.gradients()
        bufs = [g["depth"]]
        if eng.cfg.use_correspondence_weights:
            bufs.append(g["weights"])
        if len(params) > len(bufs):
            bufs.append(g["focal"])
        return bufs

    def run_backward(self):
        eng = self.engine
        eng.backward_phase(self.scales.get("flow"), self.scales.get("tracking"), with_tracking=self.track_done)
        out = []
        for p, buf in zip(self._params, self._grad_buffers(self._params)):
            # a fresh alias of the persistent buffer: autograd adopts it as .grad without a copy
            out.append(buf.detach().view(p.shape))
        return tuple(out)

    def snapshot(self) -> ModelOutput:
        """Detached ModelOutput of the step the forward half evaluated (for logging / visualisers
        that read the output after the losses): poses and intrinsics come from the engine's buffers."""
        eng, model = self.engine, self.model
        b, f = self.batch.videos.shape[:2]
        with torch.no_grad():
            k4 = eng.intrinsics_k4().reshape(b, f, 4).clone()
            rt = eng.rt.reshape(b, f - 1, 3, 4).clone()
            k = torch.zeros(b, f, 3, 3, device=k4.device)
            k[..., 0, 0], k[..., 1, 1], k[..., 0, 2], k[..., 1, 2], k[..., 2, 2] = \
                k4[..., 0], k4[..., 1], k4[..., 2], k4[..., 3], 1.0
            bo = self.backbone_out
            if bo is None:
                bo = model.backbone.forward(self.batch, self.flows)
            weights = bo.weights if model.cfg.use_correspondence_weights else torch.ones_like(bo.weights)
            return ModelOutput(bo.depths.detach(), None, k, ops.pose_chain(rt), weights.detach(), relative=rt, k4=k4,
                               k_mode="const" if eng._gt else "shared_focal")


def _bind(out: ModelOutput, model, batch: Batch, flows: Flows, global_step: int,
          backbone_out: Optional[BackboneOutput]):
    """Make `out` the output of a fused step: `depths` is the parameter itself (explicit depth) or the network
    backbone's output, as are a network backbone's `backward_correspondence_weights`; ModelOutput.__getattr__
    takes every attribute that is not set from materialize(out)."""
    d = out.__dict__
    d["_fused"], d["_full"] = FusedStep(model, batch, flows, global_step, backbone_out), None
    if backbone_out is None:
        d["depths"] = model.backbone.depth[None]
    else:
        weights = backbone_out.weights
        if not model.cfg.use_correspondence_weights:  # model.py:67-68
            weights = torch.ones_like(weights)
        d["depths"], d["backward_correspondence_weights"] = backbone_out.depths, weights


def materialize(out: ModelOutput) -> ModelOutput:
    """What the output of a fused step computes when it is read: before the losses the differentiable per-op
    evaluation (which retires the fused step for this iteration), after them the detached snapshot of the step."""
    d = out.__dict__
    if d["_full"] is None:
        fused = d["_fused"]
        if fused.flow_done:  # the fused losses already consumed this output: values only
            d["_full"] = fused.snapshot()
        else:
            fused.dead = True
            d["_full"] = fused.model._forward_materialized(fused.batch, fused.flows, fused.global_step,
                                                           fused.backbone_out)
    return d["_full"]


class LazyModelOutput(ModelOutput):
    """ModelOutput of a fused step whose intrinsics come out of the step (a regressed focal length, or the softmin
    sweep's): everything but `depths` (and a network backbone's weights) is computed when (and only if) somebody
    reads it, through materialize()."""

    def __init__(self, model, batch: Batch, flows: Flows, global_step: int,
                 backbone_out: Optional[BackboneOutput] = None):
        _bind(self, model, batch, flows, global_step, backbone_out)


def fused_output(model, batch: Batch, flows: Flows, global_step: int,
                 backbone_out: Optional[BackboneOutput] = None) -> ModelOutput:
    """The output Model.forward returns for a step the losses evaluate on the fused halves.  With ground-truth
    intrinsics the step does not change K: the output is an ordinary ModelOutput that holds the batch's intrinsics
    and k_mode "const" (reading them keeps the step fused, as in the per-op path they are the batch's own), and
    computes its poses, k4 and surfaces when they are read.  Otherwise a LazyModelOutput."""
    from .model import IntrinsicsGroundTruth
    if not isinstance(model.intrinsics, IntrinsicsGroundTruth):
        return LazyModelOutput(model, batch, flows, global_step, backbone_out)
    out = ModelOutput.__new__(ModelOutput)
    _bind(out, model, batch, flows, global_step, backbone_out)
    out.__dict__.update(intrinsics=batch.intrinsics, k_mode="const")
    return out


class _VideosStep:
    """One step of B networks' overfits on the packed split halves (network_videos_step): the state that
    _StepRoot and the two _LossNodes share.  Its scales are (B,) grad_outputs, one per video."""

    def __init__(self, engine, params, focal_params):
        self.engine, self._params, self._focal_params = engine, params, focal_params
        self.scales = {}
        self.track_done = False

    def run_backward(self):
        eng = self.engine
        dev = eng.rt.device
        zeros = torch.zeros(eng.B, dtype=torch.float32, device=dev)
        # a loss that did not reach the objective has no grad_output: its gradient is 0, not 1
        flow = self.scales.get("flow", zeros)
        track = self.scales.get("tracking") if self.track_done else None
        eng.backward_phase(flow, track, with_tracking=track is not None)
        # the packed (T, H, W) / (T - B, H, W) buffers, as the step's inputs
        out = [eng._g_depth.detach().view(self._params[0].shape)]
        if len(self._params) > 1:
            out.append(eng._g_w.detach().view(self._params[1].shape))
        # each model's own d loss / d focal (copies: the buffer is rewritten by the next step)
        out += [eng._g_focal[b].detach().clone().view(p.shape) for b, p in enumerate(self._focal_params)]
        return tuple(out)


def network_videos_step(engine, depths: Tensor, weights: Optional[Tensor], global_step: int,
                        training: bool = True, intrinsics=None):
    """One fused step of B networks' overfits, each network on its own video (a FusedOverfitter bound to a list of
    B network Models).  `depths` (T, H, W) and, with correspondence weights, `weights` (T - B, H, W) are the step's
    network outputs, packed along the frame axis (the caller concatenates its networks' outputs under autograd).
    Returns the (B,) weighted flow losses and tracking losses (zeros while the tracking loss is off), outputs of
    one root node: autograd calls its backward once, with one grad_output per video and loss, and it runs the
    backward half and hands d loss / d depths, d loss / d weights and each model's d loss / d focal length to
    autograd.  Video b gets what a one-video network-bound fused step on it gets, its gradients scaled by its own
    grad_output.

    Ground-truth intrinsics: the engine reads its videos' `batch.intrinsics` when it is built.  `intrinsics` (the
    list of B (1, F_b, 3, 3) tensors, or a (B, F, 3, 3) tensor for a tensor batch) is this step's K, copied into the
    step before its forward half without a host synchronisation, as the one-video surface reads `batch.intrinsics`
    on every step (a loader's new K, or the same tensors rewritten in place); None keeps the K the step last read."""
    eng = engine
    if not getattr(eng, "_net_videos", False):
        raise ValueError("flowmap_b200: network_videos_step needs a FusedOverfitter bound to a list of network Models")
    cfg = eng.cfg
    inputs = [depths.to(torch.float32).contiguous()]
    if cfg.use_correspondence_weights:
        if weights is None:
            raise ValueError("flowmap_b200: a step with correspondence weights needs `weights`")
        inputs.append(weights.to(torch.float32).contiguous())
    if intrinsics is not None:
        if not eng._gt:
            raise ValueError("flowmap_b200: `intrinsics` serves ground-truth K (cfg.intrinsics = 'ground_truth')")
        eng._write_k4(intrinsics)
    # the focal gradients handed to autograd are copies (_VideosStep.run_backward): no .grad aliases the buffer
    focal_params = [p for m in eng.models for p in m._fused_params(global_step, [])]
    tracking = cfg.use_tracking and global_step >= cfg.tracking_enable_after
    step = _VideosStep(eng, inputs, focal_params)
    flow = eng.forward_phase(global_step, training=training, depth=inputs[0].detach(),
                             weights=inputs[1].detach() if len(inputs) > 1 else None, tracking=tracking)
    track = eng.track_losses() if tracking else torch.zeros_like(flow)
    step.track_done = tracking
    token = _StepRoot.apply(step, *inputs, *focal_params)
    return (_LossNode.apply(token, step, "flow", flow),
            _LossNode.apply(token, step, "tracking", track))
