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
    """One loss of the step: value computed by the forward half, gradient deferred to the root."""

    @staticmethod
    def forward(ctx, token, step, which, value):
        ctx.step, ctx.which = step, which
        return value.clone()  # the engine's buffer is overwritten by the next step

    @staticmethod
    def backward(ctx, g):
        ctx.step.scales[ctx.which] = g.reshape(()).to(torch.float32).contiguous()
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
