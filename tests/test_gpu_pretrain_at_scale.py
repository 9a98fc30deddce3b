"""`-m gpu`: the fused pretraining step (pretrain.py, model_wrapper_pretrain.py on the packed layout of
fm_overfit_step_videos) at the reference's own batch -- 16 videos of 8 x 128 x 192, 8192 sweep points, 60
candidates, Procrustes on 1000 points (config/pretrain.yaml, config/frame_sampler/pretrain.yaml,
config/model/intrinsics/softmin.yaml) -- against the float64 oracle evaluated one video at a time under the
pooled mask sum (tests/pretrain_checks.py, pinned to the reference's Model + LossFlow by
tests/test_pretrain_golden.py).

The backbone is `FixedBackbone` below: its parameters are the batch's depths and correspondence weights, so
d loss / d depths and d loss / d weights are its parameter gradients.  Every video of the reference batch has
its own flow or depth regime and its own mask scale, so a normaliser, sweep pair, focal length or pair that
belongs to another video is a large error; launch_geometry asserts that the flow kernel's block ranges cross
videos on this device.  Tolerances: max(floor, 4 x the float32 oracle's own error) in every metric.

Also: the all-pixel window (W = 192) and dense (W = 190) Procrustes paths, no correspondence weights, l1 and
l2; videos and batches whose masks are all zero; a loader that rewrites the same Flows tensors in place, and
Flows that are non-contiguous views; the un-injected sweep sample; bf16 backbone outputs; five Adam steps of a
small network against its float64 twin on the CPU."""
import math
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F
from torch import nn

from conftest import max_abs, rel_l2
from flow_regime_checks import border_band, start_point
from pretrain_checks import pretrain_oracle
from test_gpu_packed_videos_at_scale import launch_geometry

pytestmark = pytest.mark.gpu

B_, F_, H_, W_ = 16, 8, 128, 192  # config/pretrain.yaml: batch 16, 8 frames, 128 x 192 crops
SWEEP, PROC = 8192, 1000
FLOW_KINDS = ("iid", "shift", "leave", "outliers", "zoom", "scene")
# every video its own regime: the six flow regimes, five depth regimes and a wide depth spread, then four
# of them again on other seeds
REGIMES = ("iid", "centre_far", "shift", "horizon", "leave", "scale_small", "outliers", "scale_large", "zoom",
           "corner_weights", "scene", "wide", "shift", "zoom", "outliers", "iid")
FLOORS = dict(loss=2e-5, share=2e-5, focal=2e-5, pose=1e-4, depth=1e-3, depth_frame=1e-3, depth_border=1e-3,
              weights=1e-3, weights_pair=1e-3)


@pytest.fixture(autouse=True)
def _threads():
    torch.set_num_threads(min(16, torch.get_num_threads()))


# ------------------------------------------------------------------------------------------------ inputs
@dataclass
class FixedCfg:
    name: str
    b: int


class FixedBackbone(nn.Module):
    """Returns its parameters: the batch's depths (B, F, H, W) and correspondence weights (B, F-1, H, W)."""

    def __init__(self, cfg, num_frames, image_shape):
        super().__init__()
        self.cfg, self.calls = cfg, 0
        self.depths = nn.Parameter(torch.ones(cfg.b, num_frames, *image_shape))
        self.weights = nn.Parameter(torch.full((cfg.b, num_frames - 1, *image_shape), 0.5))

    def forward(self, batch, flows):
        from flowmap_b200.types import BackboneOutput
        self.calls += 1
        return BackboneOutput(self.depths, self.weights)


def _register():
    from flowmap_b200.model import BACKBONES
    BACKBONES["test_fixed"] = FixedBackbone


def _regime_video(kind, f, h, w, seed):
    """Float64 depth (F, H, W), weights (F-1, H, W) and the four flow tensors of one video in a flow or depth
    regime (oracle.flow_regime / depth_regime) at a start point (flow_regime_checks.start_point); `wide`:
    smooth depths from tens to thousands."""
    from oracle import flowmap_oracle as O
    g = torch.Generator().manual_seed(seed + 2)
    if kind in O.DEPTH_REGIMES:
        depth, fl, _, logits = O.depth_regime(kind, f, h, w, seed=seed)
    else:
        depth, fl, _, _ = O.flow_regime("iid" if kind == "wide" else kind, f, h, w, seed=seed)
        logits = 0.01 * torch.randn(1, f - 1, h, w, generator=g, dtype=torch.float64)
        if kind == "wide":
            low = torch.rand(f, 1, 4, 6, generator=g, dtype=torch.float64)
            depth = 10.0 ** (1.3 + 2.2 * F.interpolate(low, (h, w), mode="bilinear", align_corners=False))
            depth = depth.reshape(1, f, h, w)
    assert bool(torch.isfinite(depth).all()), (kind, seed)
    depth, _ = start_point(depth, 1.0, seed=seed + 1)
    weights = torch.sigmoid(100.0 * logits)
    return depth[0], weights[0], [t[0] for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)]


def _inputs(kinds, f=F_, h=H_, w=W_, seed=0, mask_scales=None):
    """(depths, weights, [fwd, bwd, fmask, bmask]) float64 (B, ...) tensors; video v's masks x mask_scales[v]
    (default 0.85 ** v: every video its own mask sum)."""
    per = [_regime_video(k, f, h, w, seed + 17 * v) for v, k in enumerate(kinds)]
    scales = mask_scales if mask_scales is not None else [0.85 ** v for v in range(len(kinds))]
    flows = [torch.stack([p[2][i] for p in per]) for i in range(4)]
    s = torch.tensor(scales, dtype=torch.float64)[:, None, None, None]
    flows[2], flows[3] = flows[2] * s, flows[3] * s
    return torch.stack([p[0] for p in per]), torch.stack([p[1] for p in per]), flows


def _flows(fl, dev):
    from flowmap_b200.types import Flows
    return Flows(*(t.to(dev, torch.float32).contiguous() for t in fl))


def _model(b, f=F_, h=H_, w=W_, use_weights=True, points=PROC, mapping="huber", inject=True):
    from flowmap_b200.loss import LossFlowCfg, MappingHuberCfg, MappingL1Cfg, MappingL2Cfg, get_losses
    from flowmap_b200.model import ExtrinsicsProcrustesCfg, IntrinsicsSoftminCfg, Model, ModelCfg
    from flowmap_b200.types import Batch
    _register()
    dev = torch.device("cuda:0")
    icfg = IntrinsicsSoftminCfg("softmin", SWEEP, 0.5, 2.0, 60, None)
    model = Model(ModelCfg(FixedCfg("test_fixed", b), icfg, ExtrinsicsProcrustesCfg("procrustes", points, False),
                           use_weights), f, (h, w)).to(dev)
    if inject:
        n = min(SWEEP, h * w)
        model.intrinsics.injected_indices = torch.randperm(h * w, generator=torch.Generator().manual_seed(3))[:n].to(dev)
    m = {"huber": MappingHuberCfg("huber", 0.01), "l1": MappingL1Cfg("l1"), "l2": MappingL2Cfg("l2")}[mapping]
    losses = get_losses([LossFlowCfg(0, 1000.0, "flow", m)])
    batch = Batch(torch.zeros(b, f, 3, h, w, device=dev), torch.arange(f, device=dev)[None].expand(b, f),
                  ["s"] * b, ["d"] * b)
    return model, losses, batch


def _load(model, depths, weights):
    with torch.no_grad():
        model.backbone.depths.copy_(depths.to(torch.float32))
        model.backbone.weights.copy_(weights.to(torch.float32))


def _step(model, losses, batch, flows, fused=True, scale=None, step=0):
    """One pretraining step without the optimiser.  Returns the loss, the (B,) per-video shares of the fused
    step (None per-op), each video's focal length (fx normalised as the reference's), the extrinsics and the
    backbone's parameter gradients (d loss / d depths, d loss / d weights or None)."""
    from flowmap_b200.model import Model
    Model.fused_enabled = fused
    try:
        model.zero_grad(set_to_none=True)
        out = model(batch, flows, step)
        total = sum(l.forward(batch, flows, None, out, step) for l in losses)
        (total if scale is None else total * scale).backward()
        fused_step = out.__dict__.get("_fused")
        is_fused = type(out).__name__ == "LazyModelOutput" and fused_step.flow_done and not fused_step.dead
        assert is_fused == fused, (fused, is_fused)
        share = fused_step.engine._loss.detach().double().cpu().clone() if fused else None
        h, w = batch.videos.shape[-2:]
        k4 = out.k4.detach().double().cpu()
        bb = model.backbone
        return dict(loss=float(total.detach()), share=share, focal=k4[:, 0, 0] * w / math.sqrt(h * w),
                    ext=out.extrinsics.detach().double().cpu(), g_depth=bb.depths.grad.detach().double().cpu(),
                    g_w=None if bb.weights.grad is None else bb.weights.grad.detach().double().cpu())
    finally:
        Model.fused_enabled = True


def _oracles(model, depths, weights, fl, sweep_idx=None, mapping="huber"):
    """{64: float64 oracle, 32: float32 oracle} of the step, with the model's sweep sample and point set."""
    h, w = depths.shape[-2:]
    from flowmap_b200.types import Flows
    flows = Flows(*fl)
    if sweep_idx is None:
        sweep_idx = model.intrinsics.injected_indices
    pidx = model.extrinsics.select_indices(h, w, "cpu")
    cand = model.intrinsics.focal_length_candidates.detach().double().cpu()
    uw = model.cfg.use_correspondence_weights
    return {bits: pretrain_oracle(depths, weights, flows, sweep_idx, cand, pidx, mapping, dt, uw)
            for bits, dt in ((64, torch.float64), (32, torch.float32))}


# ------------------------------------------------------------------------------------------------ metrics
def _errors(got, ref, videos):
    """Errors of a step against an oracle result, per video: the loss (relative), each video's share of the
    (B,) loss buffer (relative to the batch loss), focal length (relative), extrinsics (max abs over the
    video, over the larger of 1 and its largest translation), and the depth / weight gradients (relative L2
    over the video, per frame / pair and on the border band)."""
    h, w = ref["g_depth"].shape[-2:]
    band = border_band(h, w)
    e = dict(loss=abs(got["loss"] - ref["loss"]) / max(abs(ref["loss"]), 1e-30))
    per = {k: [] for k in ("share", "focal", "pose", "depth", "depth_frame", "depth_border", "weights",
                           "weights_pair")}
    for v in videos:
        if got["share"] is not None:
            per["share"].append(abs(float(got["share"][v]) - float(ref["share"][v])) / max(abs(ref["loss"]), 1e-30))
        per["focal"].append(abs(float(got["focal"][v]) - float(ref["focal"][v])) / float(ref["focal"][v]))
        re = ref["ext"][v]
        per["pose"].append(max_abs(got["ext"][v], re) / max(1.0, float(re[:, :3, 3].abs().max())))
        gd, rd = got["g_depth"][v], ref["g_depth"][v]
        per["depth"].append(rel_l2(gd, rd))
        per["depth_frame"].append(max(rel_l2(gd[i], rd[i]) for i in range(rd.shape[0])))
        per["depth_border"].append(rel_l2(gd[:, band], rd[:, band]))
        if ref["g_w"] is not None:
            gw, rw = got["g_w"][v], ref["g_w"][v]
            per["weights"].append(rel_l2(gw, rw))
            per["weights_pair"].append(max(rel_l2(gw[i], rw[i]) for i in range(rw.shape[0])))
    e.update({k: v for k, v in per.items() if v})
    return e


def _check(label, got, oracle, videos=None, floors=FLOORS):
    """Every metric of _errors within max(floor, 4 x the float32 oracle's own error); prints both."""
    videos = list(range(oracle[64]["g_depth"].shape[0])) if videos is None else videos
    errs, noise = _errors(got, oracle[64], videos), _errors(oracle[32], oracle[64], videos)
    fmt = lambda x: [f"{y:.1e}" for y in x] if isinstance(x, list) else f"{x:.1e}"  # noqa: E731
    for key in errs:
        print(f"{label} {key}: error {fmt(errs[key])} | float32 oracle {fmt(noise[key])}")
    for key, got_e in errs.items():
        for i, (a, n) in enumerate(zip(got_e, noise[key]) if isinstance(got_e, list) else [(got_e, noise[key])]):
            assert a <= max(floors[key], 4.0 * n), (label, key, videos[i] if isinstance(got_e, list) else None, a, n)


def _device_geometry(frames, h, w):
    p = torch.cuda.get_device_properties(0)
    geo = launch_geometry(frames, h, w, p.multi_processor_count, p.L2_cache_size)
    print(f"{len(frames)} x {frames[0]} x {h} x {w} at {p.multi_processor_count} SMs: (rounds, multi, cross)", geo)
    return geo


# ------------------------------------------------------------------------------------ the reference's batch
@pytest.fixture(scope="module")
def reference_batch():
    """The reference batch's inputs and both oracle results."""
    depths, weights, fl = _inputs(REGIMES)
    model, _, _ = _model(B_)
    return depths, weights, fl, _oracles(model, depths, weights, fl)


def test_reference_batch_against_the_float64_oracle(reference_batch):
    """B = 16, F = 8, 128 x 192, 8192 sweep points, 60 candidates, 1000 Procrustes points, Huber: the loss,
    each video's share, focal length, extrinsics and input gradients against the float64 oracle, with the flow
    kernel's block ranges crossing videos."""
    depths, weights, fl, oracle = reference_batch
    assert _device_geometry((F_,) * B_, H_, W_)["flow"][2] > 0
    m = [float(fl[2][v].sum() + fl[3][v].sum()) for v in range(B_)]
    assert len(set(round(x) for x in m)) == B_, m
    model, losses, batch = _model(B_)
    _load(model, depths, weights)
    got = _step(model, losses, batch, _flows(fl, "cuda:0"))
    assert abs(float(got["share"].sum()) - got["loss"]) <= 1e-5 * abs(got["loss"])
    assert model.backbone.calls == 1
    _check("reference batch", got, oracle)


@pytest.mark.parametrize("w", [W_, W_ - 2], ids=["window-192", "dense-190"])
def test_all_pixel_procrustes_paths(w):
    """Procrustes on every pixel at B = 16: the scatter window (W % 4 == 0) and the dense backward (W = 190,
    where the moment, dense and flow kernels' ranges all cross videos)."""
    geo = _device_geometry((F_,) * B_, H_, w)
    assert geo["flow"][2] > 0
    if w % 4:
        assert geo["moments"][2] > 0 and geo["dense"][2] > 0
    depths, weights, fl = _inputs(REGIMES, w=w, seed=100)
    model, losses, batch = _model(B_, w=w, points=None)
    _load(model, depths, weights)
    got = _step(model, losses, batch, _flows(fl, "cuda:0"))
    _check(f"all pixels W={w}", got, _oracles(model, depths, weights, fl))


SUBSET = ("scene", "shift", "horizon", "wide", "outliers", "scale_large")
# without weights: no regime whose far band only the weights keep out of the fit (horizon, centre_far,
# corner_weights), where the Procrustes fit is ill-posed even in float64
SUBSET_NO_WEIGHTS = ("scene", "shift", "zoom", "wide", "outliers", "scale_large")


@pytest.mark.parametrize("mapping,use_weights", [("huber", False), ("l1", True), ("l2", True)])
def test_weights_off_and_other_mappings(mapping, use_weights):
    """Six of the regimes at 128 x 192: without correspondence weights (ones, no weight gradient), and with
    the l1 and l2 mappings."""
    depths, weights, fl = _inputs(SUBSET if use_weights else SUBSET_NO_WEIGHTS, seed=200)
    model, losses, batch = _model(depths.shape[0], use_weights=use_weights, mapping=mapping)
    _load(model, depths, weights)
    got = _step(model, losses, batch, _flows(fl, "cuda:0"))
    assert (got["g_w"] is None) == (not use_weights)
    _check(f"{mapping} weights={use_weights}", got, _oracles(model, depths, weights, fl, mapping=mapping))


# ----------------------------------------------------------------------------------------------- mask edges
def test_a_video_without_valid_flow():
    """One video's masks all zero in a batch whose pooled sum is not: its depth and weight gradients are
    exactly zero, its share is zero, and the other videos match the oracle under the pooled sum without it."""
    kinds = ("iid", "shift", "scene", "zoom", "outliers", "leave")
    zero = 2
    depths, weights, fl = _inputs(kinds, seed=300, mask_scales=[1.0, 0.5, 0.0, 0.3, 0.8, 0.4])
    assert float(fl[2][zero].abs().sum() + fl[3][zero].abs().sum()) == 0.0
    model, losses, batch = _model(len(kinds))
    _load(model, depths, weights)
    got = _step(model, losses, batch, _flows(fl, "cuda:0"))
    assert float(got["share"][zero]) == 0.0
    assert bool((got["g_depth"][zero] == 0).all()) and bool((got["g_w"][zero] == 0).all())
    for t in (got["g_depth"], got["g_w"], got["share"], got["ext"]):
        assert bool(torch.isfinite(t).all())
    others = [v for v in range(len(kinds)) if v != zero]
    _check("zero-mask video", got, _oracles(model, depths, weights, fl), videos=others)


def test_a_batch_without_valid_flow():
    """Every mask zero ("valid_sum or 1"): loss 0, every gradient 0, nothing non-finite, on the fused and the
    per-op path alike."""
    kinds = ("iid", "shift", "scene", "zoom")
    depths, weights, fl = _inputs(kinds, seed=400, mask_scales=[0.0] * 4)
    for fused in (True, False):
        model, losses, batch = _model(len(kinds))
        _load(model, depths, weights)
        got = _step(model, losses, batch, _flows(fl, "cuda:0"), fused=fused)
        assert got["loss"] == 0.0, (fused, got["loss"])
        assert bool((got["g_depth"] == 0).all()) and bool((got["g_w"] == 0).all()), fused
        assert bool(torch.isfinite(got["ext"]).all()) and bool(torch.isfinite(got["focal"]).all()), fused
        if fused:
            assert bool((got["share"] == 0).all())


# -------------------------------------------------------------------------------------------- loader patterns
LOADER = ("zoom", "iid", "scene", "horizon")


def test_loader_rewrites_the_same_flows_tensors():
    """Three steps in which a loader copy_'s new flows and masks (and new mask scales) into the same Flows
    tensors, each step with its own grad_output scale: every step matches the oracle on its new content,
    the pooled normaliser and the scale included, and the engine is built once."""
    model, losses, batch = _model(len(LOADER))
    flows, engines = None, set()
    for s, scale in enumerate((1.0, 0.5, 2.0)):
        depths, weights, fl = _inputs(LOADER[s:] + LOADER[:s], seed=500 + 10 * s,
                                      mask_scales=[0.3 + 0.5 * ((v + s) % 4) for v in range(4)])
        if flows is None:
            flows = _flows(fl, "cuda:0")
        else:
            for dst, src in zip((flows.forward, flows.backward, flows.forward_mask, flows.backward_mask), fl):
                dst.copy_(src)
        _load(model, depths, weights)
        got = _step(model, losses, batch, flows, scale=scale)
        engines.add(id(model._engine))
        got = {**got, "g_depth": got["g_depth"] / scale, "g_w": got["g_w"] / scale}
        _check(f"loader step {s} (scale {scale})", got, _oracles(model, depths, weights, fl))
    assert len(engines) == 1


def test_non_contiguous_flows_views():
    """Flows passed as non-contiguous views of larger tensors (a loader's padded buffers): the step matches the
    oracle, and again after the loader rewrites the buffers behind the same views."""
    from flowmap_b200.types import Flows
    b, f, h, w = len(LOADER), F_, H_, W_
    model, losses, batch = _model(b)
    dev = torch.device("cuda:0")
    big = [torch.zeros(b, f, h + 3, w + 5, 2, device=dev), torch.zeros(b, f, h + 3, w + 5, 2, device=dev),
           torch.zeros(b, f, h + 3, w + 5, device=dev), torch.zeros(b, f, h + 3, w + 5, device=dev)]
    views = Flows(*(t[:, 1:, 2:2 + h, 3:3 + w] for t in big))
    assert not any(t.is_contiguous() for t in (views.forward, views.backward, views.forward_mask, views.backward_mask))
    for s in range(2):
        depths, weights, fl = _inputs(LOADER[::-1] if s else LOADER, seed=600 + 10 * s,
                                      mask_scales=[1.0, 0.2, 0.6, 0.45] if s else None)
        for t, src in zip(big, fl):
            t[:, 1:, 2:2 + h, 3:3 + w].copy_(src)
        _load(model, depths, weights)
        got = _step(model, losses, batch, views)
        _check(f"non-contiguous views, step {s}", got, _oracles(model, depths, weights, fl))


# ------------------------------------------------------------------------------------ un-injected sweep sample
def test_un_injected_sweep_sample(monkeypatch):
    """injected_indices None, as in real pretraining: each step draws one sample of min(8192, H W) distinct,
    in-range indices for all videos, a new one every step, and the step matches the oracle on that sample."""
    from flowmap_b200 import ops
    drawn = []
    real = ops.random_subset

    def record(num_items, n, device, seed=None):
        out = real(num_items, n, device, seed)
        drawn.append((num_items, out.detach().cpu().clone()))
        return out

    monkeypatch.setattr(ops, "random_subset", record)
    kinds = ("outliers", "scene", "wide", "shift")
    model, losses, batch = _model(len(kinds), inject=False)
    assert model.intrinsics.injected_indices is None
    depths, weights, fl = _inputs(kinds, seed=700)
    _load(model, depths, weights)
    flows = _flows(fl, "cuda:0")
    for s in range(2):
        got = _step(model, losses, batch, flows, step=s)
        assert len(drawn) == s + 1, len(drawn)  # one sample per step, shared by every video
    for num_items, idx in drawn:
        assert num_items == H_ * W_ and idx.numel() == min(SWEEP, H_ * W_)
        assert idx.unique().numel() == idx.numel() and int(idx.min()) >= 0 and int(idx.max()) < H_ * W_
    assert not torch.equal(drawn[0][1], drawn[1][1])
    _check("un-injected sample", got, _oracles(model, depths, weights, fl, sweep_idx=drawn[-1][1]))


# ---------------------------------------------------------------------------------- bf16 backbone outputs
def test_bf16_backbone_outputs():
    """A network under bf16 autocast (StandInCfg(bf16=True)) at B = 4, 128 x 192: the fused step against the
    oracle on the upcast outputs; the gradients reach the network's bf16 outputs as bf16 (rounding floor 1e-2)."""
    from test_gpu_pretrain_fused import _setup
    model, losses, batch, flows = _setup(4, f=F_, h=H_, w=W_, bf16=True)
    from flowmap_b200.model import Model
    model.zero_grad(set_to_none=True)
    out = model(batch, flows, 0)
    depths, weights = out.depths, out.backward_correspondence_weights
    assert depths.dtype == weights.dtype == torch.bfloat16
    depths.retain_grad()
    weights.retain_grad()
    total = sum(l.forward(batch, flows, None, out, 0) for l in losses)
    total.backward()
    fused = out.__dict__["_fused"]
    assert Model.fused_enabled and fused.flow_done and not fused.dead and fused.engine.B == 4
    assert depths.grad.dtype == weights.grad.dtype == torch.bfloat16
    assert all(p.grad is not None for p in model.backbone.features.parameters())
    h, w = H_, W_
    k4 = out.k4.detach().double().cpu()
    got = dict(loss=float(total.detach()), share=fused.engine._loss.detach().double().cpu(),
               focal=k4[:, 0, 0] * w / math.sqrt(h * w), ext=out.extrinsics.detach().double().cpu(),
               g_depth=depths.grad.double().cpu(), g_w=weights.grad.double().cpu())
    d64, w64 = depths.detach().double().cpu(), weights.detach().double().cpu()
    fl = [t.detach().double().cpu() for t in (flows.forward, flows.backward, flows.forward_mask, flows.backward_mask)]
    floors = {**FLOORS, **{k: 1e-2 for k in ("depth", "depth_frame", "depth_border", "weights", "weights_pair")}}
    _check("bf16 outputs", got, _oracles(model, d64, w64, fl), floors=floors)


# ------------------------------------------------------------------------------------- a short pretraining run
class ParamBackbone(nn.Module):
    """tools/pretrain_step.py's `param` backbone: depth = 1e3 / (softplus(p + 2 v) + 0.1) and weights =
    sigmoid(100 q + v' - 0.5) from per-pixel parameters shared by the batch and the videos' first / second
    channels.  Runs on any device and dtype (its float64 twin runs on the CPU)."""

    def __init__(self, cfg, num_frames, image_shape):
        super().__init__()
        g = torch.Generator().manual_seed(5)
        self.p = nn.Parameter(torch.full((num_frames, *image_shape), 1.0) + 0.5 * torch.randn(num_frames, *image_shape, generator=g))
        self.q = nn.Parameter(0.01 * torch.randn(num_frames - 1, *image_shape, generator=g))

    def forward(self, batch, flows):
        from flowmap_b200.types import BackboneOutput
        v = batch.videos.to(self.p.dtype)
        return BackboneOutput(1e3 / (F.softplus(self.p + 2.0 * v[:, :, 0]) + 0.1),
                              (100.0 * self.q + v[:, 1:, 1] - 0.5).sigmoid())


def _twin_run(start, data, dtype, steps):
    """The oracle's pretraining run on the CPU at `dtype`: the backbone's outputs -> pretrain_oracle ->
    their gradients carried into p and q -> torch.optim.Adam (lr 5e-5).  Per-step losses and focal lengths,
    and the final parameters."""
    bb = ParamBackbone(None, F_, (H_, W_)).to(dtype)
    with torch.no_grad():
        for n, p in bb.named_parameters():
            p.copy_(start[f"backbone.{n}"].to(dtype))
    opt = torch.optim.Adam(bb.parameters(), lr=5e-5)
    losses, focals = [], []
    for s in range(steps):
        videos, fl, sweep = data[s]
        from flowmap_b200.types import Batch
        batch = Batch(videos.to(dtype), None, None, None)
        out = bb(batch, None)
        cand = torch.linspace(0.5, 2.0, 60).double()  # the model's float32 candidates
        from flowmap_b200.types import Flows
        r = pretrain_oracle(out.depths, out.weights, Flows(*fl), sweep, cand,
                            torch.linspace(0, H_ * W_ - 1, PROC, dtype=torch.int64), dtype=dtype)
        opt.zero_grad()
        torch.autograd.backward([out.depths, out.weights], [r["g_depth"].to(dtype), r["g_w"].to(dtype)])
        opt.step()
        losses.append(r["loss"])
        focals.append(r["focal"])
    return losses, torch.stack(focals), {f"backbone.{n}": p.detach().double() for n, p in bb.named_parameters()}


def test_five_adam_steps_against_a_float64_twin():
    """Five torch.optim.Adam steps (lr 5e-5) of the `param` backbone at B = 4, 8 x 128 x 192, each on a new
    batch with new Flows: per-step losses, per-step focal lengths of every video and the final parameter
    deltas against the float64 twin's run, within max(floor, 4 x the float32 twin's own error).  Each step's
    videos take their flows from the flow regimes: the depth regimes' ill-conditioned fits (a far band or corner
    that only the weights keep out) leave weight gradients whose float32 error Adam's normalised update turns
    into parameter deltas of any direction."""
    from flowmap_b200.model import BACKBONES, ExtrinsicsProcrustesCfg, IntrinsicsSoftminCfg, Model, ModelCfg
    from flowmap_b200.loss import LossFlowCfg, MappingHuberCfg, get_losses
    from flowmap_b200.types import Batch
    BACKBONES["test_param"] = ParamBackbone
    b, steps, dev = 4, 5, torch.device("cuda:0")
    model = Model(ModelCfg(FixedCfg("test_param", b), IntrinsicsSoftminCfg("softmin", SWEEP, 0.5, 2.0, 60, None),
                           ExtrinsicsProcrustesCfg("procrustes", PROC, False), True), F_, (H_, W_)).to(dev)
    losses = get_losses([LossFlowCfg(0, 1000.0, "flow", MappingHuberCfg("huber", 0.01))])
    start = {n: p.detach().double().cpu().clone() for n, p in model.named_parameters()}
    data = []
    for s in range(steps):
        g = torch.Generator().manual_seed(800 + s)
        low = torch.rand(b * F_, 3, 8, 12, generator=g, dtype=torch.float64)
        videos = F.interpolate(low, (H_, W_), mode="bilinear", align_corners=False).reshape(b, F_, 3, H_, W_)
        videos = videos.float().double()
        kinds = [FLOW_KINDS[(4 * s + v) % len(FLOW_KINDS)] for v in range(b)]
        _, _, fl = _inputs(kinds, seed=900 + 10 * s)
        fl = [t.float().double() for t in fl]
        sweep = torch.randperm(H_ * W_, generator=torch.Generator().manual_seed(50 + s))[:SWEEP]
        data.append((videos, fl, sweep))
    opt = torch.optim.Adam(model.parameters(), lr=5e-5)
    got_loss, got_focal = [], []
    for s in range(steps):
        videos, fl, sweep = data[s]
        model.intrinsics.injected_indices = sweep.to(dev)
        batch = Batch(videos.to(dev, torch.float32), torch.arange(F_, device=dev)[None].expand(b, F_), ["s"] * b,
                      ["d"] * b)
        flows = _flows(fl, dev)
        opt.zero_grad(set_to_none=True)
        out = model(batch, flows, s)
        total = sum(l.forward(batch, flows, None, out, s) for l in losses)
        total.backward()
        assert out.__dict__["_fused"].flow_done and not out.__dict__["_fused"].dead
        opt.step()
        got_loss.append(float(total.detach()))
        got_focal.append(out.k4.detach().double().cpu()[:, 0, 0] * W_ / math.sqrt(H_ * W_))
    got_focal = torch.stack(got_focal)
    l64, f64, p64 = _twin_run(start, data, torch.float64, steps)
    l32, f32, p32 = _twin_run(start, data, torch.float32, steps)
    for s in range(steps):
        err, noise = abs(got_loss[s] - l64[s]) / abs(l64[s]), abs(l32[s] - l64[s]) / abs(l64[s])
        ferr = (got_focal[s] - f64[s]).abs().max().item() / f64[s].abs().min().item()
        fnoise = (f32[s] - f64[s]).abs().max().item() / f64[s].abs().min().item()
        print(f"Adam step {s}: loss {err:.1e} (float32 twin {noise:.1e}), focal {ferr:.1e} (float32 twin {fnoise:.1e})")
        assert err <= max(2e-5, 4 * noise), (s, err, noise)
        # Adam moves a parameter whose gradient is near zero by about lr either way, so the runs' parameters
        # part by O(lr) whatever the precision, and the focal length with them: a floor of 1e-4
        assert ferr <= max(1e-4, 4 * fnoise), (s, ferr, fnoise)
    for n, p in model.named_parameters():
        d_got, d64, d32 = p.detach().double().cpu() - start[n], p64[n] - start[n], p32[n] - start[n]
        err, noise = rel_l2(d_got, d64), rel_l2(d32, d64)
        print(f"Adam parameter delta {n}: {err:.1e} (float32 twin {noise:.1e})")
        assert float(d64.norm()) > 0
        # floor 2e-2: where a gradient is near zero, Adam's normalised step follows its rounding error, and the
        # kernels' fixed-point window sums round differently from any CPU float32 run (measured on an H100:
        # 1.3e-2 on q against 5.8e-4 for the float32 twin; fused and per-op updates differ by up to 1e-2)
        assert err <= max(2e-2, 4 * noise), (n, err, noise)
