"""`-m gpu`: a network backbone (the reference's default overfit: MiDaS depths and a per-pixel MLP for the
correspondence weights) on the fused halves (flowmap_b200.fused).  The backbone stays in torch and runs once
per step; the fused step takes its depths and weights as inputs and hands d loss / d depths and
d loss / d weights back to autograd, which carries them into the network.

No pretrained weights are needed: the stand-in backbones below are small CNNs with the reference
backbone's output mappings and weight head, registered in flowmap_b200.model.BACKBONES under a test name.
Checked: fused == per-op (losses and the gradient of every network parameter and of the focal length),
the fused depth / weight gradients against the float64 oracle, a short Adam run across the tracking
switch-on and the softmin -> regressed hand-over, one backbone call per step, grad_output scales and
kept gradients, and the fall-backs (bf16 autocast output, B = 2, CPU output)."""
import copy
from dataclasses import dataclass
from typing import Optional

import pytest
import torch
import torch.nn.functional as F
from torch import nn

from conftest import rel_l2

pytestmark = pytest.mark.gpu

F_, H_, W_ = 6, 40, 64


@dataclass
class StandInCfg:
    name: str
    weight_sensitivity: Optional[float]  # None: MLP weight head; else sigmoid(s * learned logits)
    mapping: str  # "original": 1e3 / (x + 0.1); "exp": exp(x / 1000) + 0.01
    bf16: bool = False  # run the network under bf16 autocast and return its bf16 outputs
    cast_output: bool = False  # return float32 outputs (the per-op twin of bf16)
    device: Optional[str] = None  # move the outputs there (a CPU output)
    spread: tuple = (0.5, 1.0)  # (network, video) terms of the mapped value: depths of about 400 to 2200


# depths from tens to thousands: a problem whose float32 gradients carry ~1e-2 of rounding error with these
# random flows (the float32 oracle's own error), so it is compared against the float64 oracle only
WIDE = (3.0, 3.5)


class StandInBackbone(nn.Module):
    """A tiny CNN in the shape of BackboneMidas: per-frame features, a one-channel depth head through the
    configured mapping, and correspondence weights from an MLP on the features of the earlier frame sampled
    at the backward flow beside those of the later frame, ending in sigmoid().clip(min=1e-4).  The depth
    head also sees the video's first channel, so that the depths span a range set by `spread` (up to tens to
    thousands), and the weight logits its second, so that a good share of the weights sit at the 1e-4 floor."""

    def __init__(self, cfg: StandInCfg, num_frames, image_shape):
        super().__init__()
        self.cfg, self.calls = cfg, 0
        c = 8
        g = torch.Generator().manual_seed(11)
        self.features = nn.Sequential(nn.Conv2d(3, c, 3, padding=1), nn.ReLU(), nn.Conv2d(c, c, 3, padding=1))
        self.depth_head = nn.Conv2d(c, 1, 1)
        if cfg.weight_sensitivity is None:
            self.head = nn.Sequential(nn.Linear(2 * c, 16), nn.ReLU(), nn.Linear(16, 8), nn.ReLU(), nn.Linear(8, 1))
        else:
            self.weights = nn.Parameter(0.01 * torch.randn(num_frames - 1, *image_shape, generator=g))

    def forward(self, batch, flows):
        self.calls += 1
        b, f, _, h, w = batch.videos.shape
        v = batch.videos.reshape(b * f, 3, h, w)
        a, s = self.cfg.spread
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=self.cfg.bf16):
            feat = self.features(v)
            u = self.depth_head(feat)
            logits = None
            if self.cfg.weight_sensitivity is None:
                fe = feat.reshape(b, f, -1, h, w)
                ys, xs = torch.meshgrid(torch.arange(h, device=v.device), torch.arange(w, device=v.device), indexing="ij")
                xy = torch.stack(((xs + 0.5) / w, (ys + 0.5) / h), -1).to(flows.backward.dtype)
                grid = (xy + flows.backward) * 2 - 1  # (b, f-1, h, w, 2)
                earlier = F.grid_sample(fe[:, :-1].reshape(b * (f - 1), -1, h, w), grid.reshape(b * (f - 1), h, w, 2).to(fe.dtype),
                                        mode="bilinear", padding_mode="zeros", align_corners=False)
                pair = torch.cat((earlier.reshape(b, f - 1, -1, h, w), fe[:, 1:]), 2).permute(0, 1, 3, 4, 2)
                logits = self.head(pair)[..., 0]
        vu = v.to(u.dtype)  # bf16 under autocast: the mappings in the network's dtype
        x = a * torch.tanh(u) + s * (2.0 * vu[:, :1] - 1.0)
        if self.cfg.mapping == "original":
            depths = 1e3 / (torch.exp(x) + 0.1)
        else:
            depths = torch.exp(1000.0 * x / 1000.0) + 0.01
        depths = depths.reshape(b, f, h, w)
        if logits is not None:
            # the later frame's second channel spreads the logits, so that a good share sits at the floor
            weights = (logits + 24.0 * vu.reshape(b, f, 3, h, w)[:, 1:, 1] - 16.0).sigmoid().clip(min=1e-4)
        else:
            weights = (self.cfg.weight_sensitivity * self.weights).sigmoid()[None].expand(b, -1, -1, -1)
        from flowmap_b200.types import BackboneOutput
        if self.cfg.cast_output:
            depths, weights = depths.float(), weights.float()
        if self.cfg.device is not None:
            depths, weights = depths.to(self.cfg.device), weights.to(self.cfg.device)
        return BackboneOutput(depths, weights)


def _register():
    from flowmap_b200.model import BACKBONES
    BACKBONES["test_stand_in"] = StandInBackbone


BACKBONE_KINDS = {
    "mlp_original": StandInCfg("test_stand_in", None, "original"),
    "mlp_exp": StandInCfg("test_stand_in", None, "exp"),
    "logits": StandInCfg("test_stand_in", 100.0, "original"),
}


def _video(f, h, w, seed, b=1):
    """Smooth random videos: depths and features that vary over the frame but not from pixel to pixel."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(b * f, 3, max(2, h // 8), max(2, w // 8), generator=g)
    return F.interpolate(low, (h, w), mode="bilinear", align_corners=False).reshape(b, f, 3, h, w)


def _setup(kind="mlp_original", intrinsics="regressed", tracking=False, use_weights=True, points=None,
           f=F_, h=H_, w=W_, seed=0, regression=None, tracking_after=0, b=1, **backbone):
    import bench
    from flowmap_b200.loss import LossFlowCfg, LossTrackingCfg, MappingHuberCfg, get_losses
    from flowmap_b200.model import (ExtrinsicsProcrustesCfg, IntrinsicsRegressedCfg, IntrinsicsSoftminCfg, Model,
                                    ModelCfg, RegressionCfg)
    from flowmap_b200.types import Batch, Flows, Tracks
    _register()
    dev = torch.device("cuda:0")
    torch.manual_seed(seed)
    if intrinsics == "regressed":
        icfg = IntrinsicsRegressedCfg("regressed", 0.85)
    else:
        reg = None if regression is None else RegressionCfg(*regression)
        icfg = IntrinsicsSoftminCfg("softmin", 500, 0.5, 2.0, 60, reg)
    bcfg = StandInCfg(**{**BACKBONE_KINDS[kind].__dict__, **backbone})
    mcfg = ModelCfg(bcfg, icfg, ExtrinsicsProcrustesCfg("procrustes", points, False), use_weights)
    model = Model(mcfg, f, (h, w)).to(dev)
    if intrinsics == "softmin":
        model.intrinsics.injected_indices = torch.randperm(h * w, generator=torch.Generator().manual_seed(3))[:500].to(dev)
    huber = MappingHuberCfg("huber", 0.01)
    lcfgs = [LossFlowCfg(0, 1000.0, "flow", huber)]
    if tracking:
        lcfgs.append(LossTrackingCfg(tracking_after, 100.0, "tracking", huber))
    losses = get_losses(lcfgs)
    inp = bench.synthetic_inputs(f, h, w, seed=seed)
    batch = Batch(_video(f, h, w, seed, b).to(dev), torch.arange(f, device=dev)[None].expand(b, f), ["s"] * b, ["d"] * b)
    flows = Flows(*(inp[k].expand(b, *inp[k].shape[1:]).contiguous().to(dev) for k in ("fwd", "bwd", "fmask", "bmask")))
    tracks = None
    if tracking:
        tracks = [Tracks(xy.to(dev), vis.to(dev), s)
                  for xy, vis, s in bench.synthetic_track_arrays(f, n_points=64, interval=3, radius=2, seed=seed)]
    return model, losses, batch, flows, tracks


def _step(model, losses, batch, flows, tracks, fused, scale=None, step=0, zero=True):
    from flowmap_b200.model import Model
    Model.fused_enabled = fused
    try:
        if zero:
            model.zero_grad(set_to_none=True)
        out = model(batch, flows, step)
        parts = [l.forward(batch, flows, tracks, out, step) for l in losses]
        total = sum(parts)
        (total if scale is None else total * scale).backward()
        grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
        return [float(p.detach()) for p in parts], grads, out
    finally:
        Model.fused_enabled = True


def _assert_close(pa, ga, pb, gb, softmin, grad_tol=None):
    """test_gpu_dropin_fused.py's tolerances: losses 1e-6, focal 5e-4, the rest 2e-5 (2e-4 in the softmin
    stage, where d loss / d focal feeds the sweep's backward)."""
    for a, b in zip(pa, pb):
        assert abs(a - b) <= 1e-6 * abs(a), (pa, pb)
    assert set(ga) == set(gb), (sorted(ga), sorted(gb))
    for name in ga:
        tol = 5e-4 if "focal" in name else (grad_tol or (2e-4 if softmin else 2e-5))
        assert rel_l2(gb[name], ga[name]) <= tol, (name, rel_l2(gb[name], ga[name]))


def _is_fused(out, tracking):
    fused = out.__dict__.get("_fused")
    return (type(out).__name__ == "LazyModelOutput" and fused.flow_done and fused.track_done == tracking
            and fused.engine._network)


CASES = [(i, t, uw, pts) for i in ("regressed", "softmin") for t in (False, True) for uw in (True, False)
         for pts in (None, 1000)]


@pytest.mark.parametrize("intrinsics,tracking,use_weights,points", CASES)
def test_fused_equals_per_op(intrinsics, tracking, use_weights, points):
    model, losses, batch, flows, tracks = _setup("mlp_original", intrinsics, tracking, use_weights, points)
    pa, ga, _ = _step(model, losses, batch, flows, tracks, fused=False)
    pb, gb, out = _step(model, losses, batch, flows, tracks, fused=True)
    assert _is_fused(out, tracking)
    assert model.backbone.calls == 2
    expect = {"backbone.features.0.weight", "backbone.depth_head.weight"} | \
        ({"backbone.head.0.weight"} if use_weights else set()) | \
        ({"intrinsics.focal_length"} if intrinsics == "regressed" else set())
    assert expect <= set(gb), sorted(gb)
    _assert_close(pa, ga, pb, gb, intrinsics == "softmin")


@pytest.mark.parametrize("kind,intrinsics,tracking,w", [
    ("mlp_exp", "regressed", True, W_), ("mlp_exp", "softmin", False, W_), ("logits", "regressed", True, W_),
    ("logits", "softmin", True, W_), ("mlp_original", "regressed", True, W_ - 2), ("logits", "softmin", False, W_ - 2)])
def test_fused_equals_per_op_mappings_and_shapes(kind, intrinsics, tracking, w):
    """The exp mapping, learned logits (weight_sensitivity set), and a width that is not a multiple of 4
    (the dense Procrustes backward instead of the scatter window)."""
    model, losses, batch, flows, tracks = _setup(kind, intrinsics, tracking, w=w)
    pa, ga, _ = _step(model, losses, batch, flows, tracks, fused=False)
    pb, gb, out = _step(model, losses, batch, flows, tracks, fused=True)
    assert _is_fused(out, tracking)
    _assert_close(pa, ga, pb, gb, intrinsics == "softmin")


def _oracle_grads(depths, weights, model, flows, tracks, idx, dtype):
    """d total / d depths and d total / d weights of the float64 (or float32) oracle at the given depths and
    weights: Procrustes poses, 1000 x flow loss [+ 100 x tracking loss], K from the regressed focal length
    or the softmin sweep."""
    from oracle import flowmap_oracle as O
    _, f, h, w = depths.shape
    d = depths.detach().to("cpu", dtype).requires_grad_(True)
    wt = weights.detach().to("cpu", dtype).requires_grad_(True)
    fl = O.Flows(*(t.detach().to("cpu", dtype) for t in (flows.forward, flows.backward, flows.forward_mask,
                                                        flows.backward_mask)))
    intr = model.intrinsics
    if hasattr(intr, "focal_length_candidates"):
        cand = intr.focal_length_candidates.detach().to("cpu", dtype)
        k = O.softmin_focal(d, wt, fl.backward, intr.injected_indices.cpu(), cand)[0][:, None].expand(1, f, 3, 3)
    else:
        k = O.intrinsics_from_focal(intr.focal_length.detach().to("cpu", dtype), h, w).expand(1, f, 3, 3)
    surf = O.unproject(O.pixel_grid(h, w, dtype), d, k[:, :, None, None])
    ext = O.align_surfaces(surf, fl.backward, wt, idx)
    total = 1000.0 * O.flow_loss(surf, ext, k, fl, "huber", 0.01)
    if tracks is not None:
        ot = [O.Tracks(t.xy.to("cpu", dtype), t.visibility.cpu(), t.start_frame) for t in tracks]
        total = total + 100.0 * O.tracking_loss(surf, ext, k, ot, "huber", 0.01)
    total.backward()
    return d.grad, wt.grad


@pytest.mark.parametrize("intrinsics,tracking,w,points,spread", [
    ("regressed", True, W_, None, WIDE), ("softmin", True, W_, None, WIDE), ("regressed", True, W_, 1000, WIDE),
    ("regressed", True, W_, None, None), ("softmin", True, W_, None, None), ("regressed", True, W_ - 2, None, None),
    ("softmin", False, W_ - 2, None, None), ("regressed", True, W_, 1000, None), ("softmin", True, W_ - 2, 1000, None)])
def test_input_gradients_vs_float64_oracle(intrinsics, tracking, w, points, spread):
    """At step 0 the fused halves' d loss / d depths and d loss / d weights (all pixels with W % 4 == 0: the
    scatter window; otherwise the dense backward; 1000 points: the index path) against the float64 oracle
    on the same depths and weights, within max(5e-4, 4 x the float32 oracle's own error); depths from tens to
    thousands (WIDE) or of about 400 to 2200."""
    extra = {} if spread is None else {"spread": spread}
    model, losses, batch, flows, tracks = _setup("mlp_original", intrinsics, tracking, w=w, points=points, **extra)
    model.zero_grad(set_to_none=True)
    out = model(batch, flows, 0)
    depths, weights = out.depths, out.backward_correspondence_weights
    depths.retain_grad()
    weights.retain_grad()
    sum(l.forward(batch, flows, tracks, out, 0) for l in losses).backward()
    assert _is_fused(out, tracking)
    d_, h_ = depths.detach(), depths.shape[-2]
    if spread is not None:
        assert float(d_.min()) < 100.0 and float(d_.max()) > 1000.0, (float(d_.min()), float(d_.max()))
    floor = float((weights.detach() <= 1.0001e-4).float().mean())
    assert 0.05 < floor < 0.95, floor
    idx = model.extrinsics.select_indices(h_, w, depths.device)
    idx = torch.arange(h_ * w) if idx is None else idx.cpu()
    gd64, gw64 = _oracle_grads(depths, weights, model, flows, tracks, idx, torch.float64)
    gd32, gw32 = _oracle_grads(depths, weights, model, flows, tracks, idx, torch.float32)
    for name, got, ref, f32 in (("depths", depths.grad, gd64, gd32), ("weights", weights.grad, gw64, gw32)):
        err, noise = rel_l2(got.cpu(), ref), rel_l2(f32, ref)
        print(f"{intrinsics} tracking={tracking} w={w} points={points} spread={spread} d/d{name}: {err:.3e} "
              f"(float32 oracle {noise:.3e})")
        assert err <= max(5e-4, 4.0 * noise), (name, err, noise)


def test_adam_run_across_tracking_and_hand_over():
    """Six steps of torch.optim.Adam over the network parameters and the focal length, with the tracking
    loss switched on at step 2 and the softmin -> regressed hand-over at step 4 (window 2): fused and per-op
    runs from the same start give losses within 1e-4, the same focal estimates in the hand-over window within
    1e-5, and
    parameter updates whose relative L2 distance stays below 1e-2."""
    base, losses, batch, flows, tracks = _setup("mlp_original", "softmin", True, regression=(4, 2), tracking_after=2)
    runs = {}
    for fused in (False, True):
        model = copy.deepcopy(base)
        start = {n: p.detach().clone() for n, p in model.named_parameters()}
        opt = torch.optim.Adam(model.parameters(), lr=1e-4)
        hist = []
        for step in range(6):
            opt.zero_grad(set_to_none=True)
            parts, _, out = _step(model, losses, batch, flows, tracks, fused=fused, step=step, zero=False)
            if fused:
                assert _is_fused(out, step >= 2)
            hist.append(sum(parts))
            opt.step()
        moved = {n: (p.detach() - start[n]) for n, p in model.named_parameters()}
        runs[fused] = hist, moved, torch.stack(model.intrinsics.window).cpu()
    (ha, ma, wa), (hb, mb, wb) = runs[False], runs[True]
    for a, b in zip(ha, hb):
        assert abs(a - b) <= 1e-4 * abs(a), (ha, hb)
    assert wa.shape == wb.shape == (2,) and float((wa - wb).abs().max()) <= 1e-5, (wa, wb)
    for name in ma:
        if float(ma[name].norm()) > 0:
            assert rel_l2(mb[name], ma[name]) <= 1e-2, (name, rel_l2(mb[name], ma[name]))


def test_backbone_runs_once_per_step():
    model, losses, batch, flows, tracks = _setup("mlp_original", "regressed", True)
    bb = model.backbone
    # outputs read after the losses: a snapshot of the fused step, from the stored BackboneOutput
    pa, ga, out = _step(model, losses, batch, flows, tracks, fused=True)
    assert bb.calls == 1 and _is_fused(out, True)
    ext, k = out.extrinsics, out.intrinsics
    assert bb.calls == 1 and not ext.requires_grad and ext.shape == (1, F_, 4, 4) and k.shape == (1, F_, 3, 3)
    assert out.depths is out.__dict__["_fused"].backbone_out.depths
    # an output read before the losses retires the fused step and gives the per-op results
    model.zero_grad(set_to_none=True)
    out2 = model(batch, flows, 0)
    ext_before = out2.extrinsics
    assert bb.calls == 2 and ext_before.requires_grad and out2.__dict__["_fused"].dead
    parts = [l.forward(batch, flows, tracks, out2, 0) for l in losses]
    sum(parts).backward()
    assert bb.calls == 2
    assert torch.allclose(ext_before.detach(), ext, atol=1e-5)
    _, gc, _ = _step(model, losses, batch, flows, tracks, fused=False)
    assert bb.calls == 3
    for name, p in model.named_parameters():
        assert rel_l2(p.grad, gc[name]) <= 1e-5, name
    _assert_close([float(p) for p in parts], gc, pa, ga, False)


def test_grad_output_scale_and_kept_gradients():
    model, losses, batch, flows, tracks = _setup("mlp_original", "regressed", True)
    _, g1, _ = _step(model, losses, batch, flows, tracks, fused=True)
    _, g2, _ = _step(model, losses, batch, flows, tracks, fused=True, scale=0.25)
    for name in g1:
        assert rel_l2(g2[name], 0.25 * g1[name]) <= 1e-5, name
    model.zero_grad(set_to_none=True)
    for _ in range(2):  # two backwards accumulate
        _step(model, losses, batch, flows, tracks, fused=True, zero=False)
    for name, p in model.named_parameters():
        assert rel_l2(p.grad, 2.0 * g1[name]) <= 1e-5, name


def test_bf16_autocast_output_gets_the_float32_gradient():
    """A bf16 backbone output (autocast) is cast to float32 inside the graph: the network's float32 parameters
    get the gradient the per-op path gives the same network with its outputs cast to float32 itself."""
    model, losses, batch, flows, tracks = _setup("mlp_original", "regressed", True, bf16=True)
    twin = copy.deepcopy(model)
    twin.backbone.cfg = StandInCfg(**{**model.backbone.cfg.__dict__, "cast_output": True})
    pb, gb, out = _step(model, losses, batch, flows, tracks, fused=True)
    assert out.depths.dtype == torch.bfloat16 and _is_fused(out, True)
    pa, ga, _ = _step(twin, losses, batch, flows, tracks, fused=False)
    for name, g in gb.items():
        assert g.dtype == torch.float32, name
    _assert_close(pa, ga, pb, gb, False, grad_tol=1e-2)


def test_two_videos_and_cpu_outputs_take_the_per_op_path():
    from flowmap_b200.types import ModelOutput
    model, losses, batch, flows, _ = _setup("mlp_original", "regressed", False, b=2)
    out = model(batch, flows, 0)
    assert type(out) is ModelOutput and model.backbone.calls == 1
    sum(l.forward(batch, flows, None, out, 0) for l in losses).backward()
    assert model.backbone.features[0].weight.grad is not None and model.backbone.calls == 1
    model, losses, batch, flows, _ = _setup("mlp_original", "regressed", False, device="cpu")
    with pytest.raises(ValueError, match="CUDA tensor"):
        model(batch, flows, 0)
    assert model.backbone.calls == 1


def test_explicit_depth_step_before_the_tracking_loss_is_enabled():
    """The explicit-depth drop-in surface at a step whose tracking loss is not enabled yet (global_step <
    enable_after): the backward half takes no pose gradient from what the tracking buffers hold from an
    earlier step, and matches the per-op path."""
    from test_gpu_dropin_fused import _setup as setup_explicit, _step as step_explicit
    model, losses, batch, flows, tracks = setup_explicit("regressed", True)
    losses[1].cfg.enable_after = 1
    step_explicit(model, losses, batch, flows, tracks, fused=True, step=1)  # tracking on: fills its buffers
    pa, ga, _ = step_explicit(model, losses, batch, flows, tracks, fused=False, step=0)
    pb, gb, out = step_explicit(model, losses, batch, flows, tracks, fused=True, step=0)
    assert out.__dict__["_fused"].flow_done and not out.__dict__["_fused"].track_done
    _assert_close(pa, ga, pb, gb, False)
