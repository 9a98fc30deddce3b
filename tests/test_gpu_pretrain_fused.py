"""`-m gpu`: the pretraining step (pretrain.py, model_wrapper_pretrain.py) on the fused halves: a network
backbone over a batch of B > 1 videos, softmin intrinsics without a regression stage (one candidate sweep and
one focal length per video), Procrustes poses and LossFlow, whose batch loss is normalised by ONE mask sum
pooled over all videos (loss_flow.py:31-70).  The fused step runs on the packed layout of
fm_overfit_step_videos with that pooled sum in every video's slot.

Every video has its own content, flows and masks, and the mask sums differ by more than 2x from one video to
the next, so that a per-video normaliser or a mix-up of videos shows.  Checked: fused == per-op (losses, the
gradient of every network parameter and each video's d loss / d depths and d loss / d weights), those input
gradients against the float64 oracle, the pooled loss against one-video fused steps, grad_output scales and
accumulation, a six-step Adam run on a new batch every step, the per-op fall-backs and the refusals of the C
ABI's packed split step and of its step switch."""
import copy
import ctypes

import pytest
import torch

from conftest import rel_l2
from test_gpu_network_backbone import WIDE, BACKBONE_KINDS, StandInCfg, _assert_close, _register, _video

pytestmark = pytest.mark.gpu

F_, H_, W_ = 6, 40, 64
MASK_RATIO = 0.45  # video v's masks are scaled by MASK_RATIO ** v: mask sums more than 2x apart


def _flows(b, f, h, w, seed):
    import bench
    from flowmap_b200.types import Flows
    per = [bench.synthetic_inputs(f, h, w, seed=seed + 101 * (v + 1)) for v in range(b)]
    scale = [MASK_RATIO ** v for v in range(b)]
    return Flows(torch.cat([p["fwd"] for p in per]), torch.cat([p["bwd"] for p in per]),
                 torch.cat([p["fmask"] * s for p, s in zip(per, scale)]),
                 torch.cat([p["bmask"] * s for p, s in zip(per, scale)]))


def _mapping(name):
    from flowmap_b200.loss import MappingHuberCfg, MappingL1Cfg, MappingL2Cfg
    return {"huber": MappingHuberCfg("huber", 0.01), "l1": MappingL1Cfg("l1"), "l2": MappingL2Cfg("l2")}[name]


def _setup(b, f=F_, h=H_, w=W_, kind="mlp_original", use_weights=True, points=None, mapping="huber", seed=0,
           intrinsics="softmin", regression=None, **backbone):
    from flowmap_b200.loss import LossFlowCfg, get_losses
    from flowmap_b200.model import (ExtrinsicsProcrustesCfg, IntrinsicsGroundTruthCfg, IntrinsicsSoftminCfg, Model,
                                    ModelCfg, RegressionCfg)
    _register()
    dev = torch.device("cuda:0")
    torch.manual_seed(seed)
    if intrinsics == "ground_truth":
        icfg = IntrinsicsGroundTruthCfg("ground_truth")
    else:
        icfg = IntrinsicsSoftminCfg("softmin", 500, 0.5, 2.0, 60, None if regression is None else RegressionCfg(*regression))
    bcfg = StandInCfg(**{**BACKBONE_KINDS[kind].__dict__, **backbone})
    model = Model(ModelCfg(bcfg, icfg, ExtrinsicsProcrustesCfg("procrustes", points, False), use_weights), f, (h, w)).to(dev)
    if intrinsics == "softmin":
        model.intrinsics.injected_indices = torch.randperm(h * w, generator=torch.Generator().manual_seed(3))[:500].to(dev)
    losses = get_losses([LossFlowCfg(0, 1000.0, "flow", _mapping(mapping))])
    batch = _batch(b, f, h, w, seed, dev)
    flows = _flows(b, f, h, w, seed).to(dev)
    return model, losses, batch, flows


def _batch(b, f, h, w, seed, dev):
    from flowmap_b200.types import Batch
    k = torch.tensor([[0.9, 0.0, 0.5], [0.0, 1.2, 0.5], [0.0, 0.0, 1.0]]).expand(b, f, 3, 3)
    return Batch(_video(f, h, w, seed, b).to(dev), torch.arange(f, device=dev)[None].expand(b, f), ["s"] * b,
                 ["d"] * b, intrinsics=k.to(dev))


def _step(model, losses, batch, flows, fused, scale=None, step=0, zero=True, tracks=None):
    """One pretraining step without the optimiser: losses, the network's gradients, the ModelOutput and the
    gradients of the step's depths / weights (the backbone's outputs)."""
    from flowmap_b200.model import Model
    Model.fused_enabled = fused
    try:
        if zero:
            model.zero_grad(set_to_none=True)
        out = model(batch, flows, step)
        depths, weights = out.depths, out.backward_correspondence_weights
        depths.retain_grad()
        if weights.requires_grad:  # without correspondence weights: ones, outside the graph
            weights.retain_grad()
        parts = [l.forward(batch, flows, tracks, out, step) for l in losses]
        total = sum(parts)
        (total if scale is None else total * scale).backward()
        grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
        inputs = {"depths": depths.grad.detach().clone(),
                  "weights": None if weights.grad is None else weights.grad.detach().clone()}
        return [float(p.detach()) for p in parts], grads, out, inputs
    finally:
        Model.fused_enabled = True


def _is_fused(out, b):
    fused = out.__dict__.get("_fused")
    return (type(out).__name__ == "LazyModelOutput" and fused.flow_done and fused.engine._network and
            fused.engine.B == b and (b == 1 or fused.engine._layout is not None))


def _assert_inputs_close(ia, ib, tol):
    """Each video's d loss / d depths and d loss / d weights on its own: a gradient booked on the wrong video,
    or with its own normaliser, fails even where that video's share of the whole is small."""
    for name in ("depths", "weights"):
        if ia[name] is None:
            assert ib[name] is None
            continue
        for v in range(ia[name].shape[0]):
            err = rel_l2(ib[name][v], ia[name][v])
            assert err <= tol, (name, v, err)


CASES = [  # (B, F, W, Procrustes points, weights, backbone, mapping)
    (2, 8, W_, None, True, "mlp_exp", "huber"),
    (5, 8, W_, None, True, "logits", "l1"),
    (2, 2, W_, None, False, "mlp_original", "l2"),
    (5, 2, W_ - 2, None, True, "mlp_original", "huber"),
    (2, 8, W_ - 2, None, False, "logits", "huber"),
    (5, 8, W_, 1000, True, "mlp_original", "l2"),
    (2, 2, W_, 1000, True, "logits", "l1"),
    (5, 8, W_ - 2, 1000, False, "mlp_original", "huber"),
]


@pytest.mark.parametrize("b,f,w,points,use_weights,kind,mapping", CASES)
def test_fused_equals_per_op(b, f, w, points, use_weights, kind, mapping):
    """All pixels with W % 4 == 0 (the scatter window), W % 4 != 0 (the dense backward), 1000 Procrustes points
    (the index path); with and without correspondence weights; MLP and learned-logit weight heads; huber, l1
    and l2."""
    model, losses, batch, flows = _setup(b, f=f, w=w, kind=kind, use_weights=use_weights, points=points,
                                         mapping=mapping)
    pa, ga, out_a, ia = _step(model, losses, batch, flows, fused=False)
    assert type(out_a).__name__ == "ModelOutput"
    pb, gb, out, ib = _step(model, losses, batch, flows, fused=True)
    assert _is_fused(out, b)
    assert model.backbone.calls == 2
    expect = {"backbone.features.0.weight", "backbone.depth_head.weight"}
    if use_weights:
        expect |= {"backbone.head.0.weight"} if kind != "logits" else {"backbone.weights"}
    assert expect <= set(gb), sorted(gb)
    _assert_close(pa, ga, pb, gb, True)
    _assert_inputs_close(ia, ib, 2e-4)
    # the outputs read after the losses: a (B, F, ...) snapshot of the fused step
    assert out.extrinsics.shape == (b, f, 4, 4) and out.intrinsics.shape == (b, f, 3, 3)
    assert out.k4.shape == (b, f, 4) and out.relative.shape == (b, f - 1, 3, 4)
    assert torch.allclose(out.extrinsics, out_a.extrinsics.detach(), rtol=1e-4, atol=1e-4)
    assert torch.allclose(out.k4, out_a.k4.detach(), rtol=1e-4)


def _oracle_grads(depths, weights, model, flows, idx, dtype):
    """d total / d depths and d total / d weights of the float64 (or float32) oracle at the given depths and
    weights: the softmin sweep of every video, Procrustes poses, 1000 x LossFlow pooled over the batch."""
    from oracle import flowmap_oracle as O
    b, f, h, w = depths.shape
    d = depths.detach().to("cpu", dtype).requires_grad_(True)
    wt = weights.detach().to("cpu", dtype).requires_grad_(True)
    fl = O.Flows(*(t.detach().to("cpu", dtype) for t in (flows.forward, flows.backward, flows.forward_mask,
                                                        flows.backward_mask)))
    intr = model.intrinsics
    cand = intr.focal_length_candidates.detach().to("cpu", dtype)
    k = O.softmin_focal(d, wt, fl.backward, intr.injected_indices.cpu(), cand)[0][:, None].expand(b, f, 3, 3)
    surf = O.unproject(O.pixel_grid(h, w, dtype), d, k[:, :, None, None])
    ext = O.align_surfaces(surf, fl.backward, wt, idx)
    (1000.0 * O.flow_loss(surf, ext, k, fl, "huber", 0.01)).backward()
    return d.grad, wt.grad


@pytest.mark.parametrize("w,points,spread", [(W_, None, WIDE), (W_, None, None), (W_ - 2, None, None),
                                             (W_, 1000, None), (W_ - 2, 1000, WIDE)])
def test_input_gradients_vs_float64_oracle(w, points, spread):
    """B = 3: the fused d loss / d depths and d loss / d weights of every video against the float64 oracle,
    within max(5e-4, 4 x the float32 oracle's own error); depths from tens to thousands (WIDE) or of about
    400 to 2200."""
    extra = {} if spread is None else {"spread": spread}
    model, losses, batch, flows = _setup(3, w=w, points=points, **extra)
    _, _, out, grads = _step(model, losses, batch, flows, fused=True)
    assert _is_fused(out, 3)
    depths, weights = out.depths.detach(), out.backward_correspondence_weights.detach()
    if spread is not None:
        assert float(depths.min()) < 100.0 and float(depths.max()) > 1000.0
    h_ = depths.shape[-2]
    idx = model.extrinsics.select_indices(h_, w, depths.device)
    idx = torch.arange(h_ * w) if idx is None else idx.cpu()
    gd64, gw64 = _oracle_grads(depths, weights, model, flows, idx, torch.float64)
    gd32, gw32 = _oracle_grads(depths, weights, model, flows, idx, torch.float32)
    for name, got, ref, f32 in (("depths", grads["depths"], gd64, gd32), ("weights", grads["weights"], gw64, gw32)):
        for v in range(3):
            err, noise = rel_l2(got[v].cpu(), ref[v]), rel_l2(f32[v], ref[v])
            print(f"w={w} points={points} spread={spread} video {v} d/d{name}: {err:.3e} (float32 oracle {noise:.3e})")
            assert err <= max(5e-4, 4.0 * noise), (name, v, err, noise)


def test_pooled_normaliser_is_what_is_computed():
    """The batch's fused loss is sum_b (solo loss_b * M_b / M), solo loss_b being the fused one-video step of
    video b (normalised by its own mask sum M_b) and M the pooled sum; the per-video-normalised sum
    sum_b solo loss_b is more than 10 % away."""
    from flowmap_b200 import ops
    from flowmap_b200.types import Batch, Flows
    b = 3
    model, losses, batch, flows = _setup(b)
    (loss,), _, out, _ = _step(model, losses, batch, flows, fused=True)
    assert _is_fused(out, b)
    solo, m = [], []
    for v in range(b):
        bv = Batch(batch.videos[v:v + 1], batch.indices[v:v + 1], ["s"], ["d"])
        fv = Flows(*(getattr(flows, n)[v:v + 1].contiguous() for n in ("forward", "backward", "forward_mask",
                                                                        "backward_mask")))
        (lv,), _, out_v, _ = _step(model, losses, bv, fv, fused=True)
        assert _is_fused(out_v, 1)
        solo.append(lv)
        m.append(float(ops.mask_sum(fv.forward_mask, fv.backward_mask)))
    pooled = sum(s * mv for s, mv in zip(solo, m)) / sum(m)
    assert abs(loss - pooled) <= 1e-5 * abs(pooled), (loss, pooled)
    assert abs(sum(solo) - loss) > 0.1 * abs(loss), (sum(solo), loss)
    assert all(m[v] > 2.0 * m[v + 1] for v in range(b - 1)), m


def test_grad_output_scale_and_accumulation():
    """One d total / d loss for the whole batch: a 0.25 scale gives 0.25 x every gradient, the sweep's backward
    included (its d loss / d focal of every video comes from the scaled focal gradient), and two backwards
    accumulate."""
    model, losses, batch, flows = _setup(3)
    _, g1, _, i1 = _step(model, losses, batch, flows, fused=True)
    _, g2, out, i2 = _step(model, losses, batch, flows, fused=True, scale=0.25)
    assert _is_fused(out, 3)
    for name in g1:
        assert rel_l2(g2[name], 0.25 * g1[name]) <= 1e-5, name
    for name in ("depths", "weights"):
        for v in range(3):
            assert rel_l2(i2[name][v], 0.25 * i1[name][v]) <= 1e-5, (name, v)
    model.zero_grad(set_to_none=True)
    for _ in range(2):
        _step(model, losses, batch, flows, fused=True, zero=False)
    for name, p in model.named_parameters():
        assert rel_l2(p.grad, 2.0 * g1[name]) <= 1e-5, name


def test_adam_run_on_a_new_batch_every_step():
    """Six steps of torch.optim.Adam over the network, each on a new batch with new Flows, as a loader hands
    them out: fused and per-op runs from the same start give losses within 1e-4 and parameter updates within
    1e-2 (relative L2).  The fused engine is built once and reads each step's Flows tensors themselves."""
    base, losses, _, _ = _setup(4)
    dev = torch.device("cuda:0")
    data = [(_batch(4, F_, H_, W_, 10 + s, dev), _flows(4, F_, H_, W_, 10 + s).to(dev)) for s in range(6)]
    runs = {}
    for fused in (False, True):
        model = copy.deepcopy(base)
        start = {n: p.detach().clone() for n, p in model.named_parameters()}
        opt = torch.optim.Adam(model.parameters(), lr=1e-4)
        hist, engines = [], set()
        for step, (batch, flows) in enumerate(data):
            opt.zero_grad(set_to_none=True)
            parts, _, out, _ = _step(model, losses, batch, flows, fused=fused, step=step, zero=False)
            if fused:
                assert _is_fused(out, 4)
                eng = out.__dict__["_fused"].engine
                engines.add(id(eng))
                a = eng._args
                assert (a.fflow, a.bflow, a.fmask, a.bmask) == tuple(
                    t.data_ptr() for t in (flows.forward, flows.backward, flows.forward_mask, flows.backward_mask))
            hist.append(sum(parts))
            opt.step()
        if fused:
            assert len(engines) == 1
        runs[fused] = hist, {n: p.detach() - start[n] for n, p in model.named_parameters()}
    (ha, ma), (hb, mb) = runs[False], runs[True]
    for a, b in zip(ha, hb):
        assert abs(a - b) <= 1e-4 * abs(a), (ha, hb)
    for name in ma:
        if float(ma[name].norm()) > 0:
            assert rel_l2(mb[name], ma[name]) <= 1e-2, (name, rel_l2(mb[name], ma[name]))


def test_fall_backs_take_the_per_op_path():
    """B = 2 with softmin intrinsics and a regression stage, ground-truth intrinsics, tracks, or in eval mode:
    the step runs per-op and its output is a plain ModelOutput."""
    import bench
    from flowmap_b200.types import ModelOutput, Tracks
    for kw in ({"regression": (10, 5)}, {"intrinsics": "ground_truth"}):
        model, losses, batch, flows = _setup(2, **kw)
        out = model(batch, flows, 0)
        assert type(out) is ModelOutput
        sum(l.forward(batch, flows, None, out, 0) for l in losses).backward()
        assert model.backbone.features[0].weight.grad is not None and model.backbone.calls == 1
    model, losses, batch, flows = _setup(2)
    model.eval()
    out = model(batch, flows, 0)
    assert type(out) is ModelOutput
    # tracks are seen by the losses only: the flow loss declines the fused step before it runs anything, and
    # the output materialises per-op
    model, losses, batch, flows = _setup(2)
    tracks = [Tracks(xy.cuda(), vis.cuda(), s) for xy, vis, s in bench.synthetic_track_arrays(F_, n_points=16, seed=0)]
    pa, ga, _, ia = _step(model, losses, batch, flows, fused=False, tracks=tracks)
    pb, gb, out, ib = _step(model, losses, batch, flows, fused=True, tracks=tracks)
    fused = out.__dict__["_fused"]
    assert fused.dead and not fused.flow_done and fused.engine is None
    assert type(object.__getattribute__(out, "_full")) is ModelOutput
    _assert_close(pa, ga, pb, gb, True)
    _assert_inputs_close(ia, ib, 2e-4)


def test_packed_split_step_refusals():
    """The C ABI's packed split step takes no tracks, no parameter update and no metrics log."""
    from flowmap_b200._lib import FlowmapLibraryError, PackedTracksC
    model, losses, batch, flows = _setup(2)
    _, _, out, _ = _step(model, losses, batch, flows, fused=True)
    assert _is_fused(out, 2)
    eng = out.__dict__["_fused"].engine
    tracks = PackedTracksC()
    log = torch.zeros(4, 2, 5, device="cuda:0")
    for phase in (1, 2):
        for field, value, match in (("tracks", ctypes.pointer(tracks), "takes no tracks"),
                                    ("step", 1, "updates no parameter"), ("defer_adam", 1, "updates no parameter"),
                                    ("metrics_log", log.data_ptr(), "no metrics log")):
            with pytest.raises(FlowmapLibraryError, match=match):
                eng._call_step("fm_overfit_step_videos", phase=phase, **{field: value})


def test_step_switch_refusals():
    """The C ABI's `step` switches the update off (0) or on (1), and an update takes Adam's bias corrections
    from the step clock: fm_overfit_step refuses step = 1 without a clock and step = 2, before any launch."""
    from flowmap_b200._lib import FlowmapLibraryError, lib
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch
    f, h, w = 4, 16, 24
    dev = torch.device("cuda:0")
    batch = Batch(torch.zeros(1, f, 3, h, w, device=dev), torch.arange(f, device=dev)[None], ["s"], ["d"])
    o = FusedOverfitter(OverfitCfg(), batch, _flows(1, f, h, w, 0).to(dev), device=dev)
    assert o._args.clock is not None
    torch.cuda.synchronize()
    for fields, match in (({"step": 1, "clock": None}, "needs the step clock"),
                          ({"step": 2}, r"off \(0\) or on \(1\)")):
        n0 = lib().fm_launch_count()
        with pytest.raises(FlowmapLibraryError, match=match):
            o._call_step(**fields)
        assert lib().fm_launch_count() == n0, fields
