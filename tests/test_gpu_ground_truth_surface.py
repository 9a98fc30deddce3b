"""`-m gpu`: ground-truth intrinsics (model/intrinsics: ground_truth, calibrated data) on the reference-shaped
surface, Model.forward -> LossFlow / LossTracking -> backward(), which now runs the fused halves: explicit depth,
a network backbone on one video, and a network backbone's batch of videos (the pretraining step).  K comes with
the batch, different for every video and frame, with off-centre principal points, and is read into the step on
every step.

Bars as in the rest of the suite: loss 1e-4 relative, poses 2e-5 absolute, every gradient max(1e-4, 3x the
float32 oracle's error); comparisons between the fused and the per-op surface (Model.fused_enabled = False)
against the per-op path's run-to-run noise."""
import copy
import warnings
from contextlib import contextmanager
from dataclasses import make_dataclass, replace

import pytest
import torch

import test_gpu_fused_ground_truth_intrinsics as GT
import test_gpu_per_frame_intrinsics as PF
import test_gpu_pretrain_fused as PT
from conftest import load_golden, rel_l2
from flow_regime_checks import check, errors, kmat
from oracle import flowmap_oracle as O
from pretrain_gt_checks import pretrain_gt_oracle
from flowmap_b200.types import ModelOutput

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _threads():
    torch.set_num_threads(min(16, torch.get_num_threads()))


@contextmanager
def _path(fused):
    from flowmap_b200.model import Model
    Model.fused_enabled = fused
    try:
        yield
    finally:
        Model.fused_enabled = True


def _is_fused(out):
    """The output of a fused ground-truth step: an ordinary ModelOutput that holds the batch's K."""
    f = out.__dict__.get("_fused")
    return type(out) is ModelOutput and f is not None and f.flow_done and not f.dead and f.engine._gt


def _surface_step(model, losses, batch, flows, tracks, fused, step=0):
    """One step without the optimiser: per-loss values, the ModelOutput and the gradients of the explicit-depth
    parameters (depth, weights; None without correspondence weights)."""
    with _path(fused):
        model.zero_grad(set_to_none=True)
        out = model(batch, flows, step)
        parts = [l.forward(batch, flows, tracks, out, step) for l in losses]
        sum(parts).backward()
    assert _is_fused(out) == fused
    g_w = model.backbone.weights.grad
    return ([float(p) for p in parts], out, model.backbone.depth.grad.clone(), None if g_w is None else g_w.clone())


# ---------------------------------------------------------------------------------- 1. explicit depth
def _explicit(f, h, w, tracking, use_weights, points, seed=0):
    from flowmap_b200.overfit import OverfitCfg, build_model_and_losses
    depth, wl, flows, tracks, k = GT._video_inputs(f, h, w, seed)
    cfg = OverfitCfg(intrinsics="ground_truth", use_tracking=tracking, tracking_enable_after=0,
                     use_correspondence_weights=use_weights, procrustes_points=points)
    model, losses = build_model_and_losses(cfg, f, (h, w))
    model.to(DEV)
    with torch.no_grad():
        model.backbone.depth.copy_(depth)
        model.backbone.weights.copy_(wl)
    return model, losses, GT._batch(f, h, w, k.to(DEV)), flows.to(DEV), [t.to(DEV) for t in tracks] if tracking else None


@pytest.mark.parametrize("tracking,use_weights,points", [(False, True, None), (True, True, None), (True, False, None),
                                                         (False, False, 1000), (True, True, 1000)])
def test_explicit_depth_fused_equals_per_op(tracking, use_weights, points):
    """Flow +- tracking, correspondence weights on and off, all pixels and 1000 Procrustes points: losses,
    depth.grad and weights.grad of the fused surface against two per-op runs."""
    model, losses, batch, flows, tracks = _explicit(6, 40, 96, tracking, use_weights, points)
    a = _surface_step(model, losses, batch, flows, tracks, False)
    b = _surface_step(model, losses, batch, flows, tracks, False)
    c = _surface_step(model, losses, batch, flows, tracks, True)
    for i in range(len(a[0])):
        n, e = abs(b[0][i] - a[0][i]) / abs(a[0][i]), abs(c[0][i] - a[0][i]) / abs(a[0][i])
        assert e <= max(1e-5, 3 * n), ("loss", i, e, n)
    for i, name in ((2, "depth"), (3, "weights")):
        if a[i] is None:
            assert c[i] is None, name
            continue
        n, e = rel_l2(b[i], a[i]), rel_l2(c[i], a[i])
        print(f"tracking={tracking} weights={use_weights} points={points} d/d{name}: {e:.1e} (per-op noise {n:.1e})")
        assert e <= max(1e-4, 3 * n), (name, e, n)
    out = c[1]  # read after the losses: the fused step's K, principal points included
    assert out.k_mode == "const"
    assert torch.allclose(out.intrinsics, batch.intrinsics) and torch.allclose(out.extrinsics, a[1].extrinsics, atol=2e-5)


@pytest.mark.parametrize("fused", [False, True])
def test_dropin_step0_vs_gt_intrinsics_golden(fused):
    """Explicit depth through the surface on the inputs of gt_intrinsics_f64.npz (the reference's Model in
    float64 with a K per frame, flow + tracking): step 0's loss, poses and gradients on both paths, with the
    reference's own float32 run (gt_intrinsics.npz) as the noise."""
    from flowmap_b200.types import Batch, Flows, Tracks
    g64, g32 = load_golden("gt_intrinsics", True), load_golden("gt_intrinsics", False)
    f, h, w = g64["in_depth"].shape
    T_ = torch.as_tensor
    model, losses = PF._dropin_model(f, h, w, T_(g64["in_depth"]), T_(g64["in_wparam"]))
    batch = Batch(torch.zeros(1, f, 3, h, w, device=DEV), torch.arange(f, device=DEV)[None], ["s"], ["d"],
                  intrinsics=T_(g64["intrinsics"]).float().to(DEV))
    flows = Flows(*(T_(g64[k]).float().to(DEV) for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    trk = [Tracks(T_(g64[f"trk{i}_xy"]).float().to(DEV), T_(g64[f"trk{i}_vis"]).to(DEV), int(g64[f"trk{i}_start"]))
           for i in range(2)]
    parts, out, g_depth, g_w = _surface_step(model, losses, batch, flows, trk, fused)
    assert out.k_mode == "const"

    def ref(g):
        return dict(loss=float(g["loss"]), ext=T_(g["extrinsics"]).double(), g_depth=T_(g["g_depth"]).double(),
                    g_w=T_(g["g_wparam"]).double(), g_focal=None)

    res = dict(loss=sum(parts), ext=out.extrinsics.detach().cpu(), g_depth=g_depth.cpu(), g_w=g_w.cpu(), g_focal=None)
    check(errors(res, ref(g64)), errors(ref(g32), ref(g64)), f"surface fused={fused} vs gt_intrinsics_f64",
          loss_tol=1e-4, pose_tol=2e-5, floor=1e-4)


@pytest.mark.parametrize("fused", [False, True])
def test_dropin_adam_steps_vs_float64_oracle(fused):
    """Model(IntrinsicsGroundTruth, explicit depth) + LossFlow + LossTracking + FusedAdam on a K per frame, on
    both paths: step 0's loss, poses and gradients and every step's loss against OverfitOracle(intrinsics=
    "ground_truth") in float64, then the depth and weight updates over the run."""
    from flowmap_b200.overfit import FusedAdam
    from flowmap_b200.types import Batch, Flows, Tracks
    f, h, w = 6, 72, 136
    depth, wparam, fl, k4 = PF._inputs("zoom", "scene", 1, f, h, w, seed=61)
    depth, wparam = depth[0], wparam[0]
    kmat64 = kmat(k4)
    tracks = [O.Tracks(t.xy.float().double(), t.visibility, t.start_frame)
              for t in O.synthetic_tracks(f, n_points=300, interval=3, radius=2, seed=62, dtype=torch.float64)]
    tracks = PF._guarded_tracks(depth, wparam, fl, kmat64, tracks)
    steps = 4
    ref, st64 = PF._dropin_oracle(depth, wparam, fl, kmat64, tracks, steps, torch.float64)
    ref32, st32 = PF._dropin_oracle(depth, wparam, fl, kmat64, tracks, steps, torch.float32)
    model, losses = PF._dropin_model(f, h, w, depth, wparam)
    batch = Batch(torch.zeros(1, f, 3, h, w, device=DEV), torch.arange(f, device=DEV)[None], ["s"], ["d"],
                  intrinsics=kmat64.float().to(DEV))
    flows = Flows(*(t.float().to(DEV) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))
    trk = [Tracks(t.xy.float().to(DEV), t.visibility.to(DEV), t.start_frame) for t in tracks]
    opt = FusedAdam(model.parameters(), lr=3e-5)
    for step in range(steps):
        parts, out, g_depth, g_w = _surface_step(model, losses, batch, flows, trk, fused, step)
        total = sum(parts)
        err = abs(total - ref[step]["loss"]) / abs(ref[step]["loss"])
        n = abs(ref32[step]["loss"] - ref[step]["loss"]) / abs(ref[step]["loss"])
        print(f"fused={fused} step {step}: loss error {err:.1e} (float32 oracle {n:.1e})")
        assert err <= max(1e-4, 3 * n), (step, err, n)
        if step == 0:
            res = dict(loss=total, ext=out.extrinsics.detach().cpu(), g_depth=g_depth.cpu(), g_w=g_w.cpu(), g_focal=None)
            r64 = lambda r: dict(loss=r["loss"], ext=r["extrinsics"].double(), g_depth=r["grads"]["depth"].double(),  # noqa: E731
                                 g_w=r["grads"]["weights"].double(), g_focal=None)
            check(errors(res, r64(ref[0])), errors(r64(ref32[0]), r64(ref[0])), f"fused={fused} step 0",
                  loss_tol=1e-4, pose_tol=2e-5, floor=1e-4)
        opt.step()
    for name, p, p64, p32 in (("depth", model.backbone.depth, st64.depth, st32.depth),
                              ("weights", model.backbone.weights, st64.weights, st32.weights)):
        start = depth if name == "depth" else wparam
        e = rel_l2(p.detach().double().cpu() - start, p64.detach() - start)
        n = rel_l2(p32.detach().double() - start, p64.detach() - start)
        print(f"fused={fused} after {steps} steps: {name} update error {e:.1e} (float32 oracle {n:.1e})")
        assert e <= max(1e-3, 3 * n), (name, e, n)


def test_fused_engine_equals_per_op_surface():
    """FusedOverfitter(intrinsics="ground_truth"), graph-replayed, against the per-op surface (Model(
    IntrinsicsGroundTruth) + LossFlow + LossTracking + FusedAdam with Model.fused_enabled = False) for 8 steps:
    losses and parameter updates within 3x the per-op path's own run-to-run difference (floors 1e-5 for the
    losses, 1e-4 for the updates)."""
    steps = 8
    depth, wparam, fl, kmat64, tracks = GT._zoom_case(seed=71)
    f, h, w = depth.shape
    cfg = GT._cfg(use_tracking=True, tracking_enable_after=0)
    batch, flows, trk = GT._batch(f, h, w, kmat64.float().to(DEV)), GT._flows(fl), GT._device_tracks(tracks)
    with _path(False):
        a = GT._per_op_run(cfg, batch, flows, trk, depth, wparam, steps)
        b = GT._per_op_run(cfg, batch, flows, trk, depth, wparam, steps)
    o = GT._fused(cfg, batch, flows, trk, depth, wparam, graph=True)
    fused = [float(o.training_step()[0]) for _ in range(steps)]
    c = (fused, o.model.backbone.depth.detach().cpu(), o.model.backbone.weights.detach().cpu())
    loss_err = lambda x, y: max(abs(p - q) / abs(q) for p, q in zip(x, y))  # noqa: E731
    noise, err = loss_err(b[0], a[0]), loss_err(c[0], a[0])
    print(f"losses: fused engine vs per-op surface {err:.1e}, per-op run to run {noise:.1e}")
    assert err <= max(1e-5, 3 * noise), (err, noise)
    for i, (name, start) in enumerate((("depth", depth), ("weights", wparam)), start=1):
        s_ = start.float()
        noise, err = rel_l2(b[i] - s_, a[i] - s_), rel_l2(c[i] - s_, a[i] - s_)
        print(f"{name} update: fused engine vs per-op surface {err:.1e}, per-op run to run {noise:.1e}")
        assert err <= max(1e-4, 3 * noise), (name, err, noise)


def test_reading_the_batch_intrinsics_keeps_the_step_fused():
    """With ground-truth K the output holds the batch's intrinsics and k_mode before the losses: reading them keeps
    the step fused.  Reading the poses before the losses retires it (the per-op path), with the same numbers."""
    model, losses, batch, flows, tracks = _explicit(6, 40, 96, True, True, None)
    with _path(True):
        out = model(batch, flows, 0)
        assert type(out) is ModelOutput and out.k_mode == "const" and out.intrinsics is batch.intrinsics
        parts = [float(l.forward(batch, flows, tracks, out, 0)) for l in losses]
        assert _is_fused(out)
        out2 = model(batch, flows, 0)
        ext = out2.extrinsics  # before the losses: differentiable, per-op
        assert ext.requires_grad and out2.__dict__["_fused"].dead
        parts2 = [float(l.forward(batch, flows, tracks, out2, 0)) for l in losses]
    for a, b in zip(parts, parts2):
        assert abs(a - b) <= 1e-5 * abs(b), (a, b)


# --------------------------------------------------------------------------------- 2. K between steps
@pytest.mark.parametrize("how", ["new_tensor", "in_place"])
def test_new_k_is_used_by_the_next_step(how):
    """After a step on K1, the next step evaluates K2, whether the batch brings a new tensor or the loader
    rewrites the same one: the fused step equals the per-op step on K2 and differs from the step on K1."""
    f, h, w = 6, 40, 96
    model, losses, batch, flows, tracks = _explicit(f, h, w, True, True, None)
    k1 = _surface_step(model, losses, batch, flows, tracks, True)[0]
    k2 = GT._video_inputs(f, h, w, 1)[4].to(DEV)
    if how == "new_tensor":
        batch = replace(batch, intrinsics=k2)
    else:
        batch.intrinsics.copy_(k2)
    eng = model._engine
    fused = _surface_step(model, losses, batch, flows, tracks, True)
    assert model._engine is eng  # not rebuilt
    per_op = _surface_step(model, losses, batch, flows, tracks, False)
    assert torch.equal(eng.intrinsics_k4().cpu(), torch.stack((k2[0, :, 0, 0], k2[0, :, 1, 1], k2[0, :, 0, 2],
                                                               k2[0, :, 1, 2]), -1).cpu())
    for a, b, c in zip(fused[0], per_op[0], k1):
        assert abs(a - b) <= 1e-5 * abs(b), (a, b)
        assert abs(c - b) > 1e-3 * abs(b), (c, b)
    assert rel_l2(fused[2], per_op[2]) <= 1e-4


# ------------------------------------------------------------------------------ 3. no host synchronisation
def _sync_warnings(intrinsics):
    from flowmap_b200.overfit import FusedAdam, OverfitCfg, build_model_and_losses
    f, h, w = 6, 40, 96
    depth, wl, flows, tracks, k = GT._video_inputs(f, h, w, 0)
    cfg = OverfitCfg(intrinsics=intrinsics, use_tracking=True, tracking_enable_after=0)
    model, losses = build_model_and_losses(cfg, f, (h, w))
    model.to(DEV)
    batch, flows, tracks = GT._batch(f, h, w, k.to(DEV)), flows.to(DEV), [t.to(DEV) for t in tracks]
    opt = FusedAdam(model.parameters(), cfg.lr)

    def step(s):
        opt.zero_grad()
        out = model(batch, flows, s)
        sum(l.forward(batch, flows, tracks, out, s) for l in losses).backward()
        opt.step()
        assert out.__dict__["_fused"].flow_done

    for s in range(3):
        step(s)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            step(3)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return len([c for c in caught if "synchroniz" in str(c.message).lower()])


def test_steady_state_step_adds_no_host_synchronisation():
    gt, reg = _sync_warnings("ground_truth"), _sync_warnings("regressed")
    print(f"synchronising calls per step: ground truth {gt}, regressed {reg}")
    assert gt <= reg, (gt, reg)


# ---------------------------------------------------------------------------- 4. network backbone, one video
def _network(f, h, w, tracking, seed=0):
    from flowmap_b200.loss import LossFlowCfg, LossTrackingCfg, MappingHuberCfg, get_losses
    from flowmap_b200.model import ExtrinsicsProcrustesCfg, IntrinsicsGroundTruthCfg, Model, ModelCfg
    import tools.backbone_step  # noqa: F401  (registers bench_param)
    _, _, flows, tracks, k = GT._video_inputs(f, h, w, seed)
    torch.manual_seed(seed)
    bcfg = make_dataclass("StandInCfg", [("name", str)])("bench_param")
    model = Model(ModelCfg(bcfg, IntrinsicsGroundTruthCfg("ground_truth"),
                           ExtrinsicsProcrustesCfg("procrustes", None, False), True), f, (h, w)).to(DEV)
    huber = MappingHuberCfg("huber", 0.01)
    losses = get_losses([LossFlowCfg(0, 1000.0, "flow", huber)] +
                        ([LossTrackingCfg(0, 100.0, "tracking", huber)] if tracking else []))
    return model, losses, GT._batch(f, h, w, k.to(DEV)), flows.to(DEV), [t.to(DEV) for t in tracks] if tracking else None


def _network_step(model, losses, batch, flows, tracks, fused):
    with _path(fused):
        model.zero_grad(set_to_none=True)
        out = model(batch, flows, 0)
        d, wt = out.depths, out.backward_correspondence_weights
        d.retain_grad()
        wt.retain_grad()
        parts = [l.forward(batch, flows, tracks, out, 0) for l in losses]
        sum(parts).backward()
    assert _is_fused(out) == fused
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters()}
    return [float(p) for p in parts], grads, d.grad.clone(), wt.grad.clone(), d.detach(), wt.detach()


def _oracle_input_grads(d, wt, k, flows, tracks, dtype):
    """d total / d depths and d total / d weights of 1000 x flow [+ 100 x tracking] in the oracle."""
    b, f, h, w = d.shape
    d = d.to("cpu", dtype).requires_grad_(True)
    wt = wt.to("cpu", dtype).requires_grad_(True)
    k = k.to("cpu", dtype)
    fl = O.Flows(*(t.detach().to("cpu", dtype) for t in (flows.forward, flows.backward, flows.forward_mask,
                                                        flows.backward_mask)))
    surf = O.unproject(O.pixel_grid(h, w, dtype), d, k[:, :, None, None])
    ext = O.align_surfaces(surf, fl.backward, wt, torch.arange(h * w))
    total = 1000.0 * O.flow_loss(surf, ext, k, fl, "huber", 0.01)
    if tracks is not None:
        trk = [O.Tracks(t.xy.to("cpu", dtype), t.visibility.cpu(), t.start_frame) for t in tracks]
        total = total + 100.0 * O.tracking_loss(surf, ext, k, trk, "huber", 0.01)
    total.backward()
    return d.grad, wt.grad


@pytest.mark.parametrize("tracking", [False, True])
def test_network_backbone_one_video(tracking):
    """The bench_param stand-in on one video: fused equals per-op (losses, the network's gradients), and d loss
    / d depths, d loss / d weights meet the float64 oracle."""
    model, losses, batch, flows, tracks = _network(6, 40, 96, tracking)
    a = _network_step(model, losses, batch, flows, tracks, False)
    b = _network_step(model, losses, batch, flows, tracks, False)
    c = _network_step(model, losses, batch, flows, tracks, True)
    for i in range(len(a[0])):
        n, e = abs(b[0][i] - a[0][i]) / abs(a[0][i]), abs(c[0][i] - a[0][i]) / abs(a[0][i])
        assert e <= max(1e-5, 3 * n), ("loss", i, e, n)
    for name in a[1]:
        n, e = rel_l2(b[1][name], a[1][name]), rel_l2(c[1][name], a[1][name])
        assert e <= max(1e-4, 3 * n), (name, e, n)
    gd64, gw64 = _oracle_input_grads(c[4], c[5], batch.intrinsics, flows, tracks, torch.float64)
    gd32, gw32 = _oracle_input_grads(c[4], c[5], batch.intrinsics, flows, tracks, torch.float32)
    for name, got, r64, r32 in (("depths", c[2], gd64, gd32), ("weights", c[3], gw64, gw32)):
        err, noise = rel_l2(got.cpu(), r64), rel_l2(r32, r64)
        print(f"tracking={tracking} d/d{name}: {err:.2e} (float32 oracle {noise:.2e})")
        assert err <= max(1e-4, 3 * noise), (name, err, noise)


# ---------------------------------------------------------------------------------- 5. the pretraining batch
def _per_video_k(b, f, seed):
    """(B, F, 3, 3): each video its own per-frame zoom and off-centre principal points."""
    g = torch.Generator().manual_seed(seed)
    k = torch.zeros(b, f, 3, 3)
    k[..., 0, 0], k[..., 1, 1] = 0.6 + torch.rand(b, f, generator=g), 0.6 + torch.rand(b, f, generator=g)
    k[..., 0, 2], k[..., 1, 2] = 0.38 + 0.24 * torch.rand(b, f, generator=g), 0.38 + 0.24 * torch.rand(b, f, generator=g)
    k[..., 2, 2] = 1.0
    return k.to(DEV)


def _pretrain(b, f, h, w, points=1000, seed=0):
    model, losses, batch, flows = PT._setup(b, f=f, h=h, w=w, points=points, intrinsics="ground_truth", seed=seed)
    return model, losses, replace(batch, intrinsics=_per_video_k(b, f, seed + 5)), flows


@pytest.mark.parametrize("b,f,h,w", [(4, 6, 40, 64), (16, 8, 128, 192)])
def test_pretraining_batch_fused_equals_per_op_and_oracle(b, f, h, w):
    """B = 4, and the reference's B = 16 x 8 frames x 128 x 192, with per-video, per-frame K: fused equals per-op
    (loss, the network's gradients, each video's input gradients), and each video's d loss / d depths and
    d loss / d weights meet the ground-truth pretraining oracle (pooled mask sum, K per video)."""
    model, losses, batch, flows = _pretrain(b, f, h, w)
    pa, ga, out_a, ia = PT._step(model, losses, batch, flows, fused=False)
    pa2, ga2, _, ia2 = PT._step(model, losses, batch, flows, fused=False)
    pb, gb, out, ib = PT._step(model, losses, batch, flows, fused=True)
    assert _is_fused(out) and out.__dict__["_fused"].engine.B == b
    n, e = abs(pa2[0] - pa[0]) / abs(pa[0]), abs(pb[0] - pa[0]) / abs(pa[0])
    assert e <= max(1e-5, 3 * n), (e, n)
    for name in ga:
        n, e = rel_l2(ga2[name], ga[name]), rel_l2(gb[name], ga[name])
        assert e <= max(1e-4, 3 * n), (name, e, n)
    for name in ("depths", "weights"):
        for v in range(b):
            n, e = rel_l2(ia2[name][v], ia[name][v]), rel_l2(ib[name][v], ia[name][v])
            assert e <= max(1e-4, 3 * n), (name, v, e, n)
    assert out.k_mode == "const" and torch.allclose(out.intrinsics, batch.intrinsics)
    assert torch.allclose(out.extrinsics, out_a.extrinsics.detach(), atol=2e-5)
    d, wt = out.depths.detach(), out.backward_correspondence_weights.detach()
    pidx = model.extrinsics.select_indices(h, w, DEV)
    r64 = pretrain_gt_oracle(d, wt, flows, batch.intrinsics, pidx, dtype=torch.float64)
    r32 = pretrain_gt_oracle(d, wt, flows, batch.intrinsics, pidx, dtype=torch.float32)
    assert abs(pb[0] - r64["loss"]) <= 1e-4 * abs(r64["loss"]), (pb[0], r64["loss"])
    # the stand-in's depths are in the thousands, and so are the translations: the float32 oracle sets the bar
    e, n = float((out.extrinsics.double().cpu() - r64["ext"]).abs().max()), float((r32["ext"] - r64["ext"]).abs().max())
    assert e <= max(2e-5, 3 * n), (e, n)
    for name, key in (("depths", "g_depth"), ("weights", "g_w")):
        for v in range(b):
            err, noise = rel_l2(ib[name][v].cpu(), r64[key][v]), rel_l2(r32[key][v], r64[key][v])
            assert err <= max(1e-4, 3 * noise), (name, v, err, noise)


def test_pretraining_adam_run_on_a_new_batch_and_k_every_step():
    """Six steps of torch.optim.Adam over the network, each on a new batch with new Flows and a new K: fused and
    per-op runs from the same start give losses within 1e-4 and parameter updates within 1e-2 (relative L2); the
    engine is built once."""
    base, losses, _, _ = _pretrain(4, PT.F_, PT.H_, PT.W_)
    data = [(replace(PT._batch(4, PT.F_, PT.H_, PT.W_, 10 + s, DEV), intrinsics=_per_video_k(4, PT.F_, 20 + s)),
             PT._flows(4, PT.F_, PT.H_, PT.W_, 10 + s).to(DEV)) for s in range(6)]
    runs = {}
    for fused in (False, True):
        model = copy.deepcopy(base)
        start = {n: p.detach().clone() for n, p in model.named_parameters()}
        opt = torch.optim.Adam(model.parameters(), lr=1e-4)
        hist, engines = [], set()
        for step, (batch, flows) in enumerate(data):
            opt.zero_grad(set_to_none=True)
            parts, _, out, _ = PT._step(model, losses, batch, flows, fused=fused, step=step, zero=False)
            if fused:
                assert _is_fused(out)
                engines.add(id(out.__dict__["_fused"].engine))
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


# ------------------------------------------------------------------------------- 6. the new C entry point
def test_const_k_tracking_sweep_equals_k_carrying_sweep():
    """The split forward's K-free tracking sweep (fm_track_loss_fwd_const_k) against the K-carrying one
    (fm_track_loss_fwd_sharded) on the same inputs: the same tracking loss, and the same backward gradients
    (the constant-intrinsics backward reads the twist sums both leave)."""
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    model, losses, batch, flows, tracks = _network(6, 40, 96, True, seed=3)
    o = FusedOverfitter(OverfitCfg(intrinsics="ground_truth", weight_sensitivity=0.0, use_tracking=True,
                                   tracking_enable_after=0), batch, flows, tracks, device=DEV, model=model)
    bo = model.backbone(batch, flows)
    d, wt = bo.depths.detach().float().contiguous(), bo.weights.detach().float().contiguous()

    def run(k_carrying):
        o.forward_phase(0, depth=d, weights=wt)
        o._gt = not k_carrying  # the tracking sweep's choice only: the step's K and buffers stay constant-K
        try:
            lt = float(o.tracking_forward_phase())
        finally:
            o._gt = True
        o.backward_phase(with_tracking=True)
        g = o.gradients()
        return lt, g["depth"].clone(), g["weights"].clone()

    a, b, c = run(False), run(False), run(True)
    noise = (abs(b[0] - a[0]) / abs(a[0]), rel_l2(b[1], a[1]), rel_l2(b[2], a[2]))
    err = (abs(c[0] - a[0]) / abs(a[0]), rel_l2(c[1], a[1]), rel_l2(c[2], a[2]))
    print("K-carrying vs K-free sweep (loss, g_depth, g_weights):", [f"{e:.1e}" for e in err],
          "run to run:", [f"{e:.1e}" for e in noise])
    for name, e, n, floor in zip(("loss", "g_depth", "g_weights"), err, noise, (1e-6, 1e-5, 1e-5)):
        assert e <= max(floor, 3 * n), (name, e, n)


def test_const_k_entry_point_refuses_bad_arguments_without_launching():
    from flowmap_b200 import ops
    from flowmap_b200._lib import lib
    L = lib()
    f, h, w = 4, 16, 24
    pk = ops.PackedTracks([t.to(DEV) for t in GT._video_inputs(f, h, w, 0)[3]], DEV)
    depth, k4, ext = torch.ones(f, h, w, device=DEV), torch.ones(f, 4, device=DEV), torch.eye(4, device=DEV).repeat(f, 1, 1)
    ws = torch.empty(L.fm_track_workspace_bytes(f, pk.total), dtype=torch.uint8, device=DEV)
    loss = torch.empty(1, device=DEV)
    P = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    st = torch.cuda.current_stream().cuda_stream

    def call(depth=depth, k4=k4, ext=ext, ws=ws, mapping=0, rng=(0, 0, f)):
        return L.fm_track_loss_fwd_const_k(P(depth), P(k4), P(ext), P(pk.seg), pk.num_segments, pk.max_rows,
                                           pk.max_points, P(pk.xy), P(pk.vis), pk.total, mapping, 0.01, 100.0, P(loss),
                                           P(ws), f, h, w, *rng, st)

    torch.cuda.synchronize()
    for kw, msg in (({"depth": None}, "bad arguments"), ({"k4": None}, "bad arguments"), ({"ws": None}, "bad arguments"),
                    ({"mapping": 3}, "unknown mapping"), ({"rng": (0, 2, f + 1)}, "source-frame range")):
        n0 = L.fm_launch_count()
        assert call(**kw) != 0, kw
        assert msg in L.fm_last_error().decode(), (kw, L.fm_last_error())
        assert L.fm_launch_count() == n0, kw
    assert call() == 0
    torch.cuda.synchronize()
    assert bool(torch.isfinite(loss).all())


# ------------------------------------------------------------------------------------------- 7. fall-backs
def test_fall_backs_take_the_per_op_path():
    """Explicit depth: batch.intrinsics None or on the CPU is not fused, and the step fails in the per-op path as it
    did before (no CPU path, no K); eval mode and no_grad run per-op.  A network batch (B = 2): a softmin regression
    stage, eval mode and tracks run per-op, and the output is a plain ModelOutput."""
    import bench
    from flowmap_b200.types import ModelOutput, Tracks
    model, losses, batch, flows, tracks = _explicit(6, 40, 96, False, True, None)
    for k in (None, batch.intrinsics.cpu()):
        b = replace(batch, intrinsics=k)
        assert not model._fusable(b, flows)
        kinds = []
        for fused in (False, True):
            with _path(fused), pytest.raises((TypeError, ValueError)) as ei:
                model(b, flows, 0)
            kinds.append(type(ei.value))
        assert kinds[0] is kinds[1], kinds
    with torch.no_grad():
        assert type(model(batch, flows, 0)) is ModelOutput
    model.eval()
    assert type(model(batch, flows, 0)) is ModelOutput
    model, losses, batch, flows = PT._setup(2, regression=(10, 5))
    out = model(batch, flows, 0)
    assert type(out) is ModelOutput
    sum(l.forward(batch, flows, None, out, 0) for l in losses).backward()
    assert model.backbone.features[0].weight.grad is not None and model.backbone.calls == 1
    model, losses, batch, flows = _pretrain(2, PT.F_, PT.H_, PT.W_)
    model.eval()
    assert type(model(batch, flows, 0)) is ModelOutput
    model, losses, batch, flows = _pretrain(2, PT.F_, PT.H_, PT.W_)
    trk = [Tracks(xy.cuda(), vis.cuda(), s) for xy, vis, s in bench.synthetic_track_arrays(PT.F_, n_points=16, seed=0)]
    pa, ga, _, ia = PT._step(model, losses, batch, flows, fused=False, tracks=trk)
    pb, gb, out, ib = PT._step(model, losses, batch, flows, fused=True, tracks=trk)
    fused = out.__dict__["_fused"]
    assert fused.dead and not fused.flow_done and fused.engine is None
    assert type(out.__dict__["_full"]) is ModelOutput
    PT._assert_close(pa, ga, pb, gb, True)
    PT._assert_inputs_close(ia, ib, 2e-4)
