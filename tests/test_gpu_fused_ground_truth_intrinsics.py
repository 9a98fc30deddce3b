"""FusedOverfitter with ground-truth intrinsics (model/intrinsics: ground_truth, the configuration of calibrated
data): K comes with the batch, a different one for every frame, and the fused step computes no intrinsics
gradient (fm_overfit_step with focal = g_k4 = track_g_k4 = NULL, the K-free Procrustes backward and tracking
sweep).

- step 0 on the inputs of gt_intrinsics_f64.npz (the reference's Model in float64, flow + tracking) with the
  reference's float32 run as the noise;
- 20 graph-replayed Adam steps against the float64 OverfitOracle(intrinsics="ground_truth");
- the same run as the per-op surface (Model(IntrinsicsGroundTruth) + LossFlow + LossTracking + FusedAdam);
- the constant-intrinsics mode against the K-carrying kernels (scratch g_k4 / track_g_k4);
- packed videos (a list of Batches of different lengths, and a (B, F) tensor batch), each video with its own
  per-frame K, against its solo run;
- the metrics log, a network backbone through forward_phase / backward_phase, set_intrinsics, and the refusals.

Bars as in the rest of the suite: loss 1e-4 relative, poses 2e-5 absolute, every gradient metric max(1e-4, 3x
the float32 oracle's error); comparisons between two fused or per-op runs against their run-to-run noise."""
import ctypes

import pytest
import torch

from conftest import load_golden, rel_l2
from flow_regime_checks import check, errors, k4_regime, kmat
from oracle import flowmap_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SEED = 1234


@pytest.fixture(autouse=True)
def _threads():
    torch.set_num_threads(min(16, torch.get_num_threads()))


def _cfg(**kw):
    from flowmap_b200.overfit import OverfitCfg
    return OverfitCfg(intrinsics="ground_truth", **kw)


def _batch(f, h, w, intrinsics, extrinsics=None, b=1):
    from flowmap_b200.types import Batch
    return Batch(torch.zeros(b, f, 3, h, w, device=DEV), torch.arange(f, device=DEV)[None].expand(b, f),
                 ["s"] * b, ["d"] * b, extrinsics=extrinsics, intrinsics=intrinsics)


def _flows(fl):
    from flowmap_b200.types import Flows
    return Flows(*(t.float().to(DEV) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))


def _fused(cfg, batch, flows, tracks, depth, wparam, graph=False):
    from flowmap_b200.overfit import FusedOverfitter
    o = FusedOverfitter(cfg, batch, flows, tracks, device=DEV)
    o._clock.base_seed = SEED
    with torch.no_grad():
        o.model.backbone.depth.copy_(depth.float())
        o.model.backbone.weights.copy_(wparam.float())
    o.use_cuda_graph = graph
    return o


# ------------------------------------------------------------------------------------------------ golden
def test_step0_vs_gt_intrinsics_golden():
    """Step 0 of the fused ground-truth step on the inputs of gt_intrinsics_f64.npz: loss, extrinsics,
    g_depth and g_weights, the reference's own float32 run (gt_intrinsics.npz) as the noise."""
    from flowmap_b200.types import Flows, Tracks
    g64, g32 = load_golden("gt_intrinsics", True), load_golden("gt_intrinsics", False)
    f, h, w = g64["in_depth"].shape
    T_ = torch.as_tensor
    batch = _batch(f, h, w, T_(g64["intrinsics"]).float().to(DEV))
    flows = Flows(*(T_(g64[k]).float().to(DEV) for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    trk = [Tracks(T_(g64[f"trk{i}_xy"]).float().to(DEV), T_(g64[f"trk{i}_vis"]).to(DEV), int(g64[f"trk{i}_start"]))
           for i in range(2)]
    o = _fused(_cfg(use_tracking=True, tracking_enable_after=0), batch, flows, trk, T_(g64["in_depth"]),
               T_(g64["in_wparam"]))
    assert o._args.focal is None and o._args.g_k4 is None and o._args.track_g_k4 is None
    total, _ = o.training_step(update=False)
    g = o.gradients()
    assert g["focal"] is None

    def ref(gd):
        return dict(loss=float(gd["loss"]), ext=T_(gd["extrinsics"]).double(), g_depth=T_(gd["g_depth"]).double(),
                    g_w=T_(gd["g_wparam"]).double(), g_focal=None)

    res = dict(loss=float(total), ext=o.extrinsics().cpu(), g_depth=g["depth"].cpu(), g_w=g["weights"].cpu(),
               g_focal=None)
    check(errors(res, ref(g64)), errors(ref(g32), ref(g64)), "fused ground_truth vs gt_intrinsics_f64",
          loss_tol=1e-4, pose_tol=2e-5, floor=1e-4)


# ------------------------------------------------------------------------------- many steps, float64 oracle
def _zoom_case(f=6, h=72, w=136, seed=61):
    """The per-frame `zoom` K on the `scene` flows with guarded tracks (test_gpu_per_frame_intrinsics)."""
    import test_gpu_per_frame_intrinsics as PF
    depth, wparam, fl, k4 = PF._inputs("zoom", "scene", 1, f, h, w, seed=seed)
    depth, wparam = depth[0], wparam[0]
    kmat64 = kmat(k4)
    tracks = [O.Tracks(t.xy.float().double(), t.visibility, t.start_frame)
              for t in O.synthetic_tracks(f, n_points=300, interval=3, radius=2, seed=seed + 1, dtype=torch.float64)]
    tracks = PF._guarded_tracks(depth, wparam, fl, kmat64, tracks)
    return depth, wparam, fl, kmat64, tracks


def _device_tracks(tracks):
    from flowmap_b200.types import Tracks
    return [Tracks(t.xy.float().to(DEV), t.visibility.to(DEV), t.start_frame) for t in tracks]


def test_graph_replayed_adam_steps_vs_float64_oracle():
    """20 graph-replayed Adam steps of the fused ground-truth step (flow + tracking from step 0): every step's
    loss, and the depth and weight updates over the run, against OverfitOracle(intrinsics="ground_truth") in
    float64 with its float32 run as the noise."""
    import test_gpu_per_frame_intrinsics as PF
    steps = 20
    depth, wparam, fl, kmat64, tracks = _zoom_case()
    f, h, w = depth.shape
    ref, st64 = PF._dropin_oracle(depth, wparam, fl, kmat64, tracks, steps, torch.float64)
    ref32, st32 = PF._dropin_oracle(depth, wparam, fl, kmat64, tracks, steps, torch.float32)
    o = _fused(_cfg(use_tracking=True, tracking_enable_after=0), _batch(f, h, w, kmat64.float().to(DEV)), _flows(fl),
               _device_tracks(tracks), depth, wparam, graph=True)
    for step in range(steps):
        total, _ = o.training_step()
        err = abs(float(total) - ref[step]["loss"]) / abs(ref[step]["loss"])
        n = abs(ref32[step]["loss"] - ref[step]["loss"]) / abs(ref[step]["loss"])
        print(f"step {step}: loss {float(total):.6e} error {err:.1e} (float32 oracle {n:.1e})")
        assert err <= max(1e-4, 3 * n), (step, err, n)
    assert len(o._graphs) == 1 and o.focal_steps == 0 and o._clock.focal_steps == 0
    for name, p, p64, p32 in (("depth", o.model.backbone.depth, st64.depth, st32.depth),
                              ("weights", o.model.backbone.weights, st64.weights, st32.weights)):
        start = depth if name == "depth" else wparam
        e = rel_l2(p.detach().double().cpu() - start, p64.detach() - start)
        n = rel_l2(p32.detach().double() - start, p64.detach() - start)
        print(f"after {steps} steps: {name} update error {e:.1e} (float32 oracle {n:.1e})")
        assert e <= max(1e-3, 3 * n), (name, e, n)


# ------------------------------------------------------------------------------------ the per-op surface
def _per_op_run(cfg, batch, flows, tracks, depth, wparam, steps):
    from flowmap_b200.model import IntrinsicsGroundTruth
    from flowmap_b200.overfit import Overfitter
    o = Overfitter(cfg, batch, flows, tracks, device=DEV)
    assert isinstance(o.model.intrinsics, IntrinsicsGroundTruth)
    with torch.no_grad():
        o.model.backbone.depth.copy_(depth.float())
        o.model.backbone.weights.copy_(wparam.float())
    losses = []
    for _ in range(steps):
        total, out = o.training_step()
        assert out.k_mode == "const" and type(out).__name__ == "ModelOutput"
        losses.append(float(total))
    return losses, o.model.backbone.depth.detach().cpu(), o.model.backbone.weights.detach().cpu()


def test_fused_equals_per_op_surface():
    """The fused ground-truth step against today's path (Model(IntrinsicsGroundTruth) + LossFlow + LossTracking
    + FusedAdam) for 8 steps: losses and parameter updates within 3x the per-op path's own run-to-run
    difference (floors 1e-5 for the losses, 1e-4 for the updates)."""
    steps = 8
    depth, wparam, fl, kmat64, tracks = _zoom_case(seed=71)
    f, h, w = depth.shape
    cfg = _cfg(use_tracking=True, tracking_enable_after=0)
    batch, flows, trk = _batch(f, h, w, kmat64.float().to(DEV)), _flows(fl), _device_tracks(tracks)
    a = _per_op_run(cfg, batch, flows, trk, depth, wparam, steps)
    b = _per_op_run(cfg, batch, flows, trk, depth, wparam, steps)
    o = _fused(cfg, batch, flows, trk, depth, wparam, graph=True)
    fused = [float(o.training_step()[0]) for _ in range(steps)]
    c = (fused, o.model.backbone.depth.detach().cpu(), o.model.backbone.weights.detach().cpu())
    loss_err = lambda x, y: max(abs(p - q) / abs(q) for p, q in zip(x, y))  # noqa: E731
    noise, err = loss_err(b[0], a[0]), loss_err(c[0], a[0])
    print(f"losses: fused vs per-op {err:.1e}, per-op run to run {noise:.1e}")
    assert err <= max(1e-5, 3 * noise), (err, noise)
    for i, (name, start) in enumerate((("depth", depth), ("weights", wparam)), start=1):
        s = start.float()
        noise = rel_l2(b[i] - s, a[i] - s)
        err = rel_l2(c[i] - s, a[i] - s)
        print(f"{name} update: fused vs per-op {err:.1e}, per-op run to run {noise:.1e}")
        assert err <= max(1e-4, 3 * noise), (name, err, noise)


# ------------------------------------------------------------------------- constant-K mode vs K-carrying
def test_constant_intrinsics_mode_equals_k_carrying_kernels():
    """The step with g_k4 = track_g_k4 = NULL (K-free kernels) and with scratch buffers (today's kernels,
    whose intrinsics gradient is thrown away): loss, rt, g_depth and g_weights agree within 3x the K-free
    step's own run-to-run difference (floors: loss 1e-6 relative, rt 1e-6, gradients 1e-5)."""
    depth, wparam, fl, kmat64, tracks = _zoom_case(f=8, h=96, w=192, seed=81)
    f, h, w = depth.shape
    o = _fused(_cfg(use_tracking=True, tracking_enable_after=0), _batch(f, h, w, kmat64.float().to(DEV)), _flows(fl),
               _device_tracks(tracks), depth, wparam)

    def run():
        total, rt = o.training_step(update=False)
        g = o.gradients()
        return float(total), rt.clone(), g["depth"].clone(), g["weights"].clone()

    a, b = run(), run()
    scratch_k4, scratch_tk4 = torch.empty(f, 4, device=DEV), torch.empty(f, 4, device=DEV)
    o._args.g_k4, o._args.track_g_k4 = scratch_k4.data_ptr(), scratch_tk4.data_ptr()
    try:
        c = run()
    finally:
        o._args.g_k4 = o._args.track_g_k4 = None
    assert bool(torch.isfinite(scratch_k4).all()) and float(scratch_k4.abs().sum()) > 0  # the K path ran

    def diffs(x, y):
        return (abs(x[0] - y[0]) / abs(y[0]), float((x[1] - y[1]).abs().max()), rel_l2(x[2], y[2]), rel_l2(x[3], y[3]))

    noise, err = diffs(b, a), diffs(c, a)
    print("K-carrying vs constant-K (loss, rt, g_depth, g_weights):", [f"{e:.1e}" for e in err],
          "run to run:", [f"{e:.1e}" for e in noise])
    for name, e, n, floor in zip(("loss", "rt", "g_depth", "g_weights"), err, noise, (1e-6, 1e-6, 1e-5, 1e-5)):
        assert e <= max(floor, 3 * n), (name, e, n)


# ----------------------------------------------------------------------------------------- packed videos
def _video_inputs(f, h, w, i):
    import bench
    from flowmap_b200.types import Flows, Tracks
    inp = bench.synthetic_inputs(f, h, w, seed=10 + i)
    k = kmat(k4_regime("videos", 2, f, h, w)[i % 2]).float()[None]  # (1, f, 3, 3): its own zoom per video
    flows = Flows(inp["fwd"], inp["bwd"], inp["fmask"], inp["bmask"])
    tracks = [Tracks(xy, vis, st) for xy, vis, st in
              bench.synthetic_track_arrays(f, n_points=40 + 16 * i, interval=3, radius=2, seed=i)]
    return 1.0 + inp["depth"], inp["wparam"], flows, tracks, k


def _solo(cfg, f, h, w, v, steps):
    depth, wl, flows, tracks, k = v
    o = _fused(cfg, _batch(f, h, w, k.to(DEV)), flows.to(DEV), [t.to(DEV) for t in tracks], depth, wl, graph=True)
    losses, rts = _steps(o, steps)
    return [float(t) for t in losses], [rt[0] for rt in rts], o.model.backbone.depth.detach(), \
        o.model.backbone.weights.detach()


def _steps(o, steps):
    """Per step the totals and the poses, copied: the step's buffers are rewritten by the next one."""
    losses, rts = [], []
    for _ in range(steps):
        total, rt = o.training_step()
        losses.append(total)
        rts.append([r.clone() for r in rt] if isinstance(rt, list) else rt.clone())
    return losses, rts


def _check_solo(i, losses, rts, depth, logits, solo):
    ls, rs, ds, ws = solo
    for s, (a, b) in enumerate(zip(losses, ls)):
        assert abs(a - b) <= 1e-6 * abs(b), (i, s, a, b)
    for s, (a, b) in enumerate(zip(rts, rs)):
        assert float((a - b).abs().max()) <= 2e-6, (i, s)
    assert rel_l2(depth, ds) <= 1e-5, i
    assert float((logits - ws).abs().max()) <= 1e-5, i


@pytest.mark.parametrize("w", [96, 133])
def test_videos_of_different_lengths_equal_solo_runs(w):
    """A list of one-video Batches of 5, 2 and 7 frames, each with its own per-frame K and tracks, in one
    graph-replayed step: every video follows its solo ground-truth run (losses, poses, depth, logits).
    W = 133 takes the dense backward."""
    from flowmap_b200.overfit import FusedOverfitter
    frames, h, steps = [5, 2, 7], 40, 6
    cfg = _cfg(use_tracking=True, tracking_enable_after=0)
    vids = [_video_inputs(f, h, w, i) for i, f in enumerate(frames)]
    batches = [_batch(f, h, w, v[4].to(DEV)) for f, v in zip(frames, vids)]
    o = FusedOverfitter(cfg, batches, [v[2].to(DEV) for v in vids], [[t.to(DEV) for t in v[3]] for v in vids],
                        device=DEV)
    o._clock.base_seed = SEED
    with torch.no_grad():
        for m, v in zip(o.models, vids):
            m.backbone.depth.copy_(v[0])
            m.backbone.weights.copy_(v[1])
    o.use_cuda_graph = True
    k4 = o.intrinsics_k4()
    for i, v in enumerate(vids):  # every frame of every video reads its own K
        assert torch.equal(k4[i].cpu(), torch.stack((v[4][0, :, 0, 0], v[4][0, :, 1, 1], v[4][0, :, 0, 2],
                                                     v[4][0, :, 1, 2]), -1))
    losses, rts = _steps(o, steps)
    assert o.gradients()["focal"] is None
    for i, (f, v) in enumerate(zip(frames, vids)):
        _check_solo(i, [float(t[i]) for t in losses], [rt[i] for rt in rts],
                    o.models[i].backbone.depth.detach(), o.models[i].backbone.weights.detach(),
                    _solo(cfg, f, h, w, v, steps))


def test_tensor_batch_equals_solo_runs():
    """A (B, F) tensor batch whose batch.intrinsics (B, F, 3, 3) differ per video and frame."""
    from flowmap_b200.overfit import FusedOverfitter
    from flowmap_b200.types import Flows
    f, h, w, steps = 6, 40, 96, 6
    cfg = _cfg(use_tracking=True, tracking_enable_after=0)
    vids = [_video_inputs(f, h, w, i) for i in range(2)]
    batch = _batch(f, h, w, torch.cat([v[4] for v in vids]).to(DEV), b=2)
    flows = Flows(*(torch.cat([getattr(v[2], n) for v in vids]).to(DEV)
                    for n in ("forward", "backward", "forward_mask", "backward_mask")))
    o = FusedOverfitter(cfg, batch, flows, [[t.to(DEV) for t in v[3]] for v in vids], device=DEV)
    o._clock.base_seed = SEED
    with torch.no_grad():
        for m, v in zip(o.models, vids):
            m.backbone.depth.copy_(v[0])
            m.backbone.weights.copy_(v[1])
    o.use_cuda_graph = True
    losses, rts = _steps(o, steps)
    for i, v in enumerate(vids):
        _check_solo(i, [float(t[i]) for t in losses], [rt[i] for rt in rts],
                    o.models[i].backbone.depth.detach(), o.models[i].backbone.weights.detach(),
                    _solo(cfg, f, h, w, v, steps))


# ------------------------------------------------------------------------------------------- metrics log
def test_metrics_log():
    """The fx / fy error columns compare the frame means of the given K with themselves (<= 1e-6); the ATE
    column of the last update equals compute_ate on extrinsics()."""
    from flowmap_b200.ate import compute_ate
    depth, wparam, fl, kmat64, tracks = _zoom_case(seed=91)
    f, h, w = depth.shape
    g = torch.Generator().manual_seed(92)
    gt_ext = torch.eye(4).repeat(1, f, 1, 1)
    gt_ext[0, :, :3, 3] = torch.cumsum(0.3 * torch.randn(f, 3, generator=g), 0)
    o = _fused(_cfg(use_tracking=True, tracking_enable_after=0), _batch(f, h, w, kmat64.float().to(DEV),
                                                                        gt_ext.to(DEV)),
               _flows(fl), _device_tracks(tracks), depth, wparam, graph=True)
    o.enable_metrics_log(16)
    for _ in range(5):
        o.training_step()
    log = o.metrics_log()
    assert log["metrics/ate"].shape == (5,)
    assert float(log["train/intrinsics/fx_error"].abs().max()) <= 1e-6
    assert float(log["train/intrinsics/fy_error"].abs().max()) <= 1e-6
    ate, _, _ = compute_ate(gt_ext[0, :, :3, 3].to(DEV), o.extrinsics()[0, :, :3, 3])
    assert abs(float(log["metrics/ate"][-1]) - float(ate)) <= 1e-6 * max(1.0, float(ate)), (log["metrics/ate"], ate)


# ------------------------------------------------------------------------------------- network backbone
def test_network_backbone_halves_equal_per_op_path():
    """The `param` stand-in backbone of tools/backbone_step.py bound with model=: forward_phase /
    tracking_forward_phase / backward_phase give the per-op path's losses and d loss / d depths, d loss / d
    weights."""
    from dataclasses import make_dataclass
    from flowmap_b200.loss import LossFlowCfg, LossTrackingCfg, MappingHuberCfg, get_losses
    from flowmap_b200.model import ExtrinsicsProcrustesCfg, IntrinsicsGroundTruthCfg, Model, ModelCfg
    from flowmap_b200.overfit import FusedOverfitter
    from flowmap_b200.types import BackboneOutput
    import tools.backbone_step  # noqa: F401  (registers bench_param)
    f, h, w = 6, 40, 96
    _, _, flows, tracks, k = _video_inputs(f, h, w, 0)
    torch.manual_seed(0)
    bcfg = make_dataclass("StandInCfg", [("name", str)])("bench_param")
    model = Model(ModelCfg(bcfg, IntrinsicsGroundTruthCfg("ground_truth"), ExtrinsicsProcrustesCfg("procrustes", None, False),
                           True), f, (h, w)).to(DEV)
    batch, flows, trk = _batch(f, h, w, k.to(DEV)), flows.to(DEV), [t.to(DEV) for t in tracks]
    o = FusedOverfitter(_cfg(weight_sensitivity=0.0, use_tracking=True, tracking_enable_after=0), batch, flows, trk,
                        device=DEV, model=model)
    bo = model.backbone(batch, flows)
    d, wt = bo.depths.detach().float().contiguous(), bo.weights.detach().float().contiguous()
    lf = float(o.forward_phase(0, depth=d, weights=wt))
    lt = float(o.tracking_forward_phase())
    o.backward_phase(with_tracking=True)
    g = o.gradients()
    assert g["focal"] is None
    huber = MappingHuberCfg("huber", 0.01)
    losses = get_losses([LossFlowCfg(0, 1000.0, "flow", huber), LossTrackingCfg(0, 100.0, "tracking", huber)])
    dl, wl = d.clone().requires_grad_(True), wt.clone().requires_grad_(True)
    out = model._forward_materialized(batch, flows, 0, BackboneOutput(dl, wl))
    assert out.k_mode == "const"
    parts = [float(l.forward(batch, flows, trk, out, 0)) for l in losses]
    sum(l.forward(batch, flows, trk, out, 0) for l in losses).backward()
    print(f"flow {lf:.6e} / {parts[0]:.6e}, tracking {lt:.6e} / {parts[1]:.6e}, g_depth "
          f"{rel_l2(g['depth'].reshape(dl.shape), dl.grad):.1e}, g_weights {rel_l2(g['weights'].reshape(wl.shape), wl.grad):.1e}")
    assert abs(lf - parts[0]) <= 1e-5 * abs(parts[0]) and abs(lt - parts[1]) <= 1e-5 * abs(parts[1])
    assert rel_l2(g["depth"].reshape(dl.shape), dl.grad) <= 2e-5
    assert rel_l2(g["weights"].reshape(wl.shape), wl.grad) <= 2e-5


# ------------------------------------------------------------------------------ set_intrinsics, refusals
def test_set_intrinsics_keeps_captured_graphs():
    """set_intrinsics copies a new K into the step's buffer: a replayed graph then evaluates the new K, as a
    fresh optimiser on the same parameters and Adam state does."""
    f, h, w = 6, 40, 96
    depth, wl, flows, tracks, k = _video_inputs(f, h, w, 0)
    k2 = _video_inputs(f, h, w, 1)[4]
    cfg = _cfg(use_tracking=True, tracking_enable_after=0)
    mk = lambda kk: _fused(cfg, _batch(f, h, w, kk.to(DEV)), flows.to(DEV), [t.to(DEV) for t in tracks], depth, wl,  # noqa: E731
                           graph=True)
    o, ref = mk(k), mk(k2)
    for _ in range(3):
        o.training_step()
        ref.training_step()
    graph = o._graphs[next(iter(o._graphs))]
    o.set_intrinsics(k2.to(DEV))
    with torch.no_grad():  # the same parameters and Adam state for both from here on
        for src, dst in ((o.model.backbone.depth, ref.model.backbone.depth),
                         (o.model.backbone.weights, ref.model.backbone.weights)):
            dst.copy_(src)
        for s, r in zip(o._state, ref._state):
            if s is not None:
                r.copy_(s)
    a, b = o.training_step(), ref.training_step()
    assert o._graphs[next(iter(o._graphs))] is graph
    assert abs(float(a[0]) - float(b[0])) <= 1e-6 * abs(float(b[0])), (float(a[0]), float(b[0]))
    assert float((a[1] - b[1]).abs().max()) <= 2e-6


def test_refusals():
    from flowmap_b200.model import (BackboneExplicitDepthCfg, ExtrinsicsProcrustesCfg, IntrinsicsGroundTruthCfg,
                                    IntrinsicsRegressedCfg, Model, ModelCfg)
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    f, h, w = 5, 24, 32
    _, _, flows, tracks, k = _video_inputs(f, h, w, 0)
    flows = flows.to(DEV)
    cfg = _cfg()
    with pytest.raises(ValueError, match="intrinsics"):
        FusedOverfitter(cfg, _batch(f, h, w, None), flows, device=DEV)
    with pytest.raises(ValueError, match="intrinsics"):
        FusedOverfitter(cfg, _batch(f, h, w, k[:, :-1].to(DEV)), flows, device=DEV)
    bad = k.clone()
    bad[0, 1, 0, 0] = float("nan")
    with pytest.raises(ValueError, match="finite"):
        FusedOverfitter(cfg, _batch(f, h, w, bad.to(DEV)), flows, device=DEV)
    with pytest.raises(ValueError, match="intrinsics"):
        FusedOverfitter(cfg, [_batch(f, h, w, k.to(DEV)), _batch(f, h, w, None)], [flows, flows], device=DEV)

    def model(icfg):
        return Model(ModelCfg(BackboneExplicitDepthCfg("explicit_depth", 0.1, 100.0), icfg,
                              ExtrinsicsProcrustesCfg("procrustes", None, False), True), f, (h, w)).to(DEV)

    with pytest.raises(ValueError, match="match"):
        FusedOverfitter(cfg, _batch(f, h, w, k.to(DEV)), flows, device=DEV,
                        model=model(IntrinsicsRegressedCfg("regressed", 0.85)))
    with pytest.raises(ValueError, match="match"):
        FusedOverfitter(OverfitCfg(), _batch(f, h, w, k.to(DEV)), flows, device=DEV,
                        model=model(IntrinsicsGroundTruthCfg("ground_truth")))
    o = FusedOverfitter(cfg, _batch(f, h, w, k.to(DEV)), flows, device=DEV)
    with pytest.raises(ValueError, match="intrinsics"):
        o.set_intrinsics(k[:, :, :2].to(DEV))
    # the C ABI: constant intrinsics (g_k4 == NULL) with a focal parameter is refused
    from flowmap_b200._lib import lib
    a = o._args
    focal = torch.ones((), device=DEV)
    a.focal = focal.data_ptr()
    try:
        rc = lib().fm_overfit_step(ctypes.byref(a), torch.cuda.current_stream().cuda_stream)
    finally:
        a.focal = None
    assert rc != 0 and "constant intrinsics" in lib().fm_last_error().decode()
