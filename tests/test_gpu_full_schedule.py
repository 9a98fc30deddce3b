"""`-m gpu`: one whole overfit run of the reference's default schedule -- 2000 Adam steps, tracking from step 50,
the hand-over window over steps 900-999, the regressed focal length from step 1000 -- against the unmodified
reference's float64 run of it (tests/golden/make_golden_schedule.py, schedule_f64.npz), on the inputs of
schedule_checks.schedule_inputs.  Four runs of it: the production path (FusedOverfitter replaying one
CUDA graph per stage, with the metrics ring on), the reference-shaped surface (Model.forward -> losses ->
backward -> FusedAdam; once on the fused step's two halves, once op by op) and the packed step on a (2, F) batch
holding the scene twice.

Each bar is max(floor, 3 x the reference's own float32 error on that metric, worst so far in the run): the
float32 run (schedule.npz) is the noise floor a float32 implementation cannot beat.  The floors: 1e-4
relative on the losses and fx at every step, 5e-5 absolute on the poses at the stored steps, 1e-5 on each
window entry and the hand-over seed, 1e-3 on the per-frame (per-pair) relative L2 of the parameter updates
at the checkpoints, 1e-4 on the final depth and weight logits (relative L2 over the fixture's strided
subsample, and each frame's norm).  Besides the values, the
run must take the schedule's structure: which steps replay which graph, the device step clock, the window
size and Adam's per-parameter step counts."""
import math

import numpy as np
import pytest
import torch

import schedule_checks as S
from ate_oracle import trajectory_ate
from conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu

FLOORS = dict(loss=1e-4, fx=1e-4, pose=5e-5, window=1e-5, update=1e-3, final=1e-4, ate=1e-5, fx_error=1e-5)
TRACK_ON = 50  # loss/tracking.yaml: enable_after
HANDOVER, WINDOW = 1000, 100  # model/intrinsics/softmin.yaml: regression.after_step, regression.window
METRICS_RING = 256
F, H, W = S.FRAMES, S.HEIGHT, S.WIDTH
POSE_STEPS = set(S.POSE_STEPS)


def _load(f64):
    with np.load(GOLDEN / f"schedule{'_f64' if f64 else ''}.npz") as z:
        return {k: torch.as_tensor(z[k]) for k in z.files}


@pytest.fixture(scope="module")
def golden():
    return _load(False), _load(True)


@pytest.fixture(scope="module")
def inputs():
    return S.schedule_inputs(S.SEED)


def _cfg():
    from flowmap_b200.overfit import OverfitCfg
    return OverfitCfg(intrinsics="softmin", use_tracking=True)


def _cuda_inputs(inp, videos):
    """Batch (with the scene's poses and K), Flows and tracks of `videos` copies of the scene, on the GPU."""
    from flowmap_b200.types import Batch, Flows, Tracks
    dev = torch.device("cuda:0")
    rep = lambda t: t.float().to(dev).expand(videos, *t.shape[1:]).contiguous()  # noqa: E731
    batch = Batch(torch.zeros(1, 1, 1, 1, 1, device=dev).expand(videos, F, 3, H, W),
                  torch.arange(F, device=dev)[None].expand(videos, F), ["s"] * videos, ["d"] * videos,
                  extrinsics=rep(inp["gt_extrinsics"]), intrinsics=rep(inp["gt_intrinsics"]))
    fl = inp["flows"]
    flows = Flows(*(rep(getattr(fl, n)) for n in ("forward", "backward", "forward_mask", "backward_mask")))
    tracks = [Tracks(t.xy.float().to(dev), t.visibility.to(dev), t.start_frame) for t in inp["tracks"]]
    return batch, flows, (tracks if videos == 1 else [tracks] * videos)


class Trace:
    """What one run hands back, per video (leading dimension): every step's losses and fx, the poses at the stored
    steps, the window, the focal length the hand-over seeded and the parameters at the checkpoints, the last of
    them the final ones.  Recorded as device tensors, stacked into CPU float64 by finish()."""

    def __init__(self, videos):
        self.videos = videos
        self.loss, self.loss_flow, self.loss_tracking, self.fx, self.poses = [], [], [], [], []
        self.depth, self.wlog = {}, {}

    def step(self, s, total, fx, poses, flow=None, tracking=None):
        """After step s: its total loss, fx, [flow and tracking loss,] and at the stored steps its poses (callable)."""
        v = self.videos
        self.loss.append(total.detach().reshape(v).clone())
        self.fx.append(fx.detach().reshape(v).clone())
        if flow is not None:
            self.loss_flow.append(flow.reshape(v).clone())
            self.loss_tracking.append(tracking.reshape(v).clone())
        if s in POSE_STEPS:
            self.poses.append(poses().detach()[..., :3, :].reshape(v, F, 3, 4).clone())

    def checkpoint(self, s, depth, wlog):
        """Before step s: at the checkpoints, the parameters it is about to evaluate (s = STEPS: the final ones)."""
        if s in S.CHECKPOINTS:
            self.depth[s] = depth.detach().reshape(self.videos, F, H, W).clone()
            self.wlog[s] = wlog.detach().reshape(self.videos, F - 1, H, W).clone()

    def finish(self, window):
        v = self.videos
        st = lambda xs: torch.stack(xs, 1).double().cpu() if xs else None  # noqa: E731
        self.loss, self.loss_flow, self.loss_tracking, self.fx = (st(x) for x in (self.loss, self.loss_flow,
                                                                                self.loss_tracking, self.fx))
        self.poses = st(self.poses)
        self.window = torch.stack([x.detach().reshape(v) for x in window], 1).double().cpu() if window else \
            torch.zeros(v, 0, dtype=torch.float64)
        # the focal length step 1000 evaluated: the hand-over's seed, before its first Adam step
        self.handover = self.fx[:, HANDOVER] * W / math.sqrt(H * W)
        self.depth = {s: t.double().cpu() for s, t in self.depth.items()}
        self.wlog = {s: t.double().cpu() for s, t in self.wlog.items()}
        return self


def _run_fused(inp, videos, spy=None):
    """The production path: FusedOverfitter, CUDA graphs on, step-clock sampling; with one video the metrics ring
    (256 rows: it wraps).  `spy(key, replayed)` sees every step's graph key and whether it replayed a graph."""
    from flowmap_b200.overfit import FusedOverfitter
    batch, flows, tracks = _cuda_inputs(inp, videos)
    o = FusedOverfitter(_cfg(), batch, flows, tracks, device="cuda:0")
    o.use_cuda_graph = True
    start = inp["depth"].float().cuda()
    with torch.no_grad():
        for m in o.models:
            m.backbone.depth.copy_(start)
            m.backbone.weights.zero_()
    if videos == 1:
        o.enable_metrics_log(METRICS_RING)
    if spy is not None:
        run_body = o._run_body

        def watched(key, graphable, body, ticks_focal):
            spy(key, graphable and o._eager_runs.get(key, 0) >= 2)
            return run_body(key, graphable, body, ticks_focal)
        o._run_body = watched
    tr = Trace(videos)
    for s in range(S.STEPS):
        tr.checkpoint(s, o._depth, o._wlog)
        total, _ = o.training_step()
        tr.step(s, total, o.intrinsics_k4()[..., 0, 0], o.extrinsics, o._loss, o._track_loss)
    tr.checkpoint(S.STEPS, o._depth, o._wlog)
    return o, tr.finish(o.window)


def _run_surface(inp, per_op):
    """The reference-shaped surface: Overfitter (Model.forward -> LossFlow / LossTracking -> backward -> FusedAdam).
    Its losses run the two halves of the fused step, whose window is FusedOverfitter.forward_phase's; per_op
    (Model.fused_enabled off) evaluates op by op under autograd instead, with IntrinsicsSoftmin's own window."""
    from flowmap_b200.overfit import Overfitter
    batch, flows, tracks = _cuda_inputs(inp, 1)
    o = Overfitter(_cfg(), batch, flows, tracks, device="cuda:0")
    o.model.fused_enabled = not per_op
    bb = o.model.backbone
    with torch.no_grad():
        bb.depth.copy_(inp["depth"].float().cuda())
        bb.weights.zero_()
    tr = Trace(1)
    for s in range(S.STEPS):
        tr.checkpoint(s, bb.depth, bb.weights)
        total, out = o.training_step()
        tr.step(s, total, out.intrinsics[0, 0, 0, 0], lambda: out.extrinsics[0])
    tr.checkpoint(S.STEPS, bb.depth, bb.weights)
    return o, tr.finish(o.model.intrinsics.window)


class Checks:
    """Measured errors against their bars and structural expectations; every one is printed, then the failures
    are asserted together (a schedule bug shows in what it breaks, not only in the first thing it breaks)."""

    def __init__(self, label):
        self.label, self.rows, self.failed = label, [], []

    def add(self, name, err, bar, where=None):
        """err, bar: equal-shape tensors (or floats); `where`: the step / index of each entry."""
        err, bar = torch.as_tensor(err, dtype=torch.float64).flatten(), torch.as_tensor(bar, dtype=torch.float64).flatten()
        where = torch.arange(err.numel()) if where is None else torch.as_tensor(where).flatten()
        ratio = err / bar
        i = int(torch.nan_to_num(ratio, nan=float("inf")).argmax())
        self.rows.append(f"{name}: worst error {float(err.max()):.3e}, worst error / bar {float(ratio[i]):.3f} "
                         f"(at {int(where[i])}: {float(err[i]):.3e} vs bar {float(bar[i]):.3e})")
        if not bool((err <= bar).all()):
            bad = where[~(err <= bar)]
            self.failed.append(f"{name} at {bad[:8].tolist()}{' ...' if bad.numel() > 8 else ''}")

    def expect(self, name, got, want):
        self.rows.append(f"{name}: {'as expected' if got == want else f'{got}, expected {want}'}")
        if got != want:
            self.failed.append(f"{name}: {got}, expected {want}")

    def done(self):
        print(f"\n{self.label}, against the reference's float64 run:\n  " + "\n  ".join(self.rows))
        assert not self.failed, f"{self.label}: " + "; ".join(self.failed)


def _bar(err32, floor, dim=-1):
    """max(floor, 3 x the float32 reference's error, worst so far along `dim`)."""
    return torch.clamp(3.0 * torch.cummax(err32, dim=dim).values, min=floor)


def _upd_errors(sub, norms, g, key):
    """Worst per-frame (per-pair) relative L2 of an update's strided subsample `sub` and worst relative error of its
    per-frame norms `norms`, against the fixture `g` at checkpoint `key` (schedule_checks.reduced_update)."""
    frame = torch.arange(0, len(norms) * H * W, S.STRIDE) // (H * W)
    ref, n_ref = g[f"{key}_upd_sub"].double(), g[f"{key}_upd_norms"].double()
    per_frame = max(rel_l2(sub[frame == j], ref[frame == j]) for j in range(len(norms)))
    return per_frame, float(((norms.double() - n_ref).abs() / n_ref).max())


def _final_error(sub, norms, start_sub, g, key):
    """Relative L2 of a parameter's values over its strided subsample `sub` (the fixture keeps start + update
    there), or the worst relative error of its per-frame norms `norms`, whichever is larger."""
    ref = start_sub + g[f"{key}_upd_sub"].double()
    n_ref = g[f"{key}_norms"].double()
    return max(rel_l2(sub, ref), float(((norms.double() - n_ref).abs() / n_ref).max()))


def _compare(c, tr, v, g32, g64, start, with_parts):
    """Video v of a run against the fixture: every metric of the module docstring, into Checks c."""
    rel = lambda ours, ref: (ours - ref).abs() / ref.abs()  # noqa: E731
    steps = torch.arange(S.STEPS)
    p = f"video {v}: " if tr.videos > 1 else ""
    for name, key in (("total loss", "loss"),) + ((("flow loss", "loss_flow"), ("tracking loss", "loss_tracking"))
                                                     if with_parts else ()):
        ours = getattr(tr, key)[v]
        keep = steps >= TRACK_ON if key == "loss_tracking" else steps >= 0  # the tracking loss is 0 before
        e, e32 = rel(ours, g64[key])[keep], rel(g32[key], g64[key])[keep]
        c.add(f"{p}{name} (relative, every step)", e, _bar(e32, FLOORS["loss"], 0), steps[keep])
    if with_parts:
        c.expect(f"{p}tracking loss before step {TRACK_ON}", bool((tr.loss_tracking[v][:TRACK_ON] == 0).all()), True)
    c.add(f"{p}fx (relative, every step)", rel(tr.fx[v], g64["fx"]), _bar(rel(g32["fx"], g64["fx"]), FLOORS["fx"], 0))
    pe = (tr.poses[v] - g64["extrinsics"]).abs().flatten(1).max(dim=1).values
    pe32 = (g32["extrinsics"] - g64["extrinsics"]).abs().flatten(1).max(dim=1).values
    c.add(f"{p}poses (absolute, stored steps)", pe, _bar(pe32, FLOORS["pose"], 0), g64["pose_steps"])
    we32 = (g32["window"] - g64["window"]).abs()
    c.expect(f"{p}window entries", tr.window.shape[1], WINDOW)
    if tr.window.shape[1] == WINDOW:
        c.add(f"{p}window entries (absolute)", (tr.window[v] - g64["window"]).abs(), _bar(we32, FLOORS["window"], 0),
              torch.arange(HANDOVER - WINDOW, HANDOVER))
    he32 = max(float(we32.max()), abs(float(g32["handover"] - g64["handover"])))
    c.add(f"{p}hand-over seed (absolute)", abs(float(tr.handover[v] - g64["handover"])),
          max(FLOORS["window"], 3 * he32), [HANDOVER])
    worst32 = {"depth": 0.0, "wlog": 0.0}  # per parameter, worst so far
    for s in S.CHECKPOINTS:
        for name, label, ours, st in (("depth", "depth", tr.depth[s][v], start),
                                      ("wlog", "weight logits", tr.wlog[s][v], torch.zeros(()))):
            key, upd = f"{name}_s{s}", ours - st
            err = _upd_errors(upd.flatten()[::S.STRIDE], upd.flatten(1).norm(dim=1), g64, key)
            worst32[name] = max(worst32[name], *_upd_errors(g32[f"{key}_upd_sub"].double(), g32[f"{key}_upd_norms"],
                                                            g64, key))
            bar = max(FLOORS["update"], 3 * worst32[name])
            c.add(f"{p}{label} update at step {s} (per-frame relative L2 / norm)", err, [bar, bar], [s, s])
    for name, label, st in (("depth", "final depth", start), ("wlog", "final weight logits", torch.zeros(()))):
        key = f"{name}_s{S.STEPS}"
        ours = tr.depth[S.STEPS][v] if name == "depth" else tr.wlog[S.STEPS][v]
        st_sub = st.expand_as(ours).flatten()[::S.STRIDE]
        err = _final_error(ours.flatten()[::S.STRIDE], ours.flatten(1).norm(dim=1), st_sub, g64, key)
        err32 = _final_error(st_sub + g32[f"{key}_upd_sub"].double(), g32[f"{key}_norms"], st_sub, g64, key)
        c.add(f"{p}{label} (relative L2 / per-frame norm)", err, max(FLOORS["final"], 3 * err32), [S.STEPS])


GRAPHS = [(False, True, True), (True, False, True), (True, True, True)]  # (track_on, sweep, flow_on)


def test_production_run_replays_one_graph_per_stage_and_follows_the_reference(golden, inputs):
    """Run 1: FusedOverfitter with CUDA graphs over the whole schedule, the metrics ring wrapping."""
    g32, g64 = golden
    seen = []
    o, tr = _run_fused(inputs, 1, spy=lambda key, replayed: seen.append((key, replayed)))
    c = Checks("production path (graphs)")
    # structure: one graph per stage, captured on the stage's third step; the window steps run eagerly
    c.expect("captured graphs", sorted(o._graphs), GRAPHS)
    c.expect("eager steps", [s for s, (_, replayed) in enumerate(seen) if not replayed],
             [0, 1, TRACK_ON, TRACK_ON + 1, *range(HANDOVER - WINDOW, HANDOVER + 2)])
    c.expect("graph keys at the switches", [seen[s][0] for s in (TRACK_ON - 1, TRACK_ON, HANDOVER - 1, HANDOVER)],
             [(False, True, True), (True, True, True), (True, True, True), (True, False, True)])
    c.expect("device step clock", o._clock.buf.view(torch.int32)[:2].tolist(), [S.STEPS, S.STEPS - HANDOVER])
    _compare(c, tr, 0, g32, g64, inputs["depth"], with_parts=True)
    # the metrics ring's last 256 rows: the ATE and fx error of what each step evaluated, against the fixture's
    log = o.metrics_log()
    first = S.STEPS - METRICS_RING
    c.expect("metrics ring rows", tuple(log["metrics/ate"].shape), (METRICS_RING,))
    gt = inputs["gt_extrinsics"][0, :, :3, 3]
    rows, errs, bars, worst32 = [], [], [], 0.0
    for i, s in enumerate(S.POSE_STEPS):
        a64 = float(trajectory_ate(gt, g64["extrinsics"][i][:, :3, 3].double())[0])
        a32 = float(trajectory_ate(gt, g32["extrinsics"][i][:, :3, 3].double())[0])
        worst32 = max(worst32, abs(a32 - a64))
        if s >= first:
            rows.append(s)
            errs.append(abs(float(log["metrics/ate"][s - first]) - a64))
            bars.append(max(FLOORS["ate"], 3 * worst32))
    c.add("metrics ring: metrics/ate (absolute, stored-pose steps)", errs, bars, rows)
    fx_gt = float(inputs["gt_intrinsics"][0, :, 0, 0].mean())
    ref = (fx_gt - g64["fx"][first:]).abs()
    e32 = ((fx_gt - g32["fx"]).abs() - (fx_gt - g64["fx"]).abs()).abs()
    c.add("metrics ring: train/intrinsics/fx_error (absolute, every step)",
          (log["train/intrinsics/fx_error"].double() - ref).abs(), _bar(e32, FLOORS["fx_error"], 0)[first:],
          torch.arange(first, S.STEPS))
    c.done()


@pytest.mark.parametrize("per_op", [False, True], ids=["fused_halves", "per_op"])
def test_reference_shaped_surface_follows_the_reference(golden, inputs, per_op):
    """Run 2: Overfitter (Model.forward -> losses -> backward() -> FusedAdam) over the whole schedule, on the fused
    halves and op by op."""
    g32, g64 = golden
    o, tr = _run_surface(inputs, per_op)
    c = Checks(f"reference-shaped surface ({'per op' if per_op else 'fused halves'})")
    params = o.optimizer.params
    steps = {name: o.optimizer.steps[next(i for i, p in enumerate(params) if p is t)]
             for name, t in (("depth", o.model.backbone.depth), ("weights", o.model.backbone.weights),
                             ("focal", o.model.intrinsics.intrinsics_regressed.focal_length))}
    c.expect("Adam step counts", steps, {"depth": S.STEPS, "weights": S.STEPS, "focal": S.STEPS - HANDOVER})
    _compare(c, tr, 0, g32, g64, inputs["depth"], with_parts=False)
    c.done()


def test_packed_two_video_step_follows_the_reference(golden, inputs):
    """Run 3: the packed step on a (2, F) tensor batch holding the scene twice; each video against the fixture."""
    g32, g64 = golden
    o, tr = _run_fused(inputs, 2)
    c = Checks("packed (2, F) batch")
    c.expect("captured graphs", sorted(o._graphs), GRAPHS)
    c.expect("device step clock", o._clock.buf.view(torch.int32)[:2].tolist(), [S.STEPS, S.STEPS - HANDOVER])
    for v in range(2):
        _compare(c, tr, v, g32, g64, inputs["depth"], with_parts=True)
    c.done()
