"""Golden trajectory of one whole overfit run of the reference's default schedule, from the UNMODIFIED reference.

Run where a checkout of the reference is available (FLOWMAP_REFERENCE names its root):

    python tests/golden/make_golden_schedule.py          # both runs, side by side (~4 min on 8 cores)
    python tests/golden/make_golden_schedule.py --f64    # the float64 run only (schedule_f64.npz, the arbiter)
    python tests/golden/make_golden_schedule.py --f32    # the float32 run only (schedule.npz, the noise floor)

The schedule is the reference's configuration: overfit.yaml (max_steps 2000, lr 3e-5), loss/tracking.yaml
(enable_after 50) and model/intrinsics/softmin.yaml (8192 points, regression after_step 1000, window 100):
the tracking loss joins at step 50, the sweep's focal estimates of steps 900-999 fill the window, and at
step 1000 the focal length becomes an Adam parameter seeded with their mean.  The inputs are NOT stored:
they are tests/schedule_checks.schedule_inputs(SEED), which the GPU test regenerates.  The Lightning shell
is restated as in make_golden.py (model_wrapper_overfit.py:51-73, 104-105).  Lightning's validation steps
(every 50 steps) are skipped: they run the model forward without a gradient or an optimiser step, so they do
not change the optimisation state (the one at step 1000 repeats the same hand-over, to the same value).
The sweep's point sample is injected by patching torch.randperm with a fixed permutation: at 64 x 96 all
6144 pixels are sampled, so only the summation order depends on it.  The float64 run rebinds the name
torch.float32 before importing the reference (make_golden.py's recipe); it also checks, every 10th step,
that no predicted target of a visible track triple comes within schedule_checks.BORDER_MIN of the border of
[0,1)^2 (where validity could differ between precisions), and stores those distances.

Stored per run (about 0.4 MB): every step's total, flow and tracking loss and fx; the 100 window entries and
the hand-over seed; the poses at schedule_checks.POSE_STEPS (float32: their bar is 5e-5); at each of
CHECKPOINTS the parameters that step evaluates (before its update), the last of them the final parameters,
as schedule_checks.reduced_update.
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

REF = os.environ.get("FLOWMAP_REFERENCE", "reference")
OUT = Path(__file__).resolve().parent
ROOT = OUT.parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def run(f64: bool, threads: int):
    import schedule_checks as S
    torch.set_num_threads(threads)
    inp = S.schedule_inputs(S.SEED)  # drawn BEFORE any dtype games
    f, h, w = S.FRAMES, S.HEIGHT, S.WIDTH
    perm = torch.randperm(h * w, generator=torch.Generator().manual_seed(3))
    if f64:
        torch.float32 = torch.float64  # rebinding the name only (make_golden.py)
        torch.set_default_dtype(torch.float64)
    dtype = torch.float64 if f64 else torch.float32
    sys.path.insert(0, REF)
    os.environ["PYTHONDONTWRITEBYTECODE"] = "1"
    sys.dont_write_bytecode = True
    from flowmap.dataset.types import Batch
    from flowmap.flow.flow_predictor import Flows
    from flowmap.loss import get_losses
    from flowmap.loss.loss_flow import LossFlowCfg
    from flowmap.loss.loss_tracking import LossTrackingCfg
    from flowmap.loss.mapping.mapping_huber import MappingHuberCfg
    from flowmap.model.backbone.backbone_explicit_depth import BackboneExplicitDepthCfg
    from flowmap.model.extrinsics.extrinsics_procrustes import ExtrinsicsProcrustesCfg
    from flowmap.model.intrinsics.intrinsics_softmin import IntrinsicsSoftminCfg, RegressionCfg
    from flowmap.model.model import Model, ModelCfg
    from flowmap.tracking.track_predictor import Tracks

    # config/model/intrinsics/softmin.yaml, model/backbone/explicit_depth.yaml, loss/{flow,tracking}.yaml
    icfg = IntrinsicsSoftminCfg("softmin", 8192, 0.5, 2.0, 60, RegressionCfg(1000, 100))
    mcfg = ModelCfg(BackboneExplicitDepthCfg("explicit_depth", 0.1, 100.0), icfg,
                    ExtrinsicsProcrustesCfg("procrustes", None, False), True)
    model = Model(mcfg, f, (h, w))
    start = inp["depth"].to(dtype)
    with torch.no_grad():
        model.backbone.depth.copy_(start)
        model.backbone.weights.zero_()
    huber = MappingHuberCfg("huber", 0.01)
    losses = get_losses([LossFlowCfg(0, 1000.0, "flow", huber), LossTrackingCfg(50, 100.0, "tracking", huber)])
    tracks = [Tracks(t.xy.to(dtype), t.visibility, t.start_frame) for t in inp["tracks"]]
    batch = Batch(torch.zeros((1, 1, 1, 1, 1), dtype=dtype).expand(1, f, 3, h, w), torch.arange(f)[None], ["s"],
                  ["d"], extrinsics=inp["gt_extrinsics"].to(dtype), intrinsics=inp["gt_intrinsics"].to(dtype))
    fl = inp["flows"]
    flows = Flows(*(getattr(fl, n).to(dtype) for n in ("forward", "backward", "forward_mask", "backward_mask")))
    focal = model.intrinsics.intrinsics_regressed.focal_length

    real_randperm = torch.randperm
    torch.randperm = lambda n, **kw: perm
    opt = torch.optim.Adam(model.parameters(), lr=3e-5)  # model_wrapper_overfit.py:104-105
    rec = {k: [] for k in ("loss", "loss_flow", "loss_tracking", "fx", "extrinsics", "border_distance")}
    arrays = {}
    t0 = time.time()
    try:
        for s in range(S.STEPS + 1):
            if s in S.CHECKPOINTS:
                arrays.update(S.reduced_update(f"depth_s{s}", model.backbone.depth, start))
                arrays.update(S.reduced_update(f"wlog_s{s}", model.backbone.weights, torch.zeros(())))
            if s == S.STEPS:
                break
            opt.zero_grad()
            out = model(batch, flows, s)
            parts = [loss.forward(batch, flows, tracks, out, s) for loss in losses]
            total = sum(parts)
            if s == 1000:  # the focal length the hand-over seeded, before its first Adam step
                arrays["handover"] = np.float64(float(focal.detach()))
            total.backward()
            opt.step()
            total = total.detach()
            rec["loss"].append(float(total))
            rec["loss_flow"].append(float(parts[0].detach()))
            rec["loss_tracking"].append(float(parts[1].detach()))
            rec["fx"].append(float(out.intrinsics[0, 0, 0, 0].detach()))
            if s in S.POSE_STEPS:
                rec["extrinsics"].append(out.extrinsics.detach()[0, :, :3].float().numpy().copy())
            if s in S.BORDER_STEPS:
                with torch.no_grad():
                    d = S.border_distance(out.surfaces.detach().double(), out.extrinsics.detach().double(),
                                          out.intrinsics.detach().double(), inp["tracks"])
                rec["border_distance"].append(d)
                if f64:
                    assert d >= S.BORDER_MIN, f"step {s}: a predicted target is {d:.2e} from the border"
            if s % 100 == 0 or s == S.STEPS - 1:
                print(f"{'f64' if f64 else 'f32'} step {s}: loss {float(total):.6f} fx {rec['fx'][-1]:.6f} "
                      f"({time.time() - t0:.0f} s)", flush=True)
    finally:
        torch.randperm = real_randperm
    window = torch.stack(model.intrinsics.window).double()
    assert window.numel() == 100
    assert abs(float(window.mean()) - float(arrays["handover"])) <= (1e-12 if f64 else 1e-6)
    counts = [int(opt.state[p]["step"]) for p in (model.backbone.depth, model.backbone.weights, focal)]
    assert counts == [S.STEPS, S.STEPS, S.STEPS - 1000], counts
    path = OUT / f"schedule{'_f64' if f64 else ''}.npz"
    np.savez_compressed(
        path, frames=f, height=h, width=w, seed=S.SEED, steps=S.STEPS, stride=S.STRIDE,
        checkpoints=np.array(S.CHECKPOINTS), pose_steps=np.array(S.POSE_STEPS),
        border_steps=np.array(S.BORDER_STEPS), border_distance=np.array(rec["border_distance"]),
        loss=np.array(rec["loss"]), loss_flow=np.array(rec["loss_flow"]),
        loss_tracking=np.array(rec["loss_tracking"]), fx=np.array(rec["fx"]),
        extrinsics=np.stack(rec["extrinsics"]), window=window.numpy(), **arrays)
    print("wrote", path, f"{path.stat().st_size / 1e6:.2f} MB; smallest border distance "
          f"{min(rec['border_distance']):.3e}", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--f64", action="store_true", help="the float64 run only")
    ap.add_argument("--f32", action="store_true", help="the float32 run only")
    ap.add_argument("--threads", type=int, default=None)
    args = ap.parse_args()
    if args.f64 or args.f32:
        run(args.f64, args.threads or os.cpu_count() or 8)
        return
    # both runs at once, each in a process of its own (the float64 run rebinds torch.float32)
    threads = max(1, (os.cpu_count() or 8) // 2)
    procs = [subprocess.Popen([sys.executable, __file__, flag, "--threads", str(threads)])
             for flag in ("--f64", "--f32")]
    codes = [p.wait() for p in procs]
    if any(codes):
        sys.exit(f"make_golden_schedule: a run failed (exit codes {codes})")


if __name__ == "__main__":
    main()
