"""Times the overfit step with ground-truth intrinsics (a K per frame, no focal parameter) three ways, alternating
them in one process:

  (a) `fused_const_k`: FusedOverfitter(intrinsics="ground_truth"), graph-replayed: the constant-intrinsics step
      (focal = g_k4 = track_g_k4 = NULL), whose Procrustes backward and tracking sweep carry no K terms;
  (b) `fused_k_carrying`: the same optimiser with scratch g_k4 / track_g_k4 buffers, i.e. the K-carrying kernels
      whose intrinsics gradient nobody reads (the step before the constant-intrinsics mode existed);
  (c) `per_op`: Overfitter, the reference-shaped loop (Model(IntrinsicsGroundTruth) + LossFlow + LossTracking +
      FusedAdam), op by op.

Inputs: bench.synthetic_inputs / synthetic_track_arrays (flow + tracking loss from step 0) with a per-frame K that
zooms and moves its principal point over the video.  Step times are medians over alternating rounds of CUDA-event
timed windows that end in a device synchronisation.  A separate torch.profiler run (eager steps, no graphs) gives
the mean time per launch of k_distribute_window and k_track_src in modes (a) and (b).

Usage: python tools/gt_intrinsics_step.py [--steps K] [--warmup W] [--rounds R] [--shapes 150x360x640,41x160x224]
       [--out file.json]
Prints one JSON line per shape."""
import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from backbone_step import gpu_info  # noqa: E402
from flowmap_b200.overfit import FusedOverfitter, Overfitter, OverfitCfg  # noqa: E402
from flowmap_b200.types import Batch, Flows, Tracks  # noqa: E402


def zoom_intrinsics(f, h, w):
    """(1, f, 3, 3) normalised K: fx, fy grow 1.4x / 1.3x over the video, the principal point drifts."""
    s = (h * w) ** 0.5
    t = torch.linspace(0.0, 1.0, f)
    k = torch.zeros(1, f, 3, 3)
    k[0, :, 0, 0], k[0, :, 1, 1] = 0.8 * s / w * (1 + 0.4 * t), 0.9 * s / h * (1 + 0.3 * t)
    k[0, :, 0, 2], k[0, :, 1, 2], k[0, :, 2, 2] = 0.45 + 0.1 * t, 0.55 - 0.1 * t, 1.0
    return k


def build(f, h, w, dev):
    inp = bench.synthetic_inputs(f, h, w, seed=0)
    batch = Batch(torch.zeros(1, f, 3, h, w, device=dev), torch.arange(f, device=dev)[None], ["s"], ["d"],
                  intrinsics=zoom_intrinsics(f, h, w).to(dev))
    flows = Flows(*(inp[k].to(dev) for k in ("fwd", "bwd", "fmask", "bmask")))
    tracks = [Tracks(xy.to(dev), vis.to(dev), s) for xy, vis, s in bench.synthetic_track_arrays(f, seed=0)]
    cfg = OverfitCfg(intrinsics="ground_truth", use_tracking=True, tracking_enable_after=0)

    def init(o):
        with torch.no_grad():
            o.model.backbone.depth.copy_(inp["depth"].to(dev) + 1.0)
            o.model.backbone.weights.copy_(inp["wparam"].to(dev))
        return o

    def fused(k_carrying):
        o = init(FusedOverfitter(cfg, batch, flows, tracks, device=dev))
        if k_carrying:  # the K-carrying kernels: their intrinsics gradient goes to scratch buffers
            o._scratch = (torch.empty(f, 4, device=dev), torch.empty(f, 4, device=dev))
            o._args.g_k4, o._args.track_g_k4 = (t.data_ptr() for t in o._scratch)
        return o

    return {"fused_const_k": fused(False), "fused_k_carrying": fused(True),
            "per_op": init(Overfitter(cfg, batch, flows, tracks, device=dev))}


def timed(o, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        o.training_step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def kernel_times(o, steps):
    """Mean device time per launch (us) of the two kernels the constant-intrinsics mode specialises."""
    from torch.profiler import ProfilerActivity, profile
    o.use_cuda_graph = False
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            o.training_step()
        torch.cuda.synchronize()
    out = {}
    for name in ("k_distribute_window", "k_track_src"):
        ev = [e for e in prof.key_averages() if name in e.key]
        n = sum(e.count for e in ev)
        dev_us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in ev)
        out[name] = {"us_per_launch": round(dev_us / max(n, 1), 2), "launches": n,
                     "instantiations": sorted({e.key[:160] for e in ev})}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=5)
    ap.add_argument("--shapes", default="150x360x640,41x160x224")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gt_intrinsics_step: needs a CUDA device")
    dev = torch.device("cuda:0")
    info, rows = gpu_info(), []
    for shape in args.shapes.split(","):
        f, h, w = (int(x) for x in shape.split("x"))
        runs = build(f, h, w, dev)
        first = {name: float(o.training_step()[0]) for name, o in runs.items()}  # same parameters: same loss
        for name, o in runs.items():
            o.use_cuda_graph = name != "per_op"
            for _ in range(args.warmup):
                o.training_step()
        times = {name: [] for name in runs}
        for _ in range(args.rounds):  # alternate the three
            for name, o in runs.items():
                times[name].append(timed(o, args.steps))
        med = {name: sorted(t)[len(t) // 2] for name, t in times.items()}
        kern = {name: kernel_times(runs[name], args.profile_steps) for name in ("fused_const_k", "fused_k_carrying")}
        row = {"shape": [f, h, w], "tracking": True, "steps": args.steps, "rounds": args.rounds,
               **{f"{name}_ms": round(v, 3) for name, v in med.items()},
               "const_k_vs_k_carrying": round(med["fused_k_carrying"] / med["fused_const_k"], 3),
               "const_k_vs_per_op": round(med["per_op"] / med["fused_const_k"], 3),
               "all_ms": {name: [round(t, 3) for t in v] for name, v in times.items()},
               "first_loss": first, "kernels": kern,
               "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 2), **info}
        print(json.dumps(row), flush=True)
        rows.append(row)
        del runs
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
