"""Per-kernel profile of the fused step at the benchmark shape (150 x 360 x 640, iid flows, 30 track
segments x 1225 tracks), under torch.profiler with CUDA activities, in a run of its own:

  python tools/step_kernels.py [--steps N] [--out DIR]

Runs the full step (softmin + flow + tracking + Adam) and the flow-only step eagerly (the step graph is
not replayed, so every kernel is listed on its own stream), a few warm-up steps first.  Steps are
separated by a device synchronise.  Prints, per step kind:
  - the device time per step of every kernel (sum over its launches, mean over the profiled steps);
  - the busy time of the step (union of kernel intervals) and its span (first start to last end);
  - for the full step, the start and end of k_flow_lean and k_track_src relative to the step's first
    kernel, and how long the two overlap.
Writes step_kernels.json and the two Chrome traces under --out (default tools/_build/step_kernels);
`--trace FILE --steps N` tabulates a saved trace again."""
import argparse
import json
import re
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from flowmap_b200.overfit import FusedOverfitter, OverfitCfg  # noqa: E402
from flowmap_b200.types import Batch, Flows, Tracks  # noqa: E402

F, H, W = bench.F_, bench.H_, bench.W_


def make_overfitter(full, dev):
    inp = {k: v.to(dev).contiguous() for k, v in bench.synthetic_inputs(F, H, W, seed=0).items()}
    batch = Batch(torch.zeros(1, 1, 1, 1, 1, device=dev).expand(1, F, 3, H, W), torch.arange(F, device=dev)[None],
                  ["s"], ["d"])
    flows = Flows(inp["fwd"], inp["bwd"], inp["fmask"], inp["bmask"])
    tracks = [Tracks(xy, vis, s) for xy, vis, s in bench.synthetic_track_arrays(F, seed=0)] if full else None
    cfg = OverfitCfg(intrinsics="softmin", use_tracking=True) if full else OverfitCfg()
    o = FusedOverfitter(cfg, batch, flows, tracks, device=dev)
    with torch.no_grad():
        o.model.backbone.depth.copy_(inp["depth"])
        o.model.backbone.weights.copy_(inp["wparam"])
    o.global_step = bench.START_STEP
    if full:
        o.injected_indices = torch.randperm(H * W, generator=torch.Generator().manual_seed(3))[:8192].to(dev)
    o.use_cuda_graph = False
    return o


def short(name):
    n = name.replace("(anonymous namespace)::", "").replace("void ", "")
    return re.split(r"[<(]", n)[0].split("::")[-1]


def profile(full, steps, dev, out):
    o = make_overfitter(full, dev)
    for _ in range(5):
        o.training_step()
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for _ in range(steps):
            o.training_step()
            torch.cuda.synchronize()
    tag = "full" if full else "flow_only"
    trace = out / f"trace_{tag}.json"
    prof.export_chrome_trace(str(trace))
    return analyse(trace, steps, tag)


def analyse(trace, steps, tag):
    """Per-kernel table of a Chrome trace of `steps` identical steps (every step launches the same
    kernels, so the time-ordered kernel list splits into `steps` equal runs)."""
    ev = [e for e in json.loads(Path(trace).read_text())["traceEvents"]
          if e.get("cat") == "kernel" and "dur" in e]
    ev.sort(key=lambda e: e["ts"])
    if not ev or len(ev) % steps:
        raise SystemExit(f"step_kernels: {len(ev)} kernels do not split into {steps} equal steps")
    k = len(ev) // steps
    groups = [ev[i * k:(i + 1) * k] for i in range(steps)]
    per = {}
    busy, span, ov = [], [], []
    for g in groups:
        t0 = min(e["ts"] for e in g)
        span.append(max(e["ts"] + e["dur"] for e in g) - t0)
        iv = sorted((e["ts"], e["ts"] + e["dur"]) for e in g)
        tot, a, b = 0.0, iv[0][0], iv[0][1]
        for s, t in iv[1:]:
            if s > b:
                tot += b - a
                a, b = s, t
            else:
                b = max(b, t)
        busy.append(tot + b - a)
        for e in g:
            n = short(e["name"])
            per.setdefault(n, [0.0, 0])
            per[n][0] += e["dur"]
            per[n][1] += 1
        fl = [(e["ts"] - t0, e["ts"] + e["dur"] - t0) for e in g if short(e["name"]) == "k_flow_lean"]
        tr = [(e["ts"] - t0, e["ts"] + e["dur"] - t0) for e in g if short(e["name"]) == "k_track_src"]
        if fl and tr:
            f0, f1 = min(x[0] for x in fl), max(x[1] for x in fl)
            r0, r1 = min(x[0] for x in tr), max(x[1] for x in tr)
            ov.append({"k_flow_lean_us": [round(f0, 1), round(f1, 1)], "k_track_src_us": [round(r0, 1), round(r1, 1)],
                       "overlap_us": round(max(0.0, min(f1, r1) - max(f0, r0)), 1)})
    table = sorted(((n, v[0] / steps, v[1] / steps) for n, v in per.items()), key=lambda x: -x[1])
    print(f"== {tag} step: {steps} profiled steps, eager; busy {sum(busy) / steps / 1000:.3f} ms, "
          f"span {sum(span) / steps / 1000:.3f} ms per step")
    print(f"{'kernel':44s} {'us/step':>9s} {'launches':>9s}")
    for n, us, k in table:
        print(f"{n[:44]:44s} {us:9.1f} {k:9.1f}")
    for i, x in enumerate(ov):
        print(f"step {i}: {json.dumps(x)}")
    return {"kernels_us_per_step": {n: round(us, 2) for n, us, _ in table},
            "launches_per_step": {n: k for n, _, k in table},
            "busy_ms": sum(busy) / steps / 1000, "span_ms": sum(span) / steps / 1000, "flow_track_overlap": ov}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=str(ROOT / "tools" / "_build" / "step_kernels"))
    ap.add_argument("--trace", help="only tabulate an existing trace of --steps steps (no GPU needed)")
    args = ap.parse_args()
    if args.trace:
        analyse(args.trace, args.steps, Path(args.trace).stem)
        return
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    dev = torch.device("cuda:0")
    p = torch.cuda.get_device_properties(dev)
    res = {"device": p.name, "sm_count": p.multi_processor_count}
    print(f"device {p.name}, {p.multi_processor_count} SMs", flush=True)
    for full in (True, False):
        res["full" if full else "flow_only"] = profile(full, args.steps, dev, out)
        torch.cuda.empty_cache()
    (out / "step_kernels.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
