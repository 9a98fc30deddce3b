"""Updates per second of ONE batched FusedOverfitter (B videos per step) against B one-video
FusedOverfitters run one after the other, both replaying their steps as CUDA graphs:

  python tools/batch_throughput.py [--out result.json] [--repeats 5]

Shapes: 30 x 180 x 240 (the reference's default model resolution, cropping.image_shape 43200) for
B = 1, 2, 4, 8, and 150 x 360 x 640 for B = 1, 2.  Configurations: the full loop of the softmin stage
(focal sweep + tracking + flow loss, bench.py's track layout, regression_after = None so that every
step is the same graph) and the regressed flow-only step.

Per (shape, config, B): warm-up (graph capture), then `repeats` rounds that time the batched and the
solo runs alternately with CUDA events over at least `--seconds` of work each.  Reported: median and
min / max of the updates per second (one update = one video advanced by one step) and the ratio of the
medians.  The card's name and power limit are read in the same run."""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from flowmap_b200.overfit import FusedOverfitter, OverfitCfg  # noqa: E402
from flowmap_b200.types import Batch, Flows, Tracks  # noqa: E402

dev = torch.device("cuda:0")


def make(cfg, f, h, w, seeds):
    b = len(seeds)
    inps = [bench.synthetic_inputs(f, h, w, seed=s) for s in seeds]
    batch = Batch(torch.zeros(b, f, 3, h, w, device=dev), torch.arange(f, device=dev)[None].expand(b, f),
                  ["s"] * b, ["d"] * b)
    flows = Flows(*(torch.cat([i[k] for i in inps]).to(dev) for k in ("fwd", "bwd", "fmask", "bmask")))
    tracks = None
    if cfg.use_tracking:  # the benchmark's track layout, a different sample per video
        tracks = [[Tracks(xy, vis, st) for xy, vis, st in bench.synthetic_track_arrays(f, seed=s)] for s in seeds]
        tracks = tracks[0] if b == 1 else tracks
    o = FusedOverfitter(cfg, batch, flows, tracks, device=dev)
    o._clock.base_seed = 1234
    with torch.no_grad():
        for m, i in zip(o.models, inps):
            m.backbone.depth.copy_(1.0 + i["depth"])
            m.backbone.weights.copy_(i["wparam"])
    o.use_cuda_graph = True
    return o


def timed(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3


def measure(cfg, f, h, w, B, repeats, seconds):
    batched = make(cfg, f, h, w, list(range(B)))
    solos = [make(cfg, f, h, w, [s]) for s in range(B)]
    run_b = batched.training_step
    run_s = lambda: [o.training_step() for o in solos]  # noqa: E731
    for _ in range(4):  # two eager steps, the capture, one replay
        run_b()
        run_s()
    torch.cuda.synchronize()
    n = max(3, int(seconds / max(timed(run_b, 3) / 3, 1e-6)))
    ns = max(3, int(seconds / max(timed(run_s, 3) / 3, 1e-6)))
    ub, us = [], []
    for _ in range(repeats):  # alternate, so that both see the same state of the shared card
        ub.append(B * n / timed(run_b, n))
        us.append(B * ns / timed(run_s, ns))
    del batched, solos
    torch.cuda.empty_cache()
    return {"batched_updates_per_s": statistics.median(ub), "batched_range": [min(ub), max(ub)],
            "solo_updates_per_s": statistics.median(us), "solo_range": [min(us), max(us)],
            "speedup": statistics.median(ub) / statistics.median(us), "steps_per_window": [n, ns]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=1.0)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    cfgs = {"softmin+tracking+flow": OverfitCfg(intrinsics="softmin", regression_after=None, use_tracking=True,
                                                tracking_enable_after=0),
            "regressed flow": OverfitCfg()}
    plan = [((30, 180, 240), (1, 2, 4, 8), ("softmin+tracking+flow", "regressed flow")),
            ((150, 360, 640), (1, 2), ("softmin+tracking+flow",))]
    rows = []
    for (f, h, w), bs, names in plan:
        for name in names:
            for B in bs:
                try:
                    r = measure(cfgs[name], f, h, w, B, args.repeats, args.seconds)
                except torch.cuda.OutOfMemoryError:
                    r = {"error": "out of memory"}
                    torch.cuda.empty_cache()
                r.update({"shape": [f, h, w], "config": name, "B": B})
                print(json.dumps(r), flush=True)
                rows.append(r)
    result = {"card": card, "rows": rows}
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
