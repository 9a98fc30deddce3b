"""Videos of different lengths: ONE ragged FusedOverfitter (a list of one-video inputs) against the
eight solo runs one after the other and against the uniform batched step with every video padded to the
longest one (zero-mask frames), all replaying their steps as CUDA graphs:

  python tools/ragged_throughput.py [--out result.json] [--repeats 5]

Videos: LLFF's frame counts (20, 25, 26, 34, 41, 42, 55, 62: 305 frames) at its model shape 160 x 224,
synthetic content (bench.synthetic_inputs).  Configurations: the full loop of the softmin stage (focal
sweep + tracking + flow loss, bench.py's track layout, regression_after = None so that every step is the
same graph) and the regressed flow-only step.

Per config: warm-up (graph capture), then `repeats` rounds that time the three alternately with CUDA
events over at least `--seconds` of work each.  Reported: median and min / max of videos per second (one
video advanced by one step) and of frames per second (the frames of the real videos, 305 per step of
all eight; padding frames do not count).  The card's name and power limit are read in the same run."""
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
FRAMES = (20, 25, 26, 34, 41, 42, 55, 62)
H, W = 160, 224


def video(f, seed, pad_to=None):
    """(depth, logits, Flows (1, ...), tracks) of one synthetic video; pad_to: zero-mask frames appended."""
    i = bench.synthetic_inputs(f, H, W, seed=seed)
    depth, wl = 1.0 + i["depth"], i["wparam"]
    fl = [i["fwd"], i["bwd"], i["fmask"], i["bmask"]]
    if pad_to is not None and pad_to > f:
        extra = pad_to - f
        depth = torch.cat([depth, depth[-1:].expand(extra, -1, -1)])
        wl = torch.cat([wl, wl[-1:].expand(extra, -1, -1)])
        fl = [torch.cat([t, torch.zeros_like(t[:, :1]).expand(-1, extra, *t.shape[2:])], 1) for t in fl]
    tracks = [Tracks(xy, vis, st) for xy, vis, st in bench.synthetic_track_arrays(f, seed=seed)]
    return depth, wl, Flows(*(t.to(dev) for t in fl)), tracks


def init(o, videos):
    o._clock.base_seed = 1234
    with torch.no_grad():
        for m, (depth, wl, _, _) in zip(o.models, videos):
            m.backbone.depth.copy_(depth)
            m.backbone.weights.copy_(wl)
    o.use_cuda_graph = True
    return o


def batch_of(f, b=1):
    return Batch(torch.zeros(b, f, 3, H, W, device=dev), torch.arange(f, device=dev)[None].expand(b, f), ["s"] * b,
                 ["d"] * b)


def make_ragged(cfg):
    vids = [video(f, s) for s, f in enumerate(FRAMES)]
    tracks = [v[3] for v in vids] if cfg.use_tracking else None
    return init(FusedOverfitter(cfg, [batch_of(f) for f in FRAMES], [v[2] for v in vids], tracks, device=dev), vids)


def make_solos(cfg):
    out = []
    for s, f in enumerate(FRAMES):
        v = video(f, s)
        out.append(init(FusedOverfitter(cfg, batch_of(f), v[2], v[3] if cfg.use_tracking else None, device=dev), [v]))
    return out


def make_padded(cfg):
    F = max(FRAMES)
    vids = [video(f, s, pad_to=F) for s, f in enumerate(FRAMES)]
    flows = Flows(*(torch.cat([getattr(v[2], n) for v in vids]) for n in ("forward", "backward", "forward_mask",
                                                                          "backward_mask")))
    tracks = [v[3] for v in vids] if cfg.use_tracking else None
    return init(FusedOverfitter(cfg, batch_of(F, len(FRAMES)), flows, tracks, device=dev), vids)


def timed(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3


def measure(cfg, repeats, seconds):
    ragged, solos, padded = make_ragged(cfg), make_solos(cfg), make_padded(cfg)
    runs = {"ragged": ragged.training_step, "solo": lambda: [o.training_step() for o in solos],
            "padded": padded.training_step}
    for _ in range(4):  # two eager steps, the capture, one replay
        for fn in runs.values():
            fn()
    torch.cuda.synchronize()
    n = {k: max(3, int(seconds / max(timed(fn, 3) / 3, 1e-6))) for k, fn in runs.items()}
    vps = {k: [] for k in runs}
    for _ in range(repeats):  # alternate, so that all three see the same state of the shared card
        for k, fn in runs.items():
            vps[k].append(len(FRAMES) * n[k] / timed(fn, n[k]))
    del ragged, solos, padded
    torch.cuda.empty_cache()
    out = {"steps_per_window": n}
    for k, v in vps.items():
        fps = [x * sum(FRAMES) / len(FRAMES) for x in v]
        out[k] = {"videos_per_s": statistics.median(v), "videos_range": [min(v), max(v)],
                  "frames_per_s": statistics.median(fps), "frames_range": [min(fps), max(fps)]}
    out["ragged_over_solo"] = out["ragged"]["videos_per_s"] / out["solo"]["videos_per_s"]
    out["ragged_over_padded"] = out["ragged"]["videos_per_s"] / out["padded"]["videos_per_s"]
    return out


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
    rows = []
    for name, cfg in cfgs.items():
        r = measure(cfg, args.repeats, args.seconds)
        r.update({"frames": FRAMES, "shape": [H, W], "config": name})
        print(json.dumps(r), flush=True)
        rows.append(r)
    result = {"card": card, "rows": rows}
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
