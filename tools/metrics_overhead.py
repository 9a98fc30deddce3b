"""Cost of the per-step metrics log (FusedOverfitter.enable_metrics_log) on the C3 full step
(150 x 360 x 640, softmin + flow + tracking + Adam, replayed as a CUDA graph): two optimisers on the
same inputs, one with the log off and one with it on, timed alternately in rounds of 50 steps.
Prints the card name and power limit beside the times.
Usage: python tools/metrics_overhead.py [rounds]"""
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from flowmap_b200.overfit import FusedOverfitter, OverfitCfg  # noqa: E402
from flowmap_b200.types import Batch, Flows, Tracks  # noqa: E402

F, H, W = bench.F_, bench.H_, bench.W_
STEPS = 50
dev = torch.device("cuda:0")
inp = bench.synthetic_inputs(F, H, W, seed=0)
g = torch.Generator().manual_seed(1)
ext = torch.eye(4).repeat(1, F, 1, 1)
ext[0, :, :3, 3] = torch.cumsum(0.03 * torch.randn(F, 3, generator=g), dim=0)  # a ground-truth path
k = torch.eye(3).repeat(1, F, 1, 1)
k[..., 0, 0], k[..., 1, 1], k[..., :2, 2] = 0.85 * (H * W) ** 0.5 / W, 0.85 * (H * W) ** 0.5 / H, 0.5
batch = Batch(torch.zeros(1, 1, 1, 1, 1, device=dev).expand(1, F, 3, H, W), torch.arange(F, device=dev)[None],
              ["s"], ["d"], extrinsics=ext, intrinsics=k)
flows = Flows(*(inp[n].to(dev) for n in ("fwd", "bwd", "fmask", "bmask")))
tracks = [Tracks(xy, vis, s) for xy, vis, s in bench.synthetic_track_arrays(F, seed=0)]


def make(log: bool):
    o = FusedOverfitter(OverfitCfg(intrinsics="softmin", use_tracking=True), batch, flows, tracks, device=dev)
    with torch.no_grad():
        o.model.backbone.depth.copy_(inp["depth"])
        o.model.backbone.weights.copy_(inp["wparam"])
    o.global_step = bench.START_STEP
    o.use_cuda_graph = True
    if log:
        o.enable_metrics_log(1024)
    for _ in range(5):  # eager runs, capture, first replays
        o.training_step()
    return o


def timed(o) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(STEPS):
        o.training_step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / STEPS


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    runs = {"off": make(False), "on": make(True)}
    times = {"off": [], "on": []}
    for r in range(rounds):
        for name in (("off", "on") if r % 2 == 0 else ("on", "off")):
            times[name].append(timed(runs[name]))
    for name in ("off", "on"):
        t = sorted(times[name])
        print(f"log {name:3s}: median {t[len(t) // 2]:.4f} ms/step  min {t[0]:.4f}  max {t[-1]:.4f}  "
              f"({rounds} rounds x {STEPS} replayed C3 full steps)")
    lo = sorted(times["off"])
    spread = lo[-1] - lo[0]
    diff = sorted(times["on"])[rounds // 2] - lo[rounds // 2]
    print(f"on - off (medians): {diff:+.4f} ms/step; off spread (max - min): {spread:.4f} ms")
    log = runs["on"].metrics_log()
    print("last row:", {n: round(float(v[-1]), 6) for n, v in log.items()})
    print(f"card: {card}")


if __name__ == "__main__":
    main()
