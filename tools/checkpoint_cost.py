"""Cost of snapshotting a run (FusedOverfitter.state_dict) on the C3 full step (150 x 360 x 640, softmin +
flow + tracking + Adam, replayed as a CUDA graph): rounds of 50 steps, alternately plain and with one
state_dict() at the start of the round whose tensors are then copied to pinned host memory on a side stream,
beside the round's steps.  A round's time ends when both the steps and the copy are done.  Prints the
snapshot's size, the medians and ranges, and the card name and power limit beside them.
Usage: python tools/checkpoint_cost.py [rounds]"""
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


def cuda_tensors(x):
    """The CUDA tensors of a state, in a fixed order."""
    if isinstance(x, torch.Tensor):
        return [x] if x.is_cuda else []
    if isinstance(x, dict):
        return [t for k in x for t in cuda_tensors(x[k])]
    if isinstance(x, (list, tuple)):
        return [t for v in x for t in cuda_tensors(v)]
    return []


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    inp = bench.synthetic_inputs(F, H, W, seed=0)
    batch = Batch(torch.zeros(1, 1, 1, 1, 1, device=dev).expand(1, F, 3, H, W), torch.arange(F, device=dev)[None],
                  ["s"], ["d"])
    flows = Flows(*(inp[n].to(dev) for n in ("fwd", "bwd", "fmask", "bmask")))
    tracks = [Tracks(xy, vis, s) for xy, vis, s in bench.synthetic_track_arrays(F, seed=0)]
    o = FusedOverfitter(OverfitCfg(intrinsics="softmin", use_tracking=True), batch, flows, tracks, device=dev)
    with torch.no_grad():
        o.model.backbone.depth.copy_(inp["depth"])
        o.model.backbone.weights.copy_(inp["wparam"])
    o.global_step = bench.START_STEP
    o.use_cuda_graph = True
    for _ in range(5):  # eager runs, capture, first replays
        o.training_step()
    host = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in cuda_tensors(o.state_dict())]
    nbytes = sum(t.numel() * t.element_size() for t in host)
    side = torch.cuda.Stream(device=dev)

    def timed(snapshot: bool) -> float:
        cur = torch.cuda.current_stream()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        state = None
        if snapshot:
            state = o.state_dict()
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                for h, t in zip(host, cuda_tensors(state)):
                    h.copy_(t, non_blocking=True)
        for _ in range(STEPS):
            o.training_step()
        if snapshot:
            cur.wait_stream(side)
        e1.record()
        torch.cuda.synchronize()
        del state
        return e0.elapsed_time(e1) / STEPS

    times = {"plain": [], "snapshot": []}
    for r in range(rounds):
        for name in (("plain", "snapshot") if r % 2 == 0 else ("snapshot", "plain")):
            times[name].append(timed(name == "snapshot"))
    print(f"snapshot: {nbytes / 1e9:.3f} GB in {len(host)} device tensors")
    for name in ("plain", "snapshot"):
        t = sorted(times[name])
        print(f"{name:8s}: median {t[len(t) // 2]:.4f} ms/step  min {t[0]:.4f}  max {t[-1]:.4f}  "
              f"({rounds} rounds x {STEPS} replayed C3 full steps)")
    p, s = sorted(times["plain"]), sorted(times["snapshot"])
    diff = s[rounds // 2] - p[rounds // 2]
    print(f"snapshot - plain (medians): {diff:+.4f} ms/step = {diff * STEPS:+.2f} ms per snapshot; "
          f"plain spread (max - min): {p[-1] - p[0]:.4f} ms/step")
    print(f"card: {card}")


if __name__ == "__main__":
    main()
