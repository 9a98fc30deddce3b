"""Times the reference-shaped loop of a network-backbone overfit (Model.forward -> flow [+ tracking] loss ->
backward() -> torch.optim.Adam) with the losses evaluated op by op and on the fused halves, alternating the
two in one process.  The reference's default overfit configuration: softmin intrinsics (8192 points, 60
candidates), Procrustes on 1000 points, Huber flow loss (weight 1000) [+ tracking loss (weight 100)], lr 3e-5,
timed from step 50 on (tracking on, softmin stage).  CUDA graphs are off: autograd drives every step.

Two stand-in backbones (no pretrained weights are needed):
  * `param`: depth = 1e3 / (softplus(p) + 0.1) and weights = sigmoid(100 q) from parameters: its own cost
    is negligible, so the figures isolate the geometry;
  * `convnet`: a small CNN with 64 feature channels and the reference's weight head, make_net([2C, 128, 64, 1])
    on the earlier frame's features grid-sampled at the backward flow beside the later frame's, ending in
    sigmoid().clip(min=1e-4); depths through the `original` mapping.

Usage: python tools/backbone_step.py [--steps K] [--warmup W] [--rounds R] [--out file.json]
Prints one JSON line per (backbone, shape, tracking) case."""
import argparse
import copy
import json
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F
from torch import nn

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from flowmap_b200.loss import LossFlowCfg, LossTrackingCfg, MappingHuberCfg, get_losses  # noqa: E402
from flowmap_b200.model import (BACKBONES, ExtrinsicsProcrustesCfg, IntrinsicsSoftminCfg, Model,  # noqa: E402
                                ModelCfg, RegressionCfg)
from flowmap_b200.types import BackboneOutput, Batch, Flows, Tracks  # noqa: E402


class ParamBackbone(nn.Module):
    def __init__(self, cfg, num_frames, image_shape):
        super().__init__()
        self.p = nn.Parameter(torch.full((num_frames, *image_shape), 10.0))
        self.q = nn.Parameter(0.01 * torch.randn(num_frames - 1, *image_shape))

    def forward(self, batch, flows):
        return BackboneOutput((1e3 / (F.softplus(self.p) + 0.1))[None], (100.0 * self.q).sigmoid()[None])


class ConvBackbone(nn.Module):
    C = 64

    def __init__(self, cfg, num_frames, image_shape):
        super().__init__()
        c = self.C
        self.features = nn.Sequential(nn.Conv2d(3, 32, 3, padding=1), nn.ReLU(), nn.Conv2d(32, c, 3, padding=1),
                                      nn.ReLU())
        self.depth_head = nn.Sequential(nn.Conv2d(c, 32, 3, padding=1), nn.ReLU(), nn.Conv2d(32, 1, 1))
        self.weight_head = nn.Sequential(nn.Linear(2 * c, 128), nn.ReLU(), nn.Linear(128, 64), nn.ReLU(),
                                         nn.Linear(64, 1))

    def forward(self, batch, flows):
        b, f, _, h, w = batch.videos.shape
        feat = self.features(batch.videos.reshape(b * f, 3, h, w))
        depths = (1e3 / (F.softplus(self.depth_head(feat)) + 0.1)).reshape(b, f, h, w)
        fe = (feat / 20).reshape(b, f, -1, h, w)
        ys, xs = torch.meshgrid(torch.arange(h, device=feat.device), torch.arange(w, device=feat.device), indexing="ij")
        xy = torch.stack(((xs + 0.5) / w, (ys + 0.5) / h), -1)
        grid = ((xy + flows.backward) * 2 - 1).reshape(b * (f - 1), h, w, 2)
        earlier = F.grid_sample(fe[:, :-1].reshape(b * (f - 1), -1, h, w), grid, mode="bilinear",
                                padding_mode="zeros", align_corners=False).reshape(b, f - 1, -1, h, w)
        pair = torch.cat((earlier, fe[:, 1:]), 2).permute(0, 1, 3, 4, 2)
        weights = self.weight_head(pair).sigmoid().clip(min=1e-4)[..., 0]
        return BackboneOutput(depths, weights)


BACKBONES["bench_param"], BACKBONES["bench_convnet"] = ParamBackbone, ConvBackbone


def build(kind, f, h, w, tracking, dev):
    torch.manual_seed(0)
    icfg = IntrinsicsSoftminCfg("softmin", 8192, 0.5, 2.0, 60, RegressionCfg(1000, 100))
    from dataclasses import make_dataclass
    bcfg = make_dataclass("StandInCfg", [("name", str)])(f"bench_{kind}")
    model = Model(ModelCfg(bcfg, icfg, ExtrinsicsProcrustesCfg("procrustes", 1000, False), True), f, (h, w)).to(dev)
    huber = MappingHuberCfg("huber", 0.01)
    lcfgs = [LossFlowCfg(0, 1000.0, "flow", huber)] + ([LossTrackingCfg(50, 100.0, "tracking", huber)] if tracking else [])
    inp = bench.synthetic_inputs(f, h, w, seed=0)
    g = torch.Generator().manual_seed(1)
    low = torch.rand(f, 3, max(2, h // 16), max(2, w // 16), generator=g)
    videos = F.interpolate(low, (h, w), mode="bilinear", align_corners=False)[None].to(dev)
    batch = Batch(videos, torch.arange(f, device=dev)[None], ["s"], ["d"])
    flows = Flows(*(inp[k].to(dev) for k in ("fwd", "bwd", "fmask", "bmask")))
    tracks = [Tracks(xy.to(dev), vis.to(dev), s) for xy, vis, s in bench.synthetic_track_arrays(f, seed=0)] \
        if tracking else None
    return model, get_losses(lcfgs), batch, flows, tracks


class Loop:
    """One run of the reference's training step (model_wrapper_overfit.py:51-73, 104-105)."""

    def __init__(self, model, losses, batch, flows, tracks, fused):
        self.model, self.losses, self.batch, self.flows, self.tracks, self.fused = model, losses, batch, flows, tracks, fused
        self.opt = torch.optim.Adam(model.parameters(), lr=3e-5)
        self.step_no = 50

    def step(self):
        Model.fused_enabled = self.fused
        try:
            self.opt.zero_grad()
            out = self.model(self.batch, self.flows, self.step_no)
            total = sum(l.forward(self.batch, self.flows, self.tracks, out, self.step_no) for l in self.losses)
            total.backward()
            self.opt.step()
            self.step_no += 1
            return total.detach(), out
        finally:
            Model.fused_enabled = True


def timed(loop, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        loop.step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20).stdout.strip().splitlines()
        info["power_limit_and_max_sm_clock"] = q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        info["power_limit_and_max_sm_clock"] = None
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--cases", default="param:150x360x640,param:41x160x224,convnet:41x160x224")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("backbone_step: needs a CUDA device")
    dev = torch.device("cuda:0")
    rows = []
    info = gpu_info()
    for case in args.cases.split(","):
        kind, shape = case.split(":")
        f, h, w = (int(x) for x in shape.split("x"))
        for tracking in (False, True):
            model, losses, batch, flows, tracks = build(kind, f, h, w, tracking, dev)
            loops = {name: Loop(copy.deepcopy(model), losses, batch, flows, tracks, name == "fused")
                     for name in ("per_op", "fused")}
            first = {name: float(lp.step()[0]) for name, lp in loops.items()}
            out = loops["fused"].step()[1]
            assert type(out).__name__ == "LazyModelOutput" and out.__dict__["_fused"].flow_done, "fused halves did not run"
            for lp in loops.values():
                for _ in range(args.warmup):
                    lp.step()
            times = {name: [] for name in loops}
            for _ in range(args.rounds):  # alternate the two evaluations
                for name, lp in loops.items():
                    times[name].append(timed(lp, args.steps))
            med = {name: sorted(t)[len(t) // 2] for name, t in times.items()}
            row = {"backbone": kind, "shape": [f, h, w], "tracking": tracking, "steps": args.steps,
                   "rounds": args.rounds, "per_op_ms": round(med["per_op"], 3), "fused_ms": round(med["fused"], 3),
                   "speedup": round(med["per_op"] / med["fused"], 3),
                   "per_op_ms_all": [round(t, 3) for t in times["per_op"]],
                   "fused_ms_all": [round(t, 3) for t in times["fused"]],
                   "first_loss": first, "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 2), **info}
            print(json.dumps(row), flush=True)
            rows.append(row)
            del loops, model
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
