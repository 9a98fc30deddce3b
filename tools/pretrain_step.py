"""Times the reference's pretraining step (pretrain.py, model_wrapper_pretrain.py: Model.forward -> LossFlow ->
backward() -> torch.optim.Adam on the network) with the flow loss evaluated op by op and on the fused halves
(the packed layout of fm_overfit_step_videos), alternating the two in one process.  config/pretrain.yaml: a
batch of B videos of 8 frames cropped to 128 x 192, softmin intrinsics without a regression stage (8192
points, 60 candidates: a sweep on pair 0 of every video at every step), Procrustes on 1000 points, Huber flow
loss (weight 1000) normalised by one mask sum pooled over the batch, lr 5e-5.  A new batch and new Flows come
with every step, as from a loader (a fixed pool of pre-generated batches, cycled).  CUDA graphs are off:
autograd drives every step.

Two stand-in backbones (no pretrained weights are needed):
  * `param`: depth = 1e3 / (softplus(p + 2 v) + 0.1) and weights = sigmoid(100 q + v') from per-pixel
    parameters and the videos' first / second channels: its own cost is negligible, so the figures isolate
    the geometry;
  * `convnet`: tools/backbone_step.py's small CNN (64 feature channels, the reference's MLP weight head).

Usage: python tools/pretrain_step.py [--steps K] [--warmup W] [--rounds R] [--out file.json]
Prints one JSON line per (backbone, B) case."""
import argparse
import copy
import json
import sys
from pathlib import Path

import torch
import torch.nn.functional as F
from torch import nn

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from backbone_step import ConvBackbone, gpu_info, timed  # noqa: E402
from flowmap_b200.loss import LossFlowCfg, MappingHuberCfg, get_losses  # noqa: E402
from flowmap_b200.model import (BACKBONES, ExtrinsicsProcrustesCfg, IntrinsicsSoftminCfg, Model,  # noqa: E402
                                ModelCfg)
from flowmap_b200.types import BackboneOutput, Batch, Flows  # noqa: E402


class ParamBatchBackbone(nn.Module):
    def __init__(self, cfg, num_frames, image_shape):
        super().__init__()
        self.p = nn.Parameter(torch.full((num_frames, *image_shape), 10.0))
        self.q = nn.Parameter(0.01 * torch.randn(num_frames - 1, *image_shape))

    def forward(self, batch, flows):
        v = batch.videos
        return BackboneOutput(1e3 / (F.softplus(self.p + 2.0 * v[:, :, 0]) + 0.1),
                              (100.0 * self.q + v[:, 1:, 1] - 0.5).sigmoid())


BACKBONES["pretrain_param"], BACKBONES["pretrain_convnet"] = ParamBatchBackbone, ConvBackbone
POOL = 4  # distinct batches cycled through


def build(kind, b, f, h, w, dev):
    torch.manual_seed(0)
    from dataclasses import make_dataclass
    bcfg = make_dataclass("StandInCfg", [("name", str)])(f"pretrain_{kind}")
    icfg = IntrinsicsSoftminCfg("softmin", 8192, 0.5, 2.0, 60, None)
    model = Model(ModelCfg(bcfg, icfg, ExtrinsicsProcrustesCfg("procrustes", 1000, False), True), f, (h, w)).to(dev)
    losses = get_losses([LossFlowCfg(0, 1000.0, "flow", MappingHuberCfg("huber", 0.01))])
    data = []
    for i in range(POOL):
        g = torch.Generator().manual_seed(100 + i)
        low = torch.rand(b * f, 3, max(2, h // 16), max(2, w // 16), generator=g)
        videos = F.interpolate(low, (h, w), mode="bilinear", align_corners=False).reshape(b, f, 3, h, w)
        per = [bench.synthetic_inputs(f, h, w, seed=1000 * i + v) for v in range(b)]
        flows = Flows(*(torch.cat([p[k] for p in per]).to(dev) for k in ("fwd", "bwd", "fmask", "bmask")))
        data.append((Batch(videos.to(dev), torch.arange(f, device=dev)[None].expand(b, f), ["s"] * b, ["d"] * b),
                     flows))
    return model, losses, data


class Loop:
    """One run of the reference's pretraining step, on the next batch of the pool."""

    def __init__(self, model, losses, data, fused):
        self.model, self.losses, self.data, self.fused = model, losses, data, fused
        self.opt = torch.optim.Adam(model.parameters(), lr=5e-5)
        self.step_no = 0

    def step(self):
        batch, flows = self.data[self.step_no % len(self.data)]
        Model.fused_enabled = self.fused
        try:
            self.opt.zero_grad()
            out = self.model(batch, flows, self.step_no)
            total = sum(l.forward(batch, flows, None, out, self.step_no) for l in self.losses)
            total.backward()
            self.opt.step()
            self.step_no += 1
            return total.detach(), out
        finally:
            Model.fused_enabled = True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--cases", default="param:16,convnet:16,param:4,convnet:4,param:32,convnet:32")
    ap.add_argument("--shape", default="8x128x192")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pretrain_step: needs a CUDA device")
    dev = torch.device("cuda:0")
    f, h, w = (int(x) for x in args.shape.split("x"))
    info = gpu_info()
    rows = []
    for case in args.cases.split(","):
        kind, b = case.split(":")
        b = int(b)
        model, losses, data = build(kind, b, f, h, w, dev)
        loops = {name: Loop(copy.deepcopy(model), losses, data, name == "fused") for name in ("per_op", "fused")}
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
        row = {"backbone": kind, "batch": b, "shape": [f, h, w], "steps": args.steps, "rounds": args.rounds,
               "per_op_ms": round(med["per_op"], 3), "fused_ms": round(med["fused"], 3),
               "speedup": round(med["per_op"] / med["fused"], 3),
               "per_op_ms_all": [round(t, 3) for t in times["per_op"]],
               "fused_ms_all": [round(t, 3) for t in times["fused"]],
               "first_loss": first, "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 2), **info}
        print(json.dumps(row), flush=True)
        rows.append(row)
        del loops, model, data
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
