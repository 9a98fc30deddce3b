"""Times the reference-shaped loop with ground-truth intrinsics (model/intrinsics=ground_truth: K from the batch, a
different one for every frame, off-centre principal points), with the losses evaluated op by op
(Model.fused_enabled = False) and on the fused halves, alternating the two in one process.  CUDA graphs are off:
autograd drives every step.

  * `explicit`: the explicit-depth overfit (Overfitter: Model.forward -> flow + tracking loss -> backward() ->
    FusedAdam), all-pixel Procrustes, Huber losses (weights 1000 / 100), tracking on from step 0;
  * `param` / `convnet`: tools/backbone_step.py's stand-in backbones on one video, Procrustes on 1000 points, flow
    [+ tracking] loss, torch.optim.Adam (lr 3e-5);
  * `pretrain`: tools/pretrain_step.py's pretraining batch (`param` stand-in, B videos of 8 x 128 x 192,
    Procrustes on 1000 points, pooled flow loss, lr 5e-5) with a new batch, new Flows and a new K every step, and
    beside it the same batch with softmin intrinsics (the 60-candidate sweep of every video at every step).

Usage: python tools/gt_surface_step.py [--steps K] [--warmup W] [--rounds R] [--cases ...] [--out file.json]
Prints one JSON line per case, with the card's name and power limit."""
import argparse
import copy
import json
import sys
from dataclasses import make_dataclass, replace
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import bench  # noqa: E402
import backbone_step  # noqa: E402
import pretrain_step  # noqa: E402
from backbone_step import gpu_info, timed  # noqa: E402
from flowmap_b200.model import ExtrinsicsProcrustesCfg, IntrinsicsGroundTruthCfg, Model, ModelCfg  # noqa: E402
from flowmap_b200.overfit import OverfitCfg, Overfitter  # noqa: E402
from flowmap_b200.types import Batch, Flows, Tracks  # noqa: E402


def intrinsics(b, f, seed, dev):
    """(B, F, 3, 3) normalised K: a zoom per frame, principal points up to 0.12 off centre."""
    g = torch.Generator().manual_seed(seed)
    k = torch.zeros(b, f, 3, 3)
    k[..., 0, 0], k[..., 1, 1] = 0.6 + torch.rand(b, f, generator=g), 0.6 + torch.rand(b, f, generator=g)
    k[..., 0, 2], k[..., 1, 2] = 0.38 + 0.24 * torch.rand(b, f, generator=g), 0.38 + 0.24 * torch.rand(b, f, generator=g)
    k[..., 2, 2] = 1.0
    return k.to(dev)


class ExplicitLoop:
    """Overfitter.training_step on one path."""

    def __init__(self, f, h, w, fused, dev):
        inp = bench.synthetic_inputs(f, h, w, seed=0)
        batch = Batch(torch.zeros(1, f, 3, h, w, device=dev), torch.arange(f, device=dev)[None], ["s"], ["d"],
                      intrinsics=intrinsics(1, f, 1, dev))
        flows = Flows(*(inp[k].to(dev) for k in ("fwd", "bwd", "fmask", "bmask")))
        tracks = [Tracks(xy.to(dev), vis.to(dev), s) for xy, vis, s in bench.synthetic_track_arrays(f, seed=0)]
        cfg = OverfitCfg(intrinsics="ground_truth", use_tracking=True, tracking_enable_after=0)
        self.o = Overfitter(cfg, batch, flows, tracks, device=dev)
        with torch.no_grad():
            self.o.model.backbone.depth.copy_(1.0 + inp["depth"].to(dev))
            self.o.model.backbone.weights.copy_(inp["wparam"].to(dev))
        self.fused = fused

    def step(self):
        Model.fused_enabled = self.fused
        try:
            return self.o.training_step()
        finally:
            Model.fused_enabled = True


def network_one_video(kind, f, h, w, tracking, dev):
    model, losses, batch, flows, tracks = backbone_step.build(kind, f, h, w, tracking, dev)
    torch.manual_seed(0)
    bcfg = make_dataclass("StandInCfg", [("name", str)])(f"bench_{kind}")
    gt = Model(ModelCfg(bcfg, IntrinsicsGroundTruthCfg("ground_truth"), ExtrinsicsProcrustesCfg("procrustes", 1000, False),
                        True), f, (h, w)).to(dev)
    return gt, losses, replace(batch, intrinsics=intrinsics(1, f, 2, dev)), flows, tracks


def pretrain_models(b, f, h, w, dev):
    """The softmin pretraining model and data of tools/pretrain_step.py, and the ground-truth model with the same
    network weights on the same data, each batch with its own K."""
    soft, losses, data = pretrain_step.build("param", b, f, h, w, dev)
    bcfg = make_dataclass("StandInCfg", [("name", str)])("pretrain_param")
    gt = Model(ModelCfg(bcfg, IntrinsicsGroundTruthCfg("ground_truth"), ExtrinsicsProcrustesCfg("procrustes", 1000, False),
                        True), f, (h, w)).to(dev)
    gt.backbone.load_state_dict(soft.backbone.state_dict())
    gt_data = [(replace(bt, intrinsics=intrinsics(b, f, 10 + i, dev)), fl) for i, (bt, fl) in enumerate(data)]
    return soft, gt, losses, data, gt_data


def measure(loops, warmup, steps, rounds):
    first = {}
    for name, lp in loops.items():
        total, out = lp.step()
        first[name] = float(total.sum())
        if name.endswith("fused"):
            assert "_fused" in out.__dict__ and out.__dict__["_fused"].flow_done, f"{name}: not fused"
    for lp in loops.values():
        for _ in range(warmup):
            lp.step()
    times = {name: [] for name in loops}
    for _ in range(rounds):  # alternate the evaluations
        for name, lp in loops.items():
            times[name].append(timed(lp, steps))
    med = {name: sorted(t)[len(t) // 2] for name, t in times.items()}
    return first, med, times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--cases", default="explicit:150x360x640,explicit:41x160x224,param:41x160x224,"
                                       "convnet:41x160x224,pretrain:4,pretrain:16,pretrain:32")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gt_surface_step: needs a CUDA device")
    dev = torch.device("cuda:0")
    info = gpu_info()
    rows = []
    for case in args.cases.split(","):
        kind, shape = case.split(":")
        variants = [None]
        if kind == "explicit":
            f, h, w = (int(x) for x in shape.split("x"))
            loops = {name: ExplicitLoop(f, h, w, name == "fused", dev) for name in ("per_op", "fused")}
            variants = [("flow+tracking", loops)]
        elif kind in ("param", "convnet"):
            f, h, w = (int(x) for x in shape.split("x"))
            variants = []
            for tracking in (False, True):
                model, losses, batch, flows, tracks = network_one_video(kind, f, h, w, tracking, dev)
                loops = {name: backbone_step.Loop(copy.deepcopy(model), losses, batch, flows, tracks, name == "fused")
                         for name in ("per_op", "fused")}
                variants.append(("flow+tracking" if tracking else "flow", loops))
        else:
            b, (f, h, w) = int(shape), (8, 128, 192)
            soft, gt, losses, data, gt_data = pretrain_models(b, f, h, w, dev)
            loops = {"per_op": pretrain_step.Loop(copy.deepcopy(gt), losses, gt_data, False),
                     "fused": pretrain_step.Loop(copy.deepcopy(gt), losses, gt_data, True),
                     "softmin_per_op": pretrain_step.Loop(copy.deepcopy(soft), losses, data, False),
                     "softmin_fused": pretrain_step.Loop(copy.deepcopy(soft), losses, data, True)}
            variants = [(f"batch {b}", loops)]
        for label, loops in variants:
            first, med, times = measure(loops, args.warmup, args.steps, args.rounds)
            row = {"case": kind, "variant": label, "shape": [f, h, w], "steps": args.steps, "rounds": args.rounds,
                   **{f"{n}_ms": round(t, 3) for n, t in med.items()},
                   "speedup": round(med["per_op"] / med["fused"], 3),
                   **{f"{n}_ms_all": [round(t, 3) for t in ts] for n, ts in times.items()},
                   "first_loss": first, "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 2), **info}
            print(json.dumps(row), flush=True)
            rows.append(row)
        del variants, loops
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
