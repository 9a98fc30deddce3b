"""Times B network-backbone overfits, each network on its own video, as ONE fused step
(flowmap_b200.fused.network_videos_step on the packed split halves) against B one-video network-bound fused
steps run in turn (Model.forward -> losses -> backward(), tools/backbone_step.py's loop).  The reference's
default overfit at the LLFF crop: F = 30 frames of 160 x 224, the `convnet` stand-in backbone of
tools/backbone_step.py, softmin intrinsics (8192 points, 60 candidates), Procrustes on 1000 points, Huber flow
loss (weight 1000) + tracking loss (weight 100), torch Adam (lr 3e-5) per network.  Two stages: the softmin
sweep (from step 50: tracking on) and the regressed focal length (from step 1001).

Reports scene-steps per second (B / step time) as the median of alternating rounds of >= 1 s each, with
[min, max], the card's name and power limit read in the same run, and, at the timed shape, each video's
losses and gradients of the batched step against its solo step (max relative L2 over videos and parameters).

Usage: python tools/network_videos_step.py [--bs 1,4,8,16] [--rounds 5] [--out file.json]"""
import argparse
import copy
import json
import statistics
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import backbone_step as bs  # noqa: E402
from flowmap_b200.fused import network_videos_step  # noqa: E402
from flowmap_b200.overfit import FusedOverfitter, OverfitCfg  # noqa: E402

F_, H_, W_ = 30, 160, 224


def scenes(B, stage, dev):
    """B (model, losses, batch, flows, tracks) of one shape, each network with its own weights."""
    out = []
    idx = torch.randperm(H_ * W_, generator=torch.Generator().manual_seed(3))[:8192].to(dev)
    for b in range(B):
        torch.manual_seed(b)
        model, losses, batch, flows, tracks = bs.build("convnet", F_, H_, W_, True, dev)
        torch.manual_seed(100 + b)
        for p in model.backbone.parameters():
            p.data.mul_(1.0 + 0.05 * torch.randn_like(p))
        if out:  # one configuration for all networks (build() makes a fresh backbone cfg type every call)
            model.cfg = out[0][0].cfg
        # one softmin point sample for the batched and the solo steps (the sweep's own draw is random)
        model.intrinsics.injected_indices = idx
        if stage == "regressed":
            model.intrinsics.intrinsics_regressed.focal_length.data.fill_(1.0)
        out.append((model, losses, batch, flows, tracks))
    return out


class Batched:
    def __init__(self, vids, step0):
        self.models = [v[0] for v in vids]
        self.vids = vids
        cfg = OverfitCfg(**self.models[0]._overfit_fields(), flow_weight=1000.0, flow_enable_after=0,
                         use_tracking=True, tracking_enable_after=50, tracking_weight=100.0, mapping="huber",
                         delta=0.01)
        self.eng = FusedOverfitter(cfg, [v[2] for v in vids], [v[3] for v in vids], [v[4] for v in vids],
                                   device=vids[0][3].forward.device, model=self.models)
        self.opts = [torch.optim.Adam(m.parameters(), lr=3e-5) for m in self.models]
        self.step_no = step0

    def run(self, update=True):
        for o in self.opts:
            o.zero_grad()
        outs = [m.backbone(v[2], v[3]) for m, v in zip(self.models, self.vids)]
        depths = torch.cat([o.depths[0] for o in outs])
        weights = torch.cat([o.weights[0] for o in outs])
        flow, track = network_videos_step(self.eng, depths, weights, self.step_no)
        (flow + track).sum().backward()
        if update:
            for o in self.opts:
                o.step()
            self.step_no += 1
        return flow.detach(), track.detach()

    def step(self):
        self.run()


class Solo:
    def __init__(self, vids, step0):
        self.loops = [bs.Loop(*v, fused=True) for v in vids]
        for lp in self.loops:
            lp.step_no = step0

    def step(self):
        for lp in self.loops:
            lp.step()


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300))


def _solo_grads(model, v, step0):
    """One solo network-bound fused step on a copy of `model`: (losses, d/d depths, d/d weights, parameter
    gradients)."""
    solo = copy.deepcopy(model)
    solo.zero_grad()
    out = solo(v[2], v[3], step0)
    d, w = out.depths, out.backward_correspondence_weights
    d.retain_grad()
    w.retain_grad()
    parts = [l.forward(v[2], v[3], v[4], out, step0) for l in v[1]]
    sum(parts).backward()
    return ([float(p.detach()) for p in parts], d.grad[0], w.grad[0],
            {n: p.grad.detach().clone() for n, p in solo.named_parameters() if p.grad is not None})


def compare(vids, step0, detail=False):
    """One step of the batched and of the solo surface from the same parameters: the largest relative error
    over the videos of the losses, of d loss / d depths and d loss / d weights (the fused step's own outputs), of
    each network's whole gradient (all its parameters as one vector) and of any one parameter's gradient; with
    the same errors of a second solo step against the first (the run-to-run noise of the solo step itself).
    `detail`: also every parameter's figures, with its gradient norm."""
    copies = [(copy.deepcopy(v[0]),) + tuple(v[1:]) for v in vids]
    bt = Batched(copies, step0)
    for o in bt.opts:
        o.zero_grad()
    outs = [m.backbone(v[2], v[3]) for m, v in zip(bt.models, bt.vids)]
    depths = torch.cat([o.depths[0] for o in outs])
    weights = torch.cat([o.weights[0] for o in outs])
    depths.retain_grad()
    weights.retain_grad()
    flow, track = network_videos_step(bt.eng, depths, weights, step0)
    (flow + track).sum().backward()
    worst = {"loss": 0.0, "d_depths": 0.0, "d_weights": 0.0, "all_params": 0.0, "all_params_solo_noise": 0.0,
             "param": 0.0, "param_solo_noise": 0.0}
    rows = []
    f0 = 0
    for b, v in enumerate(vids):
        f = v[2].videos.shape[1]
        ls, gd, gw, gp = _solo_grads(v[0], v, step0)
        _, gd2, gw2, gp2 = _solo_grads(v[0], v, step0)
        for got, want in zip((float(flow[b]), float(track[b])), ls):
            worst["loss"] = max(worst["loss"], abs(got - want) / max(abs(want), 1e-30))
        worst["d_depths"] = max(worst["d_depths"], _rel(depths.grad[f0:f0 + f], gd))
        worst["d_weights"] = max(worst["d_weights"], _rel(weights.grad[f0 - b:f0 - b + f - 1], gw))
        names = [n for n, _ in copies[b][0].named_parameters() if n in gp]
        got = dict(copies[b][0].named_parameters())
        flat = lambda g: torch.cat([g[n].reshape(-1).double() for n in names])  # noqa: E731
        worst["all_params"] = max(worst["all_params"], _rel(flat({n: got[n].grad for n in names}), flat(gp)))
        worst["all_params_solo_noise"] = max(worst["all_params_solo_noise"], _rel(flat(gp2), flat(gp)))
        for n, pb in copies[b][0].named_parameters():
            if n not in gp:
                continue
            e, noise = _rel(pb.grad, gp[n]), _rel(gp2[n], gp[n])
            worst["param"] = max(worst["param"], e)
            worst["param_solo_noise"] = max(worst["param_solo_noise"], noise)
            rows.append({"video": b, "param": n, "grad_norm": float(gp[n].double().norm()),
                         "rel_l2_vs_solo": e, "rel_l2_solo_vs_solo": noise})
        f0 += f
    del bt, copies
    return worst, rows if detail else None


def timed(loop, seconds):
    """Steps of `loop` for at least `seconds`; returns the mean step time in seconds (device-synchronised)."""
    torch.cuda.synchronize()
    t0, n = time.perf_counter(), 0
    while True:
        loop.step()
        n += 1
        if n % 2 == 0:
            torch.cuda.synchronize()
            if time.perf_counter() - t0 >= seconds:
                return (time.perf_counter() - t0) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bs", default="1,4,8,16")
    ap.add_argument("--stages", default="softmin,regressed")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--compare-only", action="store_true", help="the batched-vs-solo check alone, per parameter")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("network_videos_step: needs a CUDA device")
    dev = torch.device("cuda:0")
    info = bs.gpu_info()
    rows = []
    for stage in args.stages.split(","):
        step0 = 50 if stage == "softmin" else 1001
        for B in (int(x) for x in args.bs.split(",")):
            vids = scenes(B, stage, dev)
            worst, detail = compare(vids, step0, args.compare_only)
            if args.compare_only:
                print(json.dumps({"stage": stage, "B": B, **{f"max_rel_{k}": v for k, v in worst.items()}}), flush=True)
                for r in sorted(detail, key=lambda r: -r["rel_l2_vs_solo"])[:8]:
                    print(json.dumps(r), flush=True)
                continue
            loops = {"batched": Batched(vids, step0), "solo": Solo([(copy.deepcopy(v[0]),) + tuple(v[1:])
                                                                    for v in vids], step0)}
            for lp in loops.values():
                for _ in range(args.warmup):
                    lp.step()
            rates = {k: [] for k in loops}
            for _ in range(args.rounds):  # alternating rounds
                for k, lp in loops.items():
                    rates[k].append(B / timed(lp, args.seconds))
            row = {"stage": stage, "B": B, "F": F_, "H": H_, "W": W_, **info,
                   **{f"max_rel_{k}_vs_solo": v for k, v in worst.items()}}
            for k, r in rates.items():
                row[f"{k}_scene_steps_per_s"] = round(statistics.median(r), 2)
                row[f"{k}_range"] = [round(min(r), 2), round(max(r), 2)]
            row["speedup"] = round(row["batched_scene_steps_per_s"] / row["solo_scene_steps_per_s"], 3)
            print(json.dumps(row), flush=True)
            rows.append(row)
            del loops, vids
            torch.cuda.empty_cache()
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(rows, indent=1) + "\n")


if __name__ == "__main__":
    main()
