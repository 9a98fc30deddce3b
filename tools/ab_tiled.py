"""A/B on an H100: the splat-plan path (k_moments_tiled / k_backward_tiled, TMA-staged windows,
gather-form backward) against the global-RED path (k_moments / k_distribute).

1. parity at several shapes / flow fields through the op-level C ABI: poses, depth / weight
   gradients, focal gradient;
2. fused-step trajectories with and without the plan;
3. per-launch times of the ops and of the fused step at 150 x 360 x 640.

Usage: python tools/ab_tiled.py [--quick | --tiny]     (writes tools/_build/ab_tiled.json)"""
import json
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from flowmap_b200 import ops  # noqa: E402
from flowmap_b200._lib import lib  # noqa: E402
from flowmap_b200.overfit import FusedOverfitter, OverfitCfg  # noqa: E402
from flowmap_b200.types import Batch, Flows, Tracks  # noqa: E402

dev = torch.device("cuda:0")
P = lambda x: None if x is None else x.data_ptr()  # noqa: E731


def rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def make_case(f, h, w, kind, seed=0):
    inp = bench.synthetic_inputs(f, h, w, seed=seed)
    g = torch.Generator().manual_seed(seed + 100)
    if kind == "shift":      # large coherent motion
        inp["bwd"] = inp["bwd"] + torch.tensor([0.2, -0.1])
    elif kind == "leave":    # taps leave the frame: border pile-up
        inp["bwd"] = inp["bwd"] + torch.tensor([0.3, 0.0])
    elif kind == "outliers":  # 5 % of the flows far outside any window
        m = torch.rand(1, f - 1, h, w, generator=g) < 0.05
        inp["bwd"][m] = 0.5 * torch.randn(int(m.sum()), 2, generator=g)
    elif kind == "smooth":
        coarse = 0.01 * torch.randn(f - 1, 2, (h + 15) // 16 + 1, (w + 15) // 16 + 1, generator=g)
        up = torch.nn.functional.interpolate(coarse, size=(h, w), mode="bilinear", align_corners=True)
        inp["bwd"] = up.permute(0, 2, 3, 1)[None].contiguous()
    return {k: v.to(dev).contiguous() for k, v in inp.items()}


def run_ops(c, f, h, w, plan):
    """fwd -> flow loss -> bwd through the C ABI; plan = ops.SplatPlan or None."""
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    depths = c["depth"][None].contiguous()
    logits = c["wparam"][None].contiguous()
    s_ = (h * w) ** 0.5
    k4 = torch.tensor([0.85 * s_ / w, 0.85 * s_ / h, 0.5, 0.5], device=dev).expand(1, f, 4).contiguous()
    msum = ops.mask_sum(c["fmask"], c["bmask"])
    ws = ops.workspace(1, f, h, w, dev)
    rt = torch.empty(1, f - 1, 3, 4, device=dev)
    g_depth = torch.empty_like(depths)
    g_w = torch.zeros_like(logits)
    g_k4, g_rt = torch.empty_like(k4), torch.empty_like(rt)
    loss = torch.empty((), device=dev)
    if plan is None:
        weights = torch.sigmoid(100.0 * logits)
        rc = L.fm_procrustes_fwd(P(depths), P(k4), P(c["bwd"]), P(weights), None, 0, P(rt), P(ws), 1, f, h, w, st)
    else:
        rc = L.fm_procrustes_fwd_planned(P(depths), P(k4), P(c["bwd"]), P(logits), 100.0, plan.ptr, P(rt), P(ws),
                                         f, h, w, st)
    assert rc == 0, L.fm_last_error()
    rc = L.fm_flow_loss_fwd_bwd(P(depths), P(k4), P(rt), P(c["fwd"]), P(c["bwd"]), P(c["fmask"]), P(c["bmask"]),
                                P(msum), 0, 0.01, 1000.0, 1, P(loss), P(g_depth), P(g_rt), P(g_k4), P(ws), 1, f, h, w, st)
    assert rc == 0, L.fm_last_error()
    if plan is None:
        rc = L.fm_procrustes_bwd(P(depths), P(k4), P(c["bwd"]), P(weights), None, 0, None, 1, None, P(g_depth), P(g_w),
                                 P(g_k4), P(ws), 1, f, h, w, st)
        g_w = g_w * 100.0 * weights * (1 - weights)  # chain rule of the sigmoid (the RED op takes plain weights)
    else:
        rc = L.fm_procrustes_bwd_planned(P(depths), P(k4), P(c["bwd"]), P(logits), 100.0, plan.ptr, plan.overflow_max,
                                         None, 1, P(g_depth), P(g_w), P(g_k4), P(ws), f, h, w, st)
    assert rc == 0, L.fm_last_error()
    torch.cuda.synchronize()
    g_focal = float((g_k4[0, :, 0].double() * s_ / w + g_k4[0, :, 1].double() * s_ / h).sum())
    return {"rt": rt, "loss": float(loss), "g_depth": g_depth, "g_w": g_w, "g_focal": g_focal}


def compare(f, h, w, kind):
    c = make_case(f, h, w, kind)
    plan = ops.SplatPlan(c["bwd"])
    out = {"shape": [f, h, w], "flows": kind, "plan_status": plan.status, "overflow_max": plan.overflow_max,
           "entries_per_cell": plan.entries / max(1, (f - 1) * h * w)}
    if not plan.ok:
        out["ok"] = None
        return out
    a, b = run_ops(c, f, h, w, None), run_ops(c, f, h, w, plan)
    b2 = run_ops(c, f, h, w, plan)
    out.update({"rt_abs": float((a["rt"] - b["rt"]).abs().max()), "loss_rel": abs(a["loss"] - b["loss"]) / abs(a["loss"]),
                "g_depth_rel": rel(b["g_depth"], a["g_depth"]), "g_w_rel": rel(b["g_w"], a["g_w"]),
                "g_focal_rel": abs(a["g_focal"] - b["g_focal"]) / max(abs(a["g_focal"]), 1e-30),
                "bitwise_repeatable": bool(torch.equal(b["g_depth"], b2["g_depth"]) and torch.equal(b["g_w"], b2["g_w"]))})
    out["ok"] = bool(out["rt_abs"] < 2e-6 and out["g_depth_rel"] < 2e-5 and out["g_w_rel"] < 2e-5 and
                     out["g_focal_rel"] < 2e-4)
    return out


def fused(f, h, w, kind, use_plan, steps, full):
    c = make_case(f, h, w, kind)
    batch = Batch(torch.zeros(1, 1, 1, 1, 1, device=dev).expand(1, f, 3, h, w), torch.arange(f, device=dev)[None],
                  ["s"], ["d"])
    flows = Flows(c["fwd"], c["bwd"], c["fmask"], c["bmask"])
    tracks = [Tracks(xy, vis, s) for xy, vis, s in bench.synthetic_track_arrays(f, seed=0)] if full else None
    cfg = OverfitCfg(intrinsics="softmin", use_tracking=True) if full else OverfitCfg()
    o = FusedOverfitter(cfg, batch, flows, tracks, device=dev, use_splat_plan=use_plan)
    with torch.no_grad():
        o.model.backbone.depth.copy_(c["depth"])
        o.model.backbone.weights.copy_(c["wparam"])
    o.global_step = 50
    if full:
        o.injected_indices = torch.randperm(h * w, generator=torch.Generator().manual_seed(3))[:min(8192, h * w)].to(dev)
    losses = []
    for _ in range(3):
        losses.append(float(o.training_step()[0]))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        last = o.training_step()
    e1.record()
    torch.cuda.synchronize()
    return {"ms": e0.elapsed_time(e1) / steps, "losses": losses, "final": float(last[0]),
            "depth": o.model.backbone.depth.detach().clone(), "w": o.model.backbone.weights.detach().clone(),
            "plan": None if o._plan is None else (o._plan.status, o._plan.overflow_max)}


def time_ops(f, h, w, kind="iid"):
    c = make_case(f, h, w, kind)
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    t0 = time.time()
    plan = ops.SplatPlan(c["bwd"])
    torch.cuda.synchronize()
    t_build = time.time() - t0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    plan.rebuild(c["bwd"])
    e1.record()
    torch.cuda.synchronize()
    res = {"plan_build_ms": e0.elapsed_time(e1), "plan_first_build_s": t_build, "plan_status": plan.status,
           "overflow_max": plan.overflow_max, "entries_per_cell": plan.entries / ((f - 1) * h * w),
           "plan_bytes": plan.buf.numel()}
    depths = c["depth"][None].contiguous()
    logits = c["wparam"][None].contiguous()
    weights = torch.sigmoid(100.0 * logits)
    s_ = (h * w) ** 0.5
    k4 = torch.tensor([0.85 * s_ / w, 0.85 * s_ / h, 0.5, 0.5], device=dev).expand(1, f, 4).contiguous()
    msum = ops.mask_sum(c["fmask"], c["bmask"])
    ws = ops.workspace(1, f, h, w, dev)
    rt = torch.empty(1, f - 1, 3, 4, device=dev)
    g_depth, g_w = torch.empty_like(depths), torch.empty_like(logits)
    g_k4, g_rt = torch.empty_like(k4), torch.empty_like(rt)
    loss = torch.empty((), device=dev)

    def fwd_red():
        L.fm_procrustes_fwd(P(depths), P(k4), P(c["bwd"]), P(weights), None, 0, P(rt), P(ws), 1, f, h, w, st)

    def fwd_plan():
        L.fm_procrustes_fwd_planned(P(depths), P(k4), P(c["bwd"]), P(logits), 100.0, plan.ptr, P(rt), P(ws), f, h, w, st)

    def flow():
        L.fm_flow_loss_fwd_bwd(P(depths), P(k4), P(rt), P(c["fwd"]), P(c["bwd"]), P(c["fmask"]), P(c["bmask"]), P(msum),
                               0, 0.01, 1000.0, 1, P(loss), P(g_depth), P(g_rt), P(g_k4), P(ws), 1, f, h, w, st)

    def bwd_red():
        L.fm_procrustes_bwd(P(depths), P(k4), P(c["bwd"]), P(weights), None, 0, None, 1, None, P(g_depth), P(g_w),
                            P(g_k4), P(ws), 1, f, h, w, st)

    def bwd_plan():
        L.fm_procrustes_bwd_planned(P(depths), P(k4), P(c["bwd"]), P(logits), 100.0, plan.ptr, plan.overflow_max, None, 1,
                                    P(g_depth), P(g_w), P(g_k4), P(ws), f, h, w, st)

    def timed(fn, pre, n=10):
        for _ in range(3):
            pre(); fn()
        tot = 0.0
        for _ in range(n):
            pre()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record()
            torch.cuda.synchronize()
            tot += a.elapsed_time(b)
        return tot / n
    res["fwd_red_ms"] = timed(fwd_red, lambda: None)
    res["fwd_plan_ms"] = timed(fwd_plan, lambda: None)
    res["flow_ms"] = timed(flow, fwd_red)
    res["bwd_red_ms"] = timed(bwd_red, lambda: (fwd_red(), flow()))
    res["bwd_plan_ms"] = timed(bwd_plan, lambda: (fwd_plan(), flow()))
    return res


def main():
    if "--one" in sys.argv:  # python tools/ab_tiled.py --one F H W kind   (debugging: one comparison)
        i = sys.argv.index("--one")
        f, h, w = (int(x) for x in sys.argv[i + 1:i + 4])
        print("compare", json.dumps(compare(f, h, w, sys.argv[i + 4])), flush=True)
        return
    tiny = "--tiny" in sys.argv
    quick = "--quick" in sys.argv or tiny
    out = {"compare": [], "fused": [], "timing": {}}
    shapes = [(3, 24, 32), (4, 36, 48), (3, 100, 64), (5, 72, 96)]
    if not tiny:
        shapes += [(3, 360, 640)] + ([] if quick else [(2, 720, 1280)])
    timing_only = "--timing-only" in sys.argv
    if timing_only:
        shapes = [(3, 360, 640)]
    for f, h, w in shapes:
        for kind in ("iid", "smooth", "shift", "leave", "outliers")[:1 if timing_only else 5]:
            r = compare(f, h, w, kind)
            out["compare"].append(r)
            print("compare", json.dumps(r), flush=True)
    for f, h, w, full in ((6, 72, 96, False), (12, 136, 192, True))[:1 if tiny else 2]:
        a = fused(f, h, w, "iid", False, 3, full)
        b = fused(f, h, w, "iid", True, 3, full)
        r = {"shape": [f, h, w], "full": full, "losses_red": a["losses"], "losses_plan": b["losses"],
             "depth_rel": rel(b["depth"], a["depth"]), "w_abs": float((b["w"] - a["w"]).abs().max()), "plan": b["plan"]}
        out["fused"].append(r)
        print("fused", json.dumps(r), flush=True)
    if not quick:
        f, h, w = 150, 360, 640
        for kind in ("iid", "smooth"):
            t = time_ops(f, h, w, kind)
            out["timing"][kind] = t
            print("timing", kind, json.dumps(t), flush=True)
        for full in (False, True):
            a = fused(f, h, w, "iid", False, 20, full)
            b = fused(f, h, w, "iid", True, 20, full)
            r = {"full": full, "ms_red": a["ms"], "ms_plan": b["ms"], "final_red": a["final"], "final_plan": b["final"],
                 "depth_rel": rel(b["depth"], a["depth"]), "plan": b["plan"]}
            out["timing"]["fused_full" if full else "fused_flow_only"] = r
            print("fused-timing", json.dumps(r), flush=True)
    Path(ROOT / "tools" / "_build").mkdir(exist_ok=True)
    (ROOT / "tools" / "_build" / "ab_tiled.json").write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
