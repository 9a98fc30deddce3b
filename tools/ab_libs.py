"""A/B of several BUILDS of the library on an H100 (kernel experiments are compiled as separate .so
files, e.g. with -D knobs, instead of living behind run-time switches in the product):

  python tools/ab_libs.py flowmap_b200/csrc/ab/base.so flowmap_b200/csrc/ab/x.so ... [--no-step]

Building a variant (the knobs are `#ifndef` defaults in csrc/fm_kernels.cu, e.g. FM_PATCH_LANES or
the FM_WIN_* tile / halo / blocks-per-SM of k_distribute_window):

  cd flowmap_b200/csrc && mkdir -p ab && nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 \
      --expt-extended-lambda -Xcompiler -fPIC -shared -DFM_PATCH_LANES=4 -o ab/lanes4.so fm_kernels.cu fm_io.cu

(`git stash` + a normal build gives the committed state as the first, reference build.)

For every build: results of the three path ops at a small and at the benchmark shape against the
FIRST build (poses, loss, depth / weight / intrinsics gradients), CUDA-event times of the three ops
at 150 x 360 x 640 on iid and on smooth flows, and the fused full / flow-only step (trajectory
against the first build + ms per step).  Writes tools/_build/ab_libs.json."""
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from flowmap_b200 import _lib as libmod  # noqa: E402
from flowmap_b200 import ops  # noqa: E402
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
    if kind == "leave":    # taps leave the frame: clamped rows / columns
        inp["bwd"] = inp["bwd"] + torch.tensor([0.3, 0.2])
    elif kind == "smooth":
        coarse = 0.01 * torch.randn(f - 1, 2, (h + 15) // 16 + 1, (w + 15) // 16 + 1, generator=g)
        up = torch.nn.functional.interpolate(coarse, size=(h, w), mode="bilinear", align_corners=True)
        inp["bwd"] = up.permute(0, 2, 3, 1)[None].contiguous()
    return {k: v.to(dev).contiguous() for k, v in inp.items()}


class OpsCase:
    def __init__(self, f, h, w, kind):
        self.f, self.h, self.w = f, h, w
        c = self.c = make_case(f, h, w, kind)
        self.depths = c["depth"][None].contiguous()
        self.weights = torch.sigmoid(100.0 * c["wparam"][None]).contiguous()
        s_ = (h * w) ** 0.5
        self.k4 = torch.tensor([0.85 * s_ / w, 0.85 * s_ / h, 0.5, 0.5], device=dev).expand(1, f, 4).contiguous()
        self.msum = ops.mask_sum(c["fmask"], c["bmask"])
        self.ws = ops.workspace(1, f, h, w, dev)
        self.rt = torch.empty(1, f - 1, 3, 4, device=dev)
        self.g_depth, self.g_w = torch.empty_like(self.depths), torch.empty_like(self.weights)
        self.g_k4, self.g_rt = torch.empty_like(self.k4), torch.empty_like(self.rt)
        self.loss = torch.empty((), device=dev)
        self.st = torch.cuda.current_stream().cuda_stream

    def fwd(self, L):
        rc = L.fm_procrustes_fwd(P(self.depths), P(self.k4), P(self.c["bwd"]), P(self.weights), None, 0, P(self.rt),
                                 P(self.ws), 1, self.f, self.h, self.w, self.st)
        assert rc == 0, L.fm_last_error()

    def flow(self, L):
        c = self.c
        rc = L.fm_flow_loss_fwd_bwd(P(self.depths), P(self.k4), P(self.rt), P(c["fwd"]), P(c["bwd"]), P(c["fmask"]),
                                    P(c["bmask"]), P(self.msum), 0, 0.01, 1000.0, 1, P(self.loss), P(self.g_depth),
                                    P(self.g_rt), P(self.g_k4), P(self.ws), 1, self.f, self.h, self.w, self.st)
        assert rc == 0, L.fm_last_error()

    def bwd(self, L):
        rc = L.fm_procrustes_bwd(P(self.depths), P(self.k4), P(self.c["bwd"]), P(self.weights), None, 0, None, 1, None,
                                 P(self.g_depth), P(self.g_w), P(self.g_k4), P(self.ws), 1, self.f, self.h, self.w,
                                 self.st)
        assert rc == 0, L.fm_last_error()

    def results(self, L):
        self.g_w.zero_()
        self.fwd(L); self.flow(L); self.bwd(L)
        torch.cuda.synchronize()
        return {"rt": self.rt.clone(), "loss": float(self.loss), "g_depth": self.g_depth.clone(),
                "g_w": self.g_w.clone(), "g_k4": self.g_k4.clone()}

    def times(self, L, n=20):
        def timed(fn, pre):
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
        return {"fwd_ms": timed(lambda: self.fwd(L), lambda: None),
                "flow_ms": timed(lambda: self.flow(L), lambda: self.fwd(L)),
                "bwd_ms": timed(lambda: self.bwd(L), lambda: (self.fwd(L), self.flow(L)))}


def fused(f, h, w, steps, full):
    """The fused step on whatever library flowmap_b200._lib currently holds."""
    c = make_case(f, h, w, "iid")
    batch = Batch(torch.zeros(1, 1, 1, 1, 1, device=dev).expand(1, f, 3, h, w), torch.arange(f, device=dev)[None],
                  ["s"], ["d"])
    flows = Flows(c["fwd"], c["bwd"], c["fmask"], c["bmask"])
    tracks = [Tracks(xy, vis, s) for xy, vis, s in bench.synthetic_track_arrays(f, seed=0)] if full else None
    cfg = OverfitCfg(intrinsics="softmin", use_tracking=True) if full else OverfitCfg()
    o = FusedOverfitter(cfg, batch, flows, tracks, device=dev)
    with torch.no_grad():
        o.model.backbone.depth.copy_(c["depth"])
        o.model.backbone.weights.copy_(c["wparam"])
    o.global_step = 50
    if full:
        o.injected_indices = torch.randperm(h * w, generator=torch.Generator().manual_seed(3))[:min(8192, h * w)].to(dev)
    losses = [float(o.training_step()[0]) for _ in range(5)]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        o.training_step()
    e1.record()
    torch.cuda.synchronize()
    return {"ms": e0.elapsed_time(e1) / steps, "losses": losses,
            "depth": o.model.backbone.depth.detach().clone(), "w": o.model.backbone.weights.detach().clone()}


def main():
    paths = [a for a in sys.argv[1:] if not a.startswith("--") and not a.isdigit()]
    with_step = "--no-step" not in sys.argv
    libs = [(Path(p).stem, libmod.load_library(ROOT / p)) for p in paths]
    out = {}
    ref = {}
    small = [(4, 36, 48, "iid"), (3, 100, 64, "leave"), (5, 72, 96, "leave"), (3, 100, 64, "smooth")]
    big = [(150, 360, 640, "iid"), (150, 360, 640, "smooth")]
    if "--shape" in sys.argv:  # e.g. --shape 150 720 1280: time the ops at another shape instead
        i = sys.argv.index("--shape")
        f_, h_, w_ = (int(x) for x in sys.argv[i + 1:i + 4])
        big = [(f_, h_, w_, "iid")]

    cases = {key: OpsCase(*key) for key in small + big}
    for name, L in libs:
        rec = out[name] = {"parity": [], "times": {}}
        for key in small + big:
            r = cases[key].results(L)
            if name == libs[0][0]:
                ref[key] = r
                continue
            b = ref[key]
            e = {"case": list(key), "rt_abs": float((r["rt"] - b["rt"]).abs().max()),
                 "loss_rel": abs(r["loss"] - b["loss"]) / abs(b["loss"]), "g_depth_rel": rel(r["g_depth"], b["g_depth"]),
                 "g_w_rel": rel(r["g_w"], b["g_w"]), "g_k4_rel": rel(r["g_k4"], b["g_k4"])}
            e["ok"] = bool(e["rt_abs"] < 2e-6 and e["loss_rel"] < 1e-6 and e["g_depth_rel"] < 2e-5 and
                           e["g_w_rel"] < 2e-5 and e["g_k4_rel"] < 2e-4)
            rec["parity"].append(e)
            print(name, "parity", json.dumps(e), flush=True)
        for key in big:
            t = cases[key].times(L)
            rec["times"][key[3]] = t
            print(name, "times", key[3], json.dumps(t), flush=True)
    del cases
    torch.cuda.empty_cache()
    if with_step:
        base = {}
        for name, L in libs:
            libmod._lib = L  # the package's ops / fused step now run on this build
            for full in ((False,) if "--shape" in sys.argv else (False, True)):
                small_run = fused(8, 72, 96, 3, full)
                r = fused(*big[0][:3], 30, full)
                key = "full" if full else "flow_only"
                if name == libs[0][0]:
                    base[key] = (small_run, r)
                b_small, b_big = base[key]
                e = {"ms": r["ms"], "losses": r["losses"], "small_depth_rel": rel(small_run["depth"], b_small["depth"]),
                     "small_w_abs": float((small_run["w"] - b_small["w"]).abs().max()),
                     "depth_rel": rel(r["depth"], b_big["depth"]), "w_abs": float((r["w"] - b_big["w"]).abs().max())}
                out[name]["step_" + key] = e
                print(name, "step", key, json.dumps(e), flush=True)
    Path(ROOT / "tools" / "_build").mkdir(exist_ok=True)
    (ROOT / "tools" / "_build" / "ab_libs.json").write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
