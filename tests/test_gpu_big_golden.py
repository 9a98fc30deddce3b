"""`-m gpu`: parity AT THE BENCHMARKED SHAPES against fixtures generated from the unmodified
reference (tests/golden/make_golden_big.py): BASELINE configs[1] (30 x 360 x 480, flow + tracks),
configs[2] (150 x 360 x 640, the full loop that bench.py times: softmin intrinsics + flow +
tracking + Adam) and a 24-frame slice of configs[3] (720 x 1280, flow loss only).

The inputs are regenerated from the seeds (bench.synthetic_inputs / synthetic_track_arrays); the
fixtures hold the reference's float32 outputs in reduced form: loss parts, all poses, fx, and per
tensor the per-frame L2 norms plus a strided subsample.  Tolerance: 1e-4 relative (north_star) on
loss / poses / intrinsics; gradients are judged against the reference's float64 run (big_*_f64.npz)
with max(1e-4, the reference's own float32-vs-float64 noise) -- on these rough synthetic depths the
reference's float32 gradients are themselves 2-6e-4 away from float64.
"""
import numpy as np
import pytest
import torch

from conftest import GOLDEN, max_abs, rel_l2

pytestmark = pytest.mark.gpu

CASES = {
    "c2": dict(intrinsics="softmin", tracking=True),
    "c3": dict(intrinsics="softmin", tracking=True),
    "c4slice": dict(intrinsics="regressed", tracking=False),
}


def _load(which, f64=False):
    with np.load(GOLDEN / f"big_{which}{'_f64' if f64 else ''}.npz") as z:
        return {k: z[k] for k in z.files}


def _grad_errors(norms, sub, g, key):
    return (float(np.max(np.abs(norms - g[key + "_norms"]) / np.maximum(g[key + "_norms"], 1e-30))),
            rel_l2(sub, g[key + "_sub"]))


def _reduced(t, stride):
    t = t.detach()
    return t.double().flatten(1).norm(dim=1).cpu().numpy(), t.flatten()[::stride].float().cpu().numpy()


def _make(which, g, fused=True):
    import bench
    from flowmap_b200.overfit import FusedOverfitter, Overfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows, Tracks
    f, h, w, seed = int(g["frames"]), int(g["height"]), int(g["width"]), int(g["seed"])
    inp = bench.synthetic_inputs(f, h, w, seed=seed)
    dev = torch.device("cuda:0")
    batch = Batch(torch.zeros(1, 1, 1, 1, 1, device=dev).expand(1, f, 3, h, w), torch.arange(f, device=dev)[None],
                  ["s"], ["d"])
    flows = Flows(*(inp[k].to(dev) for k in ("fwd", "bwd", "fmask", "bmask")))
    case = CASES[which]
    tracks = None
    if case["tracking"]:
        tracks = [Tracks(xy, vis, s) for xy, vis, s in bench.synthetic_track_arrays(f, seed=seed)]
    cfg = OverfitCfg(intrinsics=case["intrinsics"], use_tracking=case["tracking"])
    if fused:
        o = FusedOverfitter(cfg, batch, flows, tracks, device=dev)
    else:
        o = Overfitter(cfg, batch, flows, tracks, device=dev)
    with torch.no_grad():
        o.model.backbone.depth.copy_(inp["depth"])
        o.model.backbone.weights.copy_(inp["wparam"])
    o.global_step = int(g["start_step"])
    if case["intrinsics"] == "softmin":
        idx = torch.as_tensor(g["softmin_indices"], device=dev)
        if fused:
            o.injected_indices = idx
        else:
            o.model.intrinsics.injected_indices = idx
    return o, inp


@pytest.mark.parametrize("which", ["c2", "c3", "c4slice"], ids=lambda k: f"{k}-red")  # red: the global-RED backward
def test_fused_step_gradients_at_benchmark_shapes(which):
    """First step, no update: loss parts, poses, fx and the full gradients vs the reference."""
    g, g64 = _load(which), _load(which, f64=True)
    o, _ = _make(which, g)
    stride = int(g["stride"])
    total, _ = o.training_step(update=False)
    torch.cuda.synchronize()
    errs = {"loss": abs(float(total) - float(g["loss"][0])) / abs(float(g["loss"][0])),
            "loss_flow": abs(float(o._loss) - float(g["loss_flow"][0])) / abs(float(g["loss_flow"][0])),
            "pose": max_abs(o.extrinsics()[0].cpu(), g["extrinsics"][0]),
            "fx": abs(float(o.intrinsics_k4()[0, 0]) - float(g["fx"][0])) / float(g["fx"][0])}
    if CASES[which]["tracking"]:
        errs["loss_tracking"] = abs(float(o._track_loss) - float(g["loss_tracking"][0])) / abs(float(g["loss_tracking"][0]))
    # Gradients: the arbiter is the reference's float64 run; the reference's own float32 run is the
    # noise floor (at these rough-depth shapes it is 2-6e-4 away from float64).  Bar: 1e-4, or the
    # reference's own float32 noise where that is larger -- and our error must stay below that noise.
    gr = o.gradients()
    noise = {}
    for name, key in (("depth", "g_depth"), ("weights", "g_wparam")):
        norms, sub = _reduced(gr[name], stride)
        errs[key + "_norms"], errs[key + "_sub"] = _grad_errors(norms, sub, g64, key)
        noise[key + "_norms"], noise[key + "_sub"] = _grad_errors(g[key + "_norms"], g[key + "_sub"], g64, key)
    if "g_focal" in g:
        errs["g_focal"] = abs(float(gr["focal"]) - float(g64["g_focal"])) / abs(float(g64["g_focal"]))
        noise["g_focal"] = abs(float(g["g_focal"]) - float(g64["g_focal"])) / abs(float(g64["g_focal"]))
    print(which, "errors vs the reference (float64 arbiter for gradients):", errs, "| reference float32 noise:", noise)
    assert errs["pose"] <= 5e-5, errs
    for k, v in errs.items():
        if k != "pose":
            assert v <= max(1e-4, noise.get(k, 0.0)), (k, errs, noise)


@pytest.mark.parametrize("which", ["c2", "c3", "c4slice"])
def test_fused_adam_trajectory_at_benchmark_shapes(which):
    """Three optimisation steps (Adam) from the same start: per-step loss / poses / fx and the
    final parameters vs the reference's trajectory."""
    g = _load(which)
    o, inp = _make(which, g)
    stride = int(g["stride"])
    steps = len(g["loss"])
    errs = {"loss": 0.0, "pose": 0.0, "fx": 0.0}
    for s in range(steps):
        total, _ = o.training_step()
        errs["loss"] = max(errs["loss"], abs(float(total) - float(g["loss"][s])) / abs(float(g["loss"][s])))
        errs["pose"] = max(errs["pose"], max_abs(o.extrinsics()[0].cpu(), g["extrinsics"][s]))
        errs["fx"] = max(errs["fx"], abs(float(o.intrinsics_k4()[0, 0]) - float(g["fx"][s])) / float(g["fx"][s]))
    for name, key, init in (("depth", "depth_final", inp["depth"]), ("weights", "wparam_final", inp["wparam"])):
        p = getattr(o.model.backbone, name)
        norms, sub = _reduced(p, stride)
        errs[key + "_norms"] = float(np.max(np.abs(norms - g[key + "_norms"]) / np.maximum(g[key + "_norms"], 1e-30)))
        errs[key + "_sub"] = rel_l2(sub, g[key + "_sub"])
        # the UPDATE itself (Adam's first steps are ~ lr * sign(gradient): elements whose gradient is
        # within float32 noise of zero may flip, hence the looser bound on this one)
        init_sub = init.flatten()[::stride].numpy()
        errs[key + "_update"] = rel_l2(sub - init_sub, g[key + "_sub"] - init_sub)
    print(which, "trajectory errors vs the reference:", errs)
    assert errs["loss"] <= 1e-4 and errs["fx"] <= 1e-4 and errs["pose"] <= 5e-5, errs
    for key in ("depth_final", "wparam_final"):
        # three Adam steps move a parameter by ~1e-4: the update carries the information, the
        # parameter itself only has to stay where the reference's is
        assert errs[key + "_norms"] <= 1e-4 and errs[key + "_sub"] <= 1e-3, errs
        assert errs[key + "_update"] <= 2e-2, errs


@pytest.mark.parametrize("which", ["c2", "c3"])
def test_dropin_surface_trajectory_at_benchmark_shapes(which):
    """The same three steps through the reference-shaped surface (Model.forward + LossFlow /
    LossTracking.forward + backward + FusedAdam), i.e. what install() exposes."""
    g = _load(which)
    o, inp = _make(which, g, fused=False)
    stride = int(g["stride"])
    errs = {"loss": 0.0, "pose": 0.0}
    for s in range(len(g["loss"])):
        total, out = o.training_step()
        errs["loss"] = max(errs["loss"], abs(float(total) - float(g["loss"][s])) / abs(float(g["loss"][s])))
        errs["pose"] = max(errs["pose"], max_abs(out.extrinsics[0].cpu(), g["extrinsics"][s]))
    for name, key, init in (("depth", "depth_final", inp["depth"]), ("weights", "wparam_final", inp["wparam"])):
        _, sub = _reduced(getattr(o.model.backbone, name), stride)
        init_sub = init.flatten()[::stride].numpy()
        errs[key + "_update"] = rel_l2(sub - init_sub, g[key + "_sub"] - init_sub)
    print(which, "drop-in trajectory errors vs the reference:", errs)
    assert errs["loss"] <= 1e-4 and errs["pose"] <= 5e-5, errs
    assert errs["depth_final_update"] <= 2e-2 and errs["wparam_final_update"] <= 2e-2, errs
