"""Helpers shared by the CPU and GPU flow-regime tests (test_host_emulation.py,
test_gpu_flow_regimes.py): the oracle's loss, poses and gradients at float64 and float32 on the
same inputs, and error metrics that look at the depth gradient per frame and on its one-pixel border
band and at the weight gradient per frame pair.  A wrong tile, pair or image edge vanishes in a
whole-tensor relative L2 error; it does not vanish in these."""
import torch

from conftest import max_abs, rel_l2
from test_gpu_parity import _oracle_flow_step


def start_point(depth, focal, seed):
    """The parameters a step starts from: depth x (1 + N(0, 0.02^2)) and 1.05 x the focal length.
    In the `scene` regime the exact depth and focal length are a stationary point of the loss, where
    the focal-length gradient is a sum of per-frame terms that cancel to 1 part in 200 and its
    relative error measures nothing but that cancellation; a step from nearby has real gradients."""
    gen = torch.Generator().manual_seed(seed)
    return depth * (1.0 + 0.02 * torch.randn(depth.shape, generator=gen, dtype=depth.dtype)), 1.05 * focal


def oracle_steps(depth, wparam, flows, focal=0.85, indices=None, softmin=None, **kw):
    """{64: float64 result, 32: float32 result} of one flow-loss step (_oracle_flow_step) on
    float64 inputs depth (b, f, h, w), wparam (b, f-1, h, w) and Flows.  `indices`: the Procrustes
    point set (default: every pixel); `softmin=(indices, candidates)`: intrinsics from the candidate
    sweep, g_focal None and g_err the gradient of the sweep's errors."""
    out = {}
    for bits, dt in ((64, torch.float64), (32, torch.float32)):
        fl = type(flows)(*(t.to(dt) for t in (flows.forward, flows.backward, flows.forward_mask,
                                             flows.backward_mask)))
        sm = None if softmin is None else (softmin[0], softmin[1].to(dt))
        loss, ext, gd, gw, gf = _oracle_flow_step(depth.to(dt), wparam.to(dt), fl, focal, indices=indices,
                                                  softmin=sm, **kw)
        out[bits] = dict(loss=float(loss), ext=ext.double(), g_depth=gd.double(), g_w=gw.double(),
                         g_focal=float(gf) if softmin is None else None)
        if softmin is not None:
            out[bits]["g_err"] = gf.double()
    return out


def border_band(h, w):
    m = torch.zeros(h, w, dtype=torch.bool)
    m[0], m[-1], m[:, 0], m[:, -1] = True, True, True, True
    return m


def errors(out, ref, per_item=True):
    """Errors of `out` against `ref` (dicts with loss, ext, g_depth, g_w, g_focal; g_focal None
    when the intrinsics get no gradient).  Gradients are relative L2 errors: over the whole tensor,
    on the border band of every frame, and (per_item) for every frame / pair on its own."""
    gd, rd = out["g_depth"].double(), ref["g_depth"]
    h, w = rd.shape[-2:]
    gd, rd = gd.reshape(-1, h, w), rd.reshape(-1, h, w)
    gw, rw = out["g_w"].double().reshape(-1, h, w), ref["g_w"].reshape(-1, h, w)
    band = border_band(h, w)
    e = dict(loss=abs(float(out["loss"]) - ref["loss"]) / abs(ref["loss"]),
             pose=max_abs(out["ext"].double().reshape(ref["ext"].shape), ref["ext"]),
             depth=rel_l2(gd, rd), depth_border=rel_l2(gd[:, band], rd[:, band]), weights=rel_l2(gw, rw))
    if out.get("g_focal") is not None:
        e["focal"] = abs(float(out["g_focal"]) - ref["g_focal"]) / abs(ref["g_focal"])
    if per_item:
        e["depth_frame"] = [rel_l2(gd[i], rd[i]) for i in range(rd.shape[0])]
        e["weights_pair"] = [rel_l2(gw[i], rw[i]) for i in range(rw.shape[0])]
    return e


def check(errs, noise, label, loss_tol, pose_tol, floor, relative_fixed=False):
    """Loss and poses against fixed tolerances; every other metric (the gradients of `errors`, and
    whatever else a caller adds, such as per-frame pose twists) against max(floor, 3 x the float32
    oracle's own error in the same metric).  relative_fixed: the loss and pose tolerances too become
    max(tol, 3 x the float32 oracle's error), for inputs so badly conditioned that float32 itself
    misses the fixed ones."""
    print(label, "errors vs float64 oracle:", _fmt(errs), "| float32 oracle:", _fmt(noise))
    if relative_fixed:
        loss_tol, pose_tol = max(loss_tol, 3 * noise["loss"]), max(pose_tol, 3 * noise["pose"])
    assert errs["loss"] <= loss_tol, (label, "loss", errs["loss"])
    assert errs["pose"] <= pose_tol, (label, "pose", errs["pose"])
    for key in errs:
        if key in ("loss", "pose"):
            continue
        got, ref = errs[key], noise[key]
        if isinstance(got, list):
            for i, (a, n) in enumerate(zip(got, ref)):
                assert a <= max(floor, 3 * n), (label, f"{key}[{i}]", a, n)
        else:
            assert got <= max(floor, 3 * ref), (label, key, got, ref)


def _fmt(e):
    return {k: ([f"{x:.1e}" for x in v] if isinstance(v, list) else f"{v:.1e}") for k, v in e.items()}
