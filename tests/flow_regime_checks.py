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


K_REGIMES = ("offcentre", "zoom", "corner", "videos")


def kmat(k4):
    """(..., 3, 3) intrinsics from k4 rows (fx, fy, cx, cy), differentiably."""
    z, o = torch.zeros_like(k4[..., 0]), torch.ones_like(k4[..., 0])
    return torch.stack((torch.stack((k4[..., 0], z, k4[..., 2]), -1), torch.stack((z, k4[..., 1], k4[..., 3]), -1),
                        torch.stack((z, z, o), -1)), -2)


def k4_regime(kind, b, f, h, w):
    """Float64 per-frame intrinsics (b, f, 4) = (fx, fy, cx, cy), normalised as the reference's, for
    calibrated videos (datasets with ground-truth K) instead of one focal length at the image centre:

    - ``offcentre``: one K for every frame, principal point (0.62, 0.41), fx and fy from different focal
      lengths (fx != fy H / W);
    - ``zoom``: fx and fy grow 1.5x over the video (at different rates), the principal point drifts
      from (0.35, 0.65) to (0.65, 0.35);
    - ``corner``: principal point near (0.1, 0.9), drifting by 0.02, fx != fy H / W: the cloud's x / y
      centroid sits far off the optical axis;
    - ``videos``: every video its own zoom (b = 2: one zooms in with its centre moving right, the other
      zooms out with its centre moving left), so a pair that reads another video's K is wrong."""
    s = (h * w) ** 0.5
    t = torch.linspace(0.0, 1.0, f, dtype=torch.float64)
    one = torch.ones_like(t)
    if kind == "offcentre":
        rows = [(0.95 * s / w * one, 0.8 * s / h * one, 0.62 * one, 0.41 * one)] * b
    elif kind == "zoom":
        rows = [(0.8 * s / w * (1 + 0.5 * t), 0.9 * s / h * (1 + 0.4 * t), 0.35 + 0.3 * t, 0.65 - 0.3 * t)] * b
    elif kind == "corner":
        rows = [(0.9 * s / w * one, 0.75 * s / h * one, 0.1 + 0.02 * t, 0.9 - 0.02 * t)] * b
    elif kind == "videos":
        rows = [(0.8 * s / w * (1 + 0.5 * t), 0.9 * s / h * (1 + 0.4 * t), 0.4 + 0.2 * t, 0.45 + 0.1 * t),
                (1.2 * s / w * (1 - 0.3 * t), 1.0 * s / h * (1 - 0.25 * t), 0.6 - 0.2 * t, 0.6 - 0.15 * t)][:b]
        if b == 1:
            raise ValueError("the `videos` regime needs b >= 2")
        rows += rows[-1:] * (b - 2)
    else:
        raise ValueError(kind)
    return torch.stack([torch.stack(r, -1) for r in rows]).contiguous()


def k4_scene(k4, h, w, seed, rotation=0.08, translation=0.3, noise=0.001):
    """oracle.consistent_scene under per-frame intrinsics k4 (b, f, 4): per item, the inside of a sphere
    seen by cameras moving by 0.08 rad / 0.3 per frame, depths the exact ray / sphere hits with each frame's
    K, flows the float64 induced flows at the true per-frame K plus N(0, noise^2).  Returns float64 depth
    (b, f, h, w) and Flows."""
    from oracle import flowmap_oracle as O
    depths, fl = [], []
    for item in range(k4.shape[0]):
        g = torch.Generator().manual_seed(seed + item)
        f = k4.shape[1]
        rel = torch.eye(4, dtype=torch.float64).repeat(f - 1, 1, 1)
        ang = rotation * torch.randn(f - 1, 3, generator=g, dtype=torch.float64)
        for i in range(f - 1):
            ax, ay, az = ang[i]
            skew = torch.tensor([[0, -az, ay], [az, 0, -ax], [-ay, ax, 0]], dtype=torch.float64)
            rel[i, :3, :3] = torch.linalg.matrix_exp(skew)
        rel[:, :3, 3] = translation * torch.randn(f - 1, 3, generator=g, dtype=torch.float64)
        ext = O.pose_chain(rel[None])
        k = kmat(k4[item:item + 1])
        xy = O.pixel_grid(h, w, torch.float64)
        rays = O.unproject(xy, torch.ones(1, f, h, w, dtype=torch.float64), k[:, :, None, None])
        centre = torch.tensor([0.2, -0.1, 0.5], dtype=torch.float64)
        d = O.matvec(ext[:, :, None, None, :3, :3], rays)
        o = ext[:, :, None, None, :3, 3] - centre
        a_, b_, c_ = (d * d).sum(-1), 2 * (d * o).sum(-1), (o * o).sum(-1) - 9.0
        depth = (-b_ + torch.sqrt(b_ * b_ - 4 * a_ * c_)) / (2 * a_)
        surf = O.unproject(xy, depth, k[:, :, None, None])
        jitter = lambda: noise * torch.randn(1, f - 1, h, w, 2, generator=g, dtype=torch.float64)  # noqa: E731
        u = lambda: 0.5 + 0.5 * torch.rand(1, f - 1, h, w, generator=g, dtype=torch.float64)  # noqa: E731
        fl.append((O.forward_flow_positions(surf, ext, k) - xy + jitter(),
                   O.backward_flow_positions(surf, ext, k) - xy + jitter(), u(), u()))
        depths.append(depth)
    return torch.cat(depths), O.Flows(*(torch.cat([p[i] for p in fl]).contiguous() for i in range(4)))


def oracle_steps_k4(depth, wparam, flows, k4, indices=None):
    """{64: float64 result, 32: float32 result} of one flow-loss step (Procrustes poses, 1000 x Huber flow
    loss) on float64 inputs under per-frame intrinsics k4 (b, f, 4), a leaf of the autograd graph.  g_k4:
    d loss / d k4 with the flow loss differentiated in K too (k_mode "full"); g_k4_const: the Procrustes
    part alone (k_mode "const": the flow loss takes K as a constant).  g_depth and g_w are the same in both."""
    from oracle import flowmap_oracle as O
    out = {}
    b, f, h, w = depth.shape
    for bits, dt in ((64, torch.float64), (32, torch.float32)):
        fl = type(flows)(*(t.to(dt) for t in (flows.forward, flows.backward, flows.forward_mask,
                                             flows.backward_mask)))
        d, wp, k = (t.to(dt).clone().requires_grad_(True) for t in (depth, wparam, k4))
        km = kmat(k)
        surf = O.unproject(O.pixel_grid(h, w, dt), d, km[:, :, None, None])
        idx = torch.arange(h * w) if indices is None else indices
        ext = O.align_surfaces(surf, fl.backward, torch.sigmoid(100.0 * wp), idx)
        loss = 1000.0 * O.flow_loss(surf, ext, km, fl, "huber", 0.01)
        # "const": K reaches the loss only through the poses (the flow loss unprojects and projects with
        # a constant K)
        surf_const = O.unproject(O.pixel_grid(h, w, dt), d, km.detach()[:, :, None, None])
        loss_const = 1000.0 * O.flow_loss(surf_const, ext, km.detach(), fl, "huber", 0.01)
        gd, gw, gk = torch.autograd.grad(loss, (d, wp, k), retain_graph=True)
        (gkc,) = torch.autograd.grad(loss_const, (k,))
        out[bits] = dict(loss=float(loss.detach()), ext=ext.detach().double(), g_depth=gd.double(), g_w=gw.double(),
                         g_focal=None, g_k4=gk.double(), g_k4_const=gkc.double())
    return out


def k4_errors(g_k4, ref, noise=False):
    """The intrinsics gradient per component and per frame: for each of fx, fy, cx, cy a list over the
    frames of all items of |error| / (the component's L2 norm over those frames).  A component of one frame
    can be a sum that cancels to near zero, and its own relative error then measures only the
    cancellation; scaled by the component's size over the video, a frame or component that takes another's
    gradient still stands out.  noise: the float32 oracle's errors, every frame of a component set to its
    worst frame (which frame a float32 summation order happens to get right varies, as for the tracking
    sweep's per-frame sums)."""
    a, r = torch.as_tensor(g_k4).double().reshape(-1, 4), ref.double().reshape(-1, 4)
    out = {}
    for c, name in enumerate(("fx", "fy", "cx", "cy")):
        e = ((a[:, c] - r[:, c]).abs() / r[:, c].norm().clamp_min(1e-300)).tolist()
        out[f"k4_{name}"] = [max(e)] * len(e) if noise else e
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
