"""The Procrustes, flow-loss and tracking kernels against the float64 oracle in the flow regimes of
real videos (oracle.flow_regime): large coherent motion, correspondences that leave the frame,
outliers, zoom, and a rigid scene under large camera motion.  These reach what the few-pixel iid
flows of the other parity tests do not: bilinear_taps' clipping to the border and the pile-up of
depth-gradient taps on the first and last rows and columns, the placement of k_distribute_window's
scatter window (shifted by the tile's mean flow, clamped onto the image) and taps in its last
column and pitch padding, the float RED fall-back for taps outside the window, and the tracking
sweep's predicted-target mask under large poses.

Every gradient is checked per frame (depth) or per frame pair (weights) and on the depth gradient's
one-pixel border band, besides the whole tensor, against max(1e-4, 3x the float32 oracle's own
error in the same metric); a wrong tile, pair or edge would vanish in a whole-tensor error."""
import pytest
import torch

from conftest import max_abs
from flow_regime_checks import check, errors, oracle_steps, start_point

pytestmark = pytest.mark.gpu

KINDS = ["iid", "shift", "leave", "outliers", "zoom", "scene"]


@pytest.mark.parametrize("b,f,h,w", [(2, 3, 96, 192),    # 3 x 3 tiles of 64 x 32 per frame: every window
                                     (2, 3, 72, 136),    # edge clamped, plus free ones; partial tiles
                                     (1, 3, 72, 133)])   # odd width, W % 4 != 0: k_distribute_dense
@pytest.mark.parametrize("kind", KINDS)
def test_autograd_ops_vs_float64_oracle(kind, b, f, h, w):
    """ops.procrustes_poses + ops.flow_loss in the full, shared_focal and const intrinsics modes."""
    from oracle import flowmap_oracle as O
    from flowmap_b200 import ops
    depth, fl, focal, _ = O.flow_regime(kind, f, h, w, seed=w, b=b)
    depth, focal = start_point(depth, focal, seed=w + 1)
    wparam = 0.01 * torch.randn(b, f - 1, h, w, generator=torch.Generator().manual_seed(w + 2), dtype=torch.float64)
    refs = oracle_steps(depth, wparam, fl, focal)
    noise = errors(refs[32], refs[64])
    d = depth.float().cuda().requires_grad_(True)
    wp = wparam.float().cuda().requires_grad_(True)
    foc = torch.tensor(focal, dtype=torch.float32, device="cuda", requires_grad=True)
    s = (h * w) ** 0.5
    half = torch.tensor(0.5, device="cuda")
    k4 = torch.stack((foc * s / w, foc * s / h, half, half)).expand(b, f, 4)
    flc = [t.float().cuda() for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)]
    rt = ops.procrustes_poses(d, torch.sigmoid(100.0 * wp), k4, flc[1], None)
    ext = ops.pose_chain(rt.detach()).cpu()
    for mode in ("full", "shared_focal", "const"):
        d.grad = wp.grad = foc.grad = None
        loss = ops.flow_loss(d, rt, k4, *flc, ops.mask_sum(flc[2], flc[3]), "huber", 0.01, 1000.0, mode)
        loss.backward(retain_graph=True)
        # const: the flow loss gives the intrinsics no gradient, so foc.grad holds only the Procrustes part
        out = dict(loss=float(loss), ext=ext, g_depth=d.grad.cpu(), g_w=wp.grad.cpu(),
                   g_focal=None if mode == "const" else float(foc.grad))
        check(errors(out, refs[64]), noise, f"{kind} {b}x{f}x{h}x{w} {mode}", loss_tol=1e-4, pose_tol=2e-5,
              floor=1e-4)


def _fused_case(kind, f, h, w):
    from oracle import flowmap_oracle as O
    depth, fl, focal, ext = O.flow_regime(kind, f, h, w, seed=31)
    if kind == "scene":  # tracks of the scene itself: small residuals, large poses
        tracks = O.scene_tracks(depth[0], ext, focal, [(0, f), (2, 3), (f - 2, 2)], n_points=600, seed=32)
    else:
        tracks = O.synthetic_tracks(f, n_points=600, interval=3, radius=2, seed=32, dtype=torch.float64)
    depth, focal = start_point(depth, focal, seed=33)
    wparam = 0.01 * torch.randn(f - 1, h, w, generator=torch.Generator().manual_seed(34), dtype=torch.float64)
    return depth[0], wparam, fl, focal, tracks


@pytest.mark.parametrize("kind", ["scene", "zoom"], ids=lambda k: f"{k}-red")  # red: the global-RED backward
def test_fused_step_with_tracking_vs_float64_oracle(kind):
    """fm_overfit_step with the tracking loss."""
    from oracle import flowmap_oracle as O
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows, Tracks
    f, h, w = 6, 96, 192
    depth, wparam, fl, focal, tracks = _fused_case(kind, f, h, w)

    def oracle_step(dt):
        st = O.OverfitOracle(O.OverfitConfig(intrinsics="regressed", initial_focal=focal, use_tracking=True,
                                             tracking_enable_after=0), f, h, w, dtype=dt)
        with torch.no_grad():
            st.depth.copy_(depth.to(dt))
            st.weights.copy_(wparam.to(dt))
        flows = O.Flows(*(t.to(dt) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))
        r = st.training_step(flows, [O.Tracks(t.xy.to(dt), t.visibility, t.start_frame) for t in tracks])
        return dict(loss=r["loss"], ext=r["extrinsics"].double(), g_depth=r["grads"]["depth"].double(),
                    g_w=r["grads"]["weights"].double(), g_focal=float(r["grads"]["focal"]),
                    track=r["parts"]["tracking"])

    ref, ref32 = oracle_step(torch.float64), oracle_step(torch.float32)
    noise = errors(ref32, ref)
    batch = Batch(torch.zeros(1, 1, 1, 1, 1).expand(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    o = FusedOverfitter(OverfitCfg(initial_focal=focal, use_tracking=True, tracking_enable_after=0), batch,
                        Flows(*(t.float() for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask))),
                        [Tracks(t.xy.float(), t.visibility, t.start_frame) for t in tracks])
    with torch.no_grad():
        o.model.backbone.depth.copy_(depth.float())
        o.model.backbone.weights.copy_(wparam.float())
    loss, _ = o.training_step(update=False)
    gr = o.gradients()
    out = dict(loss=float(loss), ext=o.extrinsics().cpu(), g_depth=gr["depth"].cpu(), g_w=gr["weights"].cpu(),
               g_focal=float(gr["focal"]))
    label = f"fused {kind} {f}x{h}x{w} tracking"
    track_err = abs(float(o._track_loss) - ref["track"]) / abs(ref["track"])
    print(label, "tracking loss error", f"{track_err:.1e}")
    assert ref["track"] > 0 and track_err <= 1e-4, (label, track_err)
    check(errors(out, ref), noise, label, loss_tol=1e-4, pose_tol=2e-5, floor=1e-4)


@pytest.mark.parametrize("w", [136, 134])
def test_whole_frame_mapped_to_one_corner_stays_finite(w):
    """Every backward flow + (3, -2): every earlier-frame sample clips to the top-right corner, the
    Procrustes covariance is numerically zero and the rotation is arbitrary (the oracle's float32
    gradients are NaN there), so this is not a parity case.  The kernels must still give a finite
    loss and gradients and a proper rotation."""
    from oracle import flowmap_oracle as O
    from flowmap_b200 import ops
    b, f, h = 1, 3, 72
    depth, fl, focal, _ = O.flow_regime("iid", f, h, w, seed=9)
    wparam = 0.01 * torch.randn(b, f - 1, h, w, generator=torch.Generator().manual_seed(10))
    d = depth.float().cuda().requires_grad_(True)
    wp = wparam.cuda().requires_grad_(True)
    foc = torch.tensor(focal, device="cuda", requires_grad=True)
    s = (h * w) ** 0.5
    half = torch.tensor(0.5, device="cuda")
    k4 = torch.stack((foc * s / w, foc * s / h, half, half)).expand(b, f, 4)
    bwd = (fl.backward + torch.tensor([3.0, -2.0], dtype=torch.float64)).float().cuda()
    flc = [fl.forward.float().cuda(), bwd, fl.forward_mask.float().cuda(), fl.backward_mask.float().cuda()]
    rt = ops.procrustes_poses(d, torch.sigmoid(100.0 * wp), k4, flc[1], None)
    loss = ops.flow_loss(d, rt, k4, *flc, ops.mask_sum(flc[2], flc[3]), "huber", 0.01, 1000.0, "full")
    loss.backward()
    assert bool(torch.isfinite(loss)) and bool(torch.isfinite(rt).all())
    for g in (d.grad, wp.grad, foc.grad):
        assert bool(torch.isfinite(g).all())
    r = rt.detach()[0, :, :, :3].double().cpu()
    assert max_abs(r @ r.transpose(-1, -2), torch.eye(3, dtype=torch.float64).expand_as(r)) < 1e-5
    assert max_abs(torch.linalg.det(r), torch.ones(f - 1, dtype=torch.float64)) < 1e-5
