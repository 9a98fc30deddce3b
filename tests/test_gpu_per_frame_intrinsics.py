"""The Procrustes, flow-loss and tracking kernels, and the function-level projection surface, against the
float64 oracle under the intrinsics of calibrated videos: a K per frame, off-centre and anisotropic, and
a different K per video (flow_regime_checks.k4_regime).  Every other case of the suite shares one
focal-length K with the principal point at (0.5, 0.5) between all frames and videos; there a pair that
reads the wrong frame's or video's K, an intrinsics gradient booked on the wrong frame, or a principal
point taken as 0.5 gives the same numbers.  This is the path of `model/intrinsics: ground_truth`
(IntrinsicsGroundTruth, k_mode "const") and of ops.flow_loss's k_mode "full".

- The autograd ops: ops.procrustes_poses + ops.flow_loss in k_mode "full" and "const", at 2 x 4 x 96 x 192
  (scatter window), 2 x 3 x 72 x 136 (partial tiles) and 1 x 3 x 72 x 133 (dense backward), on the `iid`,
  `shift` and `leave` flows and a rigid scene whose flows are the induced flows at the true per-frame K;
  the index path on 1000 linspace points and on randint points with duplicates.
- ops.track_loss in both shared_k modes on 41-row segments, guarded by track_travel_checks.clear_track_kinks
  (a target's validity at the border now depends on K).
- The drop-in surface: Model with IntrinsicsGroundTruth and the explicit-depth backbone, LossFlow and
  LossTracking, on a Batch carrying the per-frame intrinsics, for 3 Adam steps.
- The function level: unproject (and ops.unproject_depth), project, reproject_points,
  compute_{forward,backward}_flow, both forms of align_surfaces, export.world_points.

Bars as in the rest of the suite: loss 1e-4 relative, poses 2e-5 absolute, every gradient metric max(1e-4,
3x the float32 oracle's error in the same metric), per frame, per pair and on the border band.  The
intrinsics gradient is checked per component and frame (flow_regime_checks.k4_errors)."""
import pytest
import torch

from conftest import max_abs, rel_l2
from flow_regime_checks import (check, errors, k4_errors, k4_regime, k4_scene, kmat, oracle_steps_k4,
                                start_point)
from oracle import flowmap_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _threads():
    torch.set_num_threads(min(16, torch.get_num_threads()))


def _inputs(kregime, flows, b, f, h, w, seed):
    """Float32-rounded (then float64) depth, weight logits, Flows and k4 of one case: the kernels get the
    same values as the oracle, so input rounding is not error."""
    k4 = k4_regime(kregime, b, f, h, w)
    if flows == "scene":
        depth, fl = k4_scene(k4, h, w, seed=seed)
    else:
        depth, fl, _, _ = O.flow_regime(flows, f, h, w, seed=seed, b=b)
    depth, _ = start_point(depth, 1.0, seed=seed + 1)
    wparam = 0.01 * torch.randn(b, f - 1, h, w, generator=torch.Generator().manual_seed(seed + 2), dtype=torch.float64)
    r = lambda t: t.float().double().contiguous()  # noqa: E731
    return r(depth), r(wparam), O.Flows(*(r(t) for t in (fl.forward, fl.backward, fl.forward_mask,
                                                         fl.backward_mask))), r(k4)


def _kernel_steps(depth, wparam, fl, k4, indices=None):
    """ops.procrustes_poses + ops.flow_loss in k_mode full and const: {mode: result}."""
    from flowmap_b200 import ops
    d = depth.float().to(DEV).requires_grad_(True)
    wp = wparam.float().to(DEV).requires_grad_(True)
    k = k4.float().to(DEV).requires_grad_(True)
    flc = [t.float().to(DEV) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)]
    idx = None if indices is None else indices.to(DEV)
    rt = ops.procrustes_poses(d, torch.sigmoid(100.0 * wp), k, flc[1], idx)
    ext = ops.pose_chain(rt.detach()).cpu()
    out = {}
    for mode in ("full", "const"):
        d.grad = wp.grad = k.grad = None
        loss = ops.flow_loss(d, rt, k, *flc, ops.mask_sum(flc[2], flc[3]), "huber", 0.01, 1000.0, mode)
        loss.backward(retain_graph=True)
        out[mode] = dict(loss=float(loss), ext=ext, g_depth=d.grad.cpu(), g_w=wp.grad.cpu(), g_focal=None,
                         g_k4=k.grad.cpu())
    return out


def _check_modes(out, refs, label):
    base = errors(refs[32], refs[64])
    for mode, gk in (("full", "g_k4"), ("const", "g_k4_const")):
        noise = dict(base, **k4_errors(refs[32][gk], refs[64][gk], noise=True))
        errs = errors(out[mode], refs[64])
        errs.update(k4_errors(out[mode]["g_k4"], refs[64][gk]))
        check(errs, noise, f"{label} {mode}", loss_tol=1e-4, pose_tol=2e-5, floor=1e-4)


SHAPES = [(2, 4, 96, 192),   # 3 x 3 tiles of 64 x 32 per frame: the scatter window
          (2, 3, 72, 136),   # partial tiles
          (1, 3, 72, 133)]   # W % 4 != 0: k_distribute_dense
CASES = ([("offcentre", fl, SHAPES[0]) for fl in ("iid", "shift", "leave", "scene")] +
         [("zoom", fl, SHAPES[0]) for fl in ("iid", "shift", "leave", "scene")] +
         [("corner", fl, SHAPES[0]) for fl in ("iid", "shift", "leave", "scene")] +
         [("videos", fl, SHAPES[0]) for fl in ("iid", "shift", "leave", "scene")] +
         [(k, "shift", SHAPES[1]) for k in ("offcentre", "zoom", "corner", "videos")] +
         [(k, fl, SHAPES[2]) for k in ("zoom", "corner") for fl in ("shift", "scene")])


@pytest.mark.parametrize("kregime,flows,shape", CASES, ids=[f"{k}-{fl}-{'x'.join(map(str, s))}" for k, fl, s in CASES])
def test_autograd_ops_vs_float64_oracle(kregime, flows, shape):
    """ops.procrustes_poses + ops.flow_loss (k_mode full and const) on all pixels."""
    b, f, h, w = shape
    depth, wparam, fl, k4 = _inputs(kregime, flows, b, f, h, w, seed=w + f)
    refs = oracle_steps_k4(depth, wparam, fl, k4)
    _check_modes(_kernel_steps(depth, wparam, fl, k4), refs, f"{kregime} {flows} {b}x{f}x{h}x{w}")


@pytest.mark.parametrize("points", ["linspace", "randint"])
@pytest.mark.parametrize("kregime", ["zoom", "corner", "videos"])
def test_index_path_vs_float64_oracle(kregime, points):
    """Procrustes on an explicit point set (the reference's 1000 linspace points; 1000 randint points, which
    repeat some pixels), the oracle on the same index tensor."""
    b, f, h, w = 2, 4, 96, 192
    depth, wparam, fl, k4 = _inputs(kregime, "shift", b, f, h, w, seed=41)
    if points == "linspace":
        idx = torch.linspace(0, h * w - 1, 1000, dtype=torch.int64)
    else:
        idx = torch.randint(0, h * w, (1000,), generator=torch.Generator().manual_seed(42))
        assert idx.unique().numel() < idx.numel()
    refs = oracle_steps_k4(depth, wparam, fl, k4, idx)
    _check_modes(_kernel_steps(depth, wparam, fl, k4, idx), refs, f"{kregime} {points} {b}x{f}x{h}x{w}")


# ---------------------------------------------------------------------------------------------- tracking
@pytest.mark.parametrize("kregime", ["offcentre", "zoom", "corner"])
def test_track_loss_vs_float64_oracle(kregime):
    """ops.track_loss on travel_scene's cameras (|t| to 10) with 1225-point uniform tracks on the reference's
    41-row segments: loss, valid count (exactly), depth gradient per frame and on the border band, pose
    twist per frame, and the intrinsics gradient per frame and component (shared_k False) or its sum over
    frames (shared_k True)."""
    import test_gpu_tracking_travel as TT
    from test_gpu_parity import twist
    f, h, w = 42, 96, 128
    depth, ext, _, tracks = TT._op_inputs(f, h, w, "uniform", seed=5)
    k4 = k4_regime(kregime, 1, f, h, w).float().double()
    label = f"track_loss {kregime} {f}x{h}x{w}"
    guarded, _, _, crossings = TT._guard(depth, ext, [ext], k4, tracks, label)
    assert crossings > 10_000, (label, crossings)
    ref, ref32 = TT._oracle(depth, ext, k4, guarded, torch.float64), TT._oracle(depth, ext, k4, guarded, torch.float32)
    rot = ext[0, :, :3, :3]
    ref_twist = twist(rot, ref["g_ext"])
    for shared in (False, True):
        out = TT._kernel(depth, ext, k4, guarded, shared)
        lab = f"{label} shared_k={shared}"
        assert out["count"] == ref["count"], (lab, "valid count", out["count"], ref["count"])
        errs = TT._op_errors(out, ref, rot, ref_twist, shared)
        noise = TT._op_errors(ref32, ref, rot, ref_twist, shared)
        if not shared:
            errs.update(k4_errors(out["g_k4"], ref["g_k4"]))
            noise.update(k4_errors(ref32["g_k4"], ref["g_k4"], noise=True))
        check(errs, noise, lab, loss_tol=1e-4, pose_tol=0.0, floor=1e-4)


# ---------------------------------------------------------------------------------------- drop-in surface
def _dropin_oracle(depth, wparam, fl, kmat64, tracks, steps, dt):
    cfg = O.OverfitConfig(intrinsics="ground_truth", use_tracking=True, tracking_enable_after=0)
    f, h, w = depth.shape
    st = O.OverfitOracle(cfg, f, h, w, dtype=dt, intrinsics=kmat64)
    with torch.no_grad():
        st.depth.copy_(depth.to(dt))
        st.weights.copy_(wparam.to(dt))
    flows = O.Flows(*(t.to(dt) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))
    trk = [O.Tracks(t.xy.to(dt), t.visibility, t.start_frame) for t in tracks]
    res = [st.training_step(flows, trk) for _ in range(steps)]
    return res, st


def _guarded_tracks(depth, wparam, fl, kmat64, tracks):
    """track_travel_checks.clear_track_kinks on the step-0 targets of the float64 oracle, with a band from the
    float32 oracle's position error: the predicted target's validity at the border depends on K, and a sample
    within rounding of it would be decided by rounding."""
    import track_travel_checks as TC
    from test_gpu_tracking_travel import _on
    f, h, w = depth.shape
    outs = []
    for dt in (torch.float64, torch.float32):
        st = O.OverfitOracle(O.OverfitConfig(intrinsics="ground_truth"), f, h, w, dtype=dt, intrinsics=kmat64)
        with torch.no_grad():
            st.depth.copy_(depth.to(dt))
            st.weights.copy_(wparam.to(dt))
            o = st.forward(O.Flows(*(t.to(dt) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask))), 0)
            outs.append(TC.track_triples(o.surfaces.to(DEV), o.extrinsics.to(DEV), o.intrinsics.to(DEV), _on(tracks, dt)))
    with torch.no_grad():
        tr64 = _on(tracks, torch.float64)
        band = TC.position_band(outs[0], outs[1], tr64)
        guarded, cleared = TC.clear_track_kinks(tr64, outs[0], band)
    samples = sum(int(t.visibility.sum()) for t in tracks)
    print(f"drop-in tracks: band {band:.1e}, guard cleared {cleared} of {samples} samples")
    assert cleared <= 0.01 * samples, (cleared, samples)
    return [O.Tracks(t.xy.cpu(), t.visibility.cpu(), t.start_frame) for t in guarded]


def _dropin_model(f, h, w, depth, wparam):
    from flowmap_b200.loss import LossFlowCfg, LossTrackingCfg, MappingHuberCfg, get_losses
    from flowmap_b200.model import (BackboneExplicitDepthCfg, ExtrinsicsProcrustesCfg, IntrinsicsGroundTruthCfg,
                                    Model, ModelCfg)
    model = Model(ModelCfg(BackboneExplicitDepthCfg("explicit_depth", 0.1, 100.0),
                           IntrinsicsGroundTruthCfg("ground_truth"), ExtrinsicsProcrustesCfg("procrustes", None, False),
                           True), f, (h, w)).to(DEV)
    with torch.no_grad():
        model.backbone.depth.copy_(depth.float())
        model.backbone.weights.copy_(wparam.float())
    huber = MappingHuberCfg("huber", 0.01)
    return model, get_losses([LossFlowCfg(0, 1000.0, "flow", huber), LossTrackingCfg(0, 100.0, "tracking", huber)])


def test_dropin_model_step0_vs_gt_intrinsics_golden():
    """The drop-in surface with IntrinsicsGroundTruth on the inputs of gt_intrinsics_f64.npz (the reference's
    Model in float64 with a K per frame, flow + tracking): step 0's loss, poses and gradients, with the
    reference's own float32 run (gt_intrinsics.npz) as the noise."""
    from conftest import load_golden
    from flowmap_b200.types import Batch, Flows, Tracks
    g64, g32 = load_golden("gt_intrinsics", True), load_golden("gt_intrinsics", False)
    f, h, w = g64["in_depth"].shape
    T_ = torch.as_tensor
    model, losses = _dropin_model(f, h, w, T_(g64["in_depth"]), T_(g64["in_wparam"]))
    batch = Batch(torch.zeros(1, f, 3, h, w, device=DEV), torch.arange(f, device=DEV)[None], ["s"], ["d"],
                  intrinsics=T_(g64["intrinsics"]).float().to(DEV))
    flows = Flows(*(T_(g64[k]).float().to(DEV) for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    trk = [Tracks(T_(g64[f"trk{i}_xy"]).float().to(DEV), T_(g64[f"trk{i}_vis"]).to(DEV), int(g64[f"trk{i}_start"]))
           for i in range(2)]
    out = model(batch, flows, 0)
    assert out.k_mode == "const" and type(out).__name__ == "ModelOutput", (type(out).__name__, out.k_mode)
    total = sum(l.forward(batch, flows, trk, out, 0) for l in losses)
    total.backward()

    def ref(g):
        return dict(loss=float(g["loss"]), ext=T_(g["extrinsics"]).double(), g_depth=T_(g["g_depth"]).double(),
                    g_w=T_(g["g_wparam"]).double(), g_focal=None)

    res = dict(loss=float(total), ext=out.extrinsics.detach().cpu(), g_depth=model.backbone.depth.grad.cpu(),
               g_w=model.backbone.weights.grad.cpu(), g_focal=None)
    check(errors(res, ref(g64)), errors(ref(g32), ref(g64)), "drop-in ground_truth vs gt_intrinsics_f64",
          loss_tol=1e-4, pose_tol=2e-5, floor=1e-4)


def test_dropin_model_with_ground_truth_intrinsics_vs_float64_oracle():
    """Model(IntrinsicsGroundTruth, explicit depth, Procrustes) + LossFlow + LossTracking on a Batch whose
    intrinsics change per frame: the per-op path in k_mode "const".  Step 0's loss, poses and gradients
    against the float64 OverfitOracle with the same K, then 3 Adam steps: every step's loss and the final
    depth and weights.  The tracks are guarded (_guarded_tracks)."""
    from flowmap_b200.types import Batch, Flows, Tracks
    f, h, w = 6, 72, 136
    depth, wparam, fl, k4 = _inputs("zoom", "scene", 1, f, h, w, seed=61)
    depth, wparam = depth[0], wparam[0]
    kmat64 = kmat(k4)
    tracks = [O.Tracks(t.xy.float().double(), t.visibility, t.start_frame)
              for t in O.synthetic_tracks(f, n_points=300, interval=3, radius=2, seed=62, dtype=torch.float64)]
    tracks = _guarded_tracks(depth, wparam, fl, kmat64, tracks)
    steps = 3
    ref, st64 = _dropin_oracle(depth, wparam, fl, kmat64, tracks, steps, torch.float64)
    ref32, st32 = _dropin_oracle(depth, wparam, fl, kmat64, tracks, steps, torch.float32)

    model, losses = _dropin_model(f, h, w, depth, wparam)
    batch = Batch(torch.zeros(1, f, 3, h, w, device=DEV), torch.arange(f, device=DEV)[None], ["s"], ["d"],
                  intrinsics=kmat64.float().to(DEV))
    flows = Flows(*(t.float().to(DEV) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))
    trk = [Tracks(t.xy.float().to(DEV), t.visibility.to(DEV), t.start_frame) for t in tracks]
    opt = torch.optim.Adam(model.parameters(), lr=3e-5)
    for step in range(steps):
        opt.zero_grad(set_to_none=True)
        out = model(batch, flows, step)
        assert out.k_mode == "const" and type(out).__name__ == "ModelOutput", (type(out).__name__, out.k_mode)
        total = sum(l.forward(batch, flows, trk, out, step) for l in losses)
        total.backward()
        label = f"drop-in ground_truth step {step}"
        err = abs(float(total) - ref[step]["loss"]) / abs(ref[step]["loss"])
        print(label, f"loss {float(total):.6e}: error {err:.1e}, float32 oracle "
                     f"{abs(ref32[step]['loss'] - ref[step]['loss']) / abs(ref[step]['loss']):.1e}")
        assert err <= 1e-4, (label, err)
        if step == 0:
            res = dict(loss=float(total), ext=out.extrinsics.detach().cpu(), g_depth=model.backbone.depth.grad.cpu(),
                       g_w=model.backbone.weights.grad.cpu(), g_focal=None)
            r64 = lambda r: dict(loss=r["loss"], ext=r["extrinsics"].double(), g_depth=r["grads"]["depth"].double(),  # noqa: E731
                                 g_w=r["grads"]["weights"].double(), g_focal=None)
            check(errors(res, r64(ref[0])), errors(r64(ref32[0]), r64(ref[0])), label, loss_tol=1e-4, pose_tol=2e-5,
                  floor=1e-4)
        opt.step()
    for name, p, p64, p32 in (("depth", model.backbone.depth, st64.depth, st32.depth),
                              ("weights", model.backbone.weights, st64.weights, st32.weights)):
        # the update of the parameters over the 3 steps (the parameters themselves agree to rounding)
        start = (depth if name == "depth" else wparam)
        e = rel_l2(p.detach().double().cpu() - start, p64.detach() - start)
        n = rel_l2(p32.detach().double() - start, p64.detach() - start)
        print(f"drop-in ground_truth after {steps} steps: {name} update error {e:.1e} (float32 oracle {n:.1e})")
        assert e <= max(1e-3, 3 * n), (name, e, n)


# ----------------------------------------------------------------------------------------- function level
def _points_case(seed=71):
    b, f, h, w = 2, 3, 20, 28
    k4 = k4_regime("videos", b, f, h, w).float().double()
    g = torch.Generator().manual_seed(seed)
    depth = (1.0 + torch.rand(b, f, h, w, generator=g, dtype=torch.float64)).float().double()
    return b, f, h, w, k4, depth, g


def test_unproject_values_and_gradients_vs_float64_oracle():
    """projection.unproject (fm_unproject_points / _bwd: g_z and g_K) and ops.unproject_depth
    (fm_unproject / _bwd) under per-frame, per-video K, against the oracle's K^-1 by autograd."""
    from flowmap_b200 import ops, projection as P
    b, f, h, w, k4, depth, g = _points_case()
    cot = torch.randn(b, f, h, w, 3, generator=g, dtype=torch.float64)

    def oracle(dt):
        z, k = (t.detach().to(dt).clone().requires_grad_(True) for t in (depth, k4))
        s = O.unproject(O.pixel_grid(h, w, dt), z, kmat(k)[:, :, None, None])
        (s * cot.to(dt)).sum().backward()
        return s.detach().double(), z.grad.double(), k.grad.double()

    (s64, gz64, gk64), (s32, gz32, gk32) = oracle(torch.float64), oracle(torch.float32)
    xy, _ = P.sample_image_grid((h, w), device=DEV)
    for name in ("projection.unproject", "ops.unproject_depth"):
        z = depth.float().to(DEV).requires_grad_(True)
        k = k4.float().to(DEV).requires_grad_(True)
        if name == "ops.unproject_depth":
            s = ops.unproject_depth(z, k)
        else:
            s = P.unproject(xy, z, kmat(k)[:, :, None, None])
        (s * cot.float().to(DEV)).sum().backward()
        es, ez, ek = rel_l2(s.detach().cpu(), s64), rel_l2(z.grad.cpu(), gz64), rel_l2(k.grad.cpu(), gk64)
        print(name, f"surfaces {es:.1e}, g_z {ez:.1e} ({rel_l2(gz32, gz64):.1e}), g_k4 {ek:.1e} "
                    f"({rel_l2(gk32, gk64):.1e})")
        assert es <= 2e-6, (name, es)
        assert ez <= max(1e-5, 3 * rel_l2(gz32, gz64)), (name, ez)
        errs, noise = k4_errors(k.grad.cpu(), gk64), k4_errors(gk32, gk64, noise=True)
        for key in errs:
            for i, (a, n) in enumerate(zip(errs[key], noise[key])):
                assert a <= max(1e-5, 3 * n), (name, key, i, a, n)


def test_project_reproject_and_induced_flows_vs_float64_oracle():
    """projection.project (with in_front, points in front of and behind the camera),
    reproject_points, compute_{forward,backward}_flow, and export.world_points under per-frame K."""
    from flowmap_b200 import export, projection as P
    b, f, h, w, k4, depth, g = _points_case(72)
    km = kmat(k4)
    ext = O.pose_chain(torch.stack([torch.stack([_rigid(g) for _ in range(f - 1)]) for _ in range(b)]))
    n = 500
    pts = torch.randn(b, f, n, 3, generator=g, dtype=torch.float64)
    pts[..., 2] = pts[..., 2].abs() + 0.5
    pts[:, :, :20, 2] = -pts[:, :, :20, 2]  # behind the camera: in_front False
    world = O.matvec(ext[:, :, None], O.to_homogeneous(pts))[..., :3]  # camera points moved to the world
    world = world.float().double()
    cam64 = O.matvec(torch.linalg.inv(ext)[:, :, None], O.to_homogeneous(world))[..., :3]
    xy64 = O.project_camera_space(cam64, km[:, :, None])
    front64 = cam64[..., 2] >= 0
    xy, front = P.project(world.float().to(DEV), ext.float().to(DEV)[:, :, None], km.float().to(DEV)[:, :, None])
    e = max_abs(xy.cpu(), xy64) / float(xy64.abs().max())
    print("project: xy error", f"{e:.1e}", "in_front mismatches", int((front.cpu() != front64).sum()))
    assert e <= 1e-5 and bool((front.cpu() == front64).all())

    # the nan_to_num branch (projection.py:56): camera-space points with z = -1e-5, so that z + eps is 0 in
    # float32, under identity extrinsics.  The reference's semantics there are its float32 arithmetic
    # (x / 0 -> +-1e8, 0 / 0 -> 0), so the float32 oracle is the reference for these points.
    edge = torch.randn(b, f, 8, 3, generator=g, dtype=torch.float64).float()
    edge[..., 2] = 1.0
    edge[:, :, :4, 2] = -1e-5
    edge[:, :, 4, :] = torch.tensor([0.0, 0.0, -1e-5])
    eye = torch.eye(4).expand(b, f, 1, 4, 4)
    xy32 = O.project_camera_space(edge, km.float()[:, :, None])
    xy, front = P.project(edge.to(DEV), eye.to(DEV), km.float().to(DEV)[:, :, None])
    assert bool((xy32.abs()[:, :, :5] > 1e6).any())  # the branch is reached
    assert torch.allclose(xy.cpu(), xy32, rtol=1e-6, atol=1e-6), (xy.cpu()[0, 0], xy32[0, 0])
    assert bool((front.cpu() == (edge[..., 2] >= 0)).all())

    xyz = pts.float().double()
    rel = torch.stack([torch.stack([_rigid(g) for _ in range(f)]) for _ in range(b)])
    xy64 = O.reproject(xyz, rel[:, :, None], km[:, :, None])
    xy = P.reproject_points(xyz.float().to(DEV), rel.float().to(DEV)[:, :, None], km.float().to(DEV)[:, :, None])
    fin = (O.matvec(rel[:, :, None], O.to_homogeneous(xyz))[..., 2]).abs() > 1e-2
    e = max_abs(xy.cpu()[fin], xy64[fin]) / float(xy64[fin].abs().max())
    print("reproject_points: error", f"{e:.1e}")
    assert e <= 1e-5

    surf = O.unproject(O.pixel_grid(h, w, torch.float64), depth, km[:, :, None, None]).float().double()
    for name, fn, ofn in (("forward", P.compute_forward_flow, O.forward_flow_positions),
                          ("backward", P.compute_backward_flow, O.backward_flow_positions)):
        r64 = ofn(surf, ext, km)
        r = fn(surf.float().to(DEV), ext.float().to(DEV), km.float().to(DEV)).cpu()
        e = max_abs(r[..., :2], r64)
        print(f"compute_{name}_flow: error {e:.1e}")
        assert e <= 2e-5, (name, e)

    wp64 = O.matvec(ext[0][:, None, None], O.to_homogeneous(surf[0]))[..., :3].reshape(-1, 3)
    wp = export.world_points(depth[0].float().to(DEV), km[0].float().to(DEV), ext[0].float().to(DEV)).cpu()
    e = max_abs(wp, wp64) / float(wp64.abs().max())
    print(f"export.world_points: error {e:.1e}")
    assert e <= 2e-6


def _rigid(g):
    a = 0.1 * torch.randn(3, generator=g, dtype=torch.float64)
    k = torch.zeros(3, 3, dtype=torch.float64)
    k[0, 1], k[0, 2], k[1, 2] = -a[2], a[1], -a[0]
    m = torch.eye(4, dtype=torch.float64)
    m[:3, :3] = torch.linalg.matrix_exp(k - k.T)
    m[:3, 3] = 0.2 * torch.randn(3, generator=g, dtype=torch.float64)
    return m


@pytest.mark.parametrize("form", ["surfaces", "depths"])
def test_align_surfaces_both_forms_vs_float64_oracle(form):
    """projection.align_surfaces(surfaces, flows, weights, indices) (gather + align_rigid kernel) and
    align_surfaces(depths, intrinsics, flows, weights) (the moment kernels) under per-frame, per-video K."""
    from flowmap_b200 import projection as P
    b, f, h, w = 2, 4, 72, 136
    depth, wparam, fl, k4 = _inputs("videos", "scene", b, f, h, w, seed=81)
    km = kmat(k4)
    wt = torch.sigmoid(100.0 * wparam)
    idx = torch.arange(h * w)

    def oracle(dt):
        s = O.unproject(O.pixel_grid(h, w, dt), depth.to(dt), km.to(dt)[:, :, None, None])
        return O.align_surfaces(s, fl.backward.to(dt), wt.to(dt), idx).double()

    e64, e32 = oracle(torch.float64), oracle(torch.float32)
    if form == "surfaces":
        s = O.unproject(O.pixel_grid(h, w, torch.float64), depth, km[:, :, None, None])
        out = P.align_surfaces(s.float().to(DEV), fl.backward.float().to(DEV), wt.float().to(DEV), idx.to(DEV))
    else:
        out = P.align_surfaces(depth.float().to(DEV), km.float().to(DEV), fl.backward.float().to(DEV),
                               wt.float().to(DEV))
    e, n = max_abs(out.cpu(), e64), max_abs(e32, e64)
    print(f"align_surfaces ({form}): pose error {e:.1e} (float32 oracle {n:.1e})")
    assert e <= max(2e-5, 3 * n)
