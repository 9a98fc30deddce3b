"""The tracking sweep (k_track_src -> k_track_apply / k_track_finalize) against the float64 oracle on the
reference's segment layout (interval 5, radius 20: 41-row segments) and on videos whose cameras travel far
from frame 0, as every real video's do.

The sweep lifts each source point to world space and brings it back per target frame, in float32; with
|t| of 10 - 40 against depths of 3 a world-scale cancellation would show here and nowhere else in the suite.
Every comparison runs on tracks guarded by track_travel_checks.clear_track_kinks (a target within rounding
of the [0,1)^2 border decides validity by rounding), and the valid count must then equal the float64
oracle's exactly.  Every oracle gets the kernel's float32 inputs upcast, so input rounding is not error.

- The op (ops.track_loss, both shared_k modes) at 42 x 96 x 128, 62 x 64 x 96 and 150 x 36 x 64 on
  travel_scene, with tracks consistent with the scene up to a small jitter (Huber's quadratic branch) and
  uniform random ones (its saturated branch): loss, depth gradient per frame and on the border band,
  pose twist per frame and the intrinsics gradient per frame (its sum over frames with shared_k).
- The gauge: every extrinsic left-multiplied by one rigid W with |W.t| in {0, 10, 100}.  Loss, count and
  depth gradient are invariant and the twists turn by W's rotation, so the kernel at each W is held to the
  W = I float64 result.
- The fused one-video step (FusedOverfitter, regressed focal length, tracking on), step 0, against the
  float64 OverfitOracle: the 42-frame `shift` video of test_gpu_packed_videos_at_scale.py with 300-point
  radius-20 tracks, and travel_scene at 150 x 36 x 64 with 1225-point consistent tracks.

Gradients are held to max(1e-4, 3 x the float32 oracle's error in the same metric)."""
import pytest
import torch

import track_travel_checks as T
from conftest import rel_l2
from oracle import flowmap_oracle as O
from flow_regime_checks import border_band, check, errors, start_point
from test_gpu_parity import twist

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
WEIGHT = 100.0  # loss/tracking.yaml
SHAPES = [(42, 96, 128), (62, 64, 96), (150, 36, 64)]
MAX_CLEARED = 0.01  # fraction of the visible samples the guard may clear


def _min_travel(f):
    """The least |t| of the last camera a case must reach: travel_scene moves 0.25 per frame."""
    return 0.24 * (f - 1)


@pytest.fixture(autouse=True)
def _threads():
    torch.set_num_threads(min(16, torch.get_num_threads()))


def _kmat(k4):
    """(1, F, 3, 3) intrinsics from k4 rows (fx, fy, cx, cy), differentiably."""
    z, o = torch.zeros_like(k4[..., 0]), torch.ones_like(k4[..., 0])
    return torch.stack((torch.stack((k4[..., 0], z, k4[..., 2]), -1), torch.stack((z, k4[..., 1], k4[..., 3]), -1),
                        torch.stack((z, z, o), -1)), -2)


def _surfaces(depth, k4, dt):
    h, w = depth.shape[-2:]
    kmat = _kmat(k4.to(DEV, dt))
    return O.unproject(O.pixel_grid(h, w, dt, DEV), depth.to(DEV, dt), kmat[:, :, None, None]), kmat


def _on(tracks, dt):
    return [O.Tracks(t.xy.to(DEV, dt), t.visibility.to(DEV), t.start_frame) for t in tracks]


def _op_inputs(f, h, w, kind, seed):
    """travel_scene's depth (1, f, h, w), extrinsics (1, f, 4, 4), k4 (1, f, 4) and 1225-point tracks on the
    reference's segments, all float32-rounded and upcast."""
    depth, _, focal, ext = T.travel_scene(f, h, w, seed=seed)
    if kind == "consistent":
        # moved by N(0, 0.003^2): residuals in Huber's quadratic branch (delta 0.01) yet far above rounding.
        # Exactly consistent tracks leave residuals of ~1e-6, and gradients that are rounding noise.
        g = torch.Generator().manual_seed(seed + 3)
        tracks = [O.Tracks(t.xy + 0.003 * torch.randn(t.xy.shape, generator=g, dtype=torch.float64), t.visibility,
                           t.start_frame)
                  for t in O.scene_tracks(depth, ext, focal, T.reference_segments(f), n_points=1225, seed=seed)]
    else:
        tracks = O.synthetic_tracks(f, 1225, seed=seed, dtype=torch.float64)
    tracks = [O.Tracks(t.xy.float().double(), t.visibility, t.start_frame) for t in tracks]
    s = (h * w) ** 0.5
    k4 = torch.tensor([focal * s / w, focal * s / h, 0.5, 0.5]).double().expand(1, f, 4).contiguous()
    return depth.float().double()[None], ext.float().double(), k4, tracks


def _guard(depth, ext64, exts32, k4, tracks, label):
    """clear_track_kinks with the float64 targets at ext64 and a band from the float32 oracle's position error
    at each of exts32.  Returns (guarded tracks on the CPU, float64 valid count before the guard, cleared,
    border crossings)."""
    with torch.no_grad():
        s64, k64 = _surfaces(depth, k4, torch.float64)
        tr64 = _on(tracks, torch.float64)
        t64 = T.track_triples(s64, ext64.to(DEV), k64, tr64)
        s32, k32 = _surfaces(depth, k4, torch.float32)
        tr32 = _on(tracks, torch.float32)
        band = max(T.position_band(t64, T.track_triples(s32, e.to(DEV, torch.float32), k32, tr32), tr64)
                   for e in exts32)
        crossings = T.border_crossings(tr64, t64)
        guarded, cleared = T.clear_track_kinks(tr64, t64, band)
        assert T.near_border_triples(guarded, t64, band) == 0
        count = sum(int(v.sum()) for _, v in t64)
    samples = sum(int(t.visibility.sum()) for t in tracks)
    print(label, f"band {band:.1e}, {crossings} border crossings, guard cleared {cleared} of {samples} samples")
    # the guard removes what rounding decides, not the data: at most 1 % of the samples (0.51 % measured, in
    # the gauge case whose band covers |W.t| = 100)
    assert cleared <= MAX_CLEARED * samples, (label, "guard cleared", cleared, samples)
    return [O.Tracks(t.xy.cpu(), t.visibility.cpu(), t.start_frame) for t in guarded], count, cleared, crossings


def _oracle(depth, ext, k4, tracks, dt):
    """Tracking loss x WEIGHT and its gradients by the oracle in dtype dt (on the device: a 150-frame video's
    segments hold 60 M triples), with the valid count."""
    d, e, k = (t.detach().to(DEV, dt).requires_grad_(True) for t in (depth, ext, k4))
    surf, kmat = _surfaces(d, k, dt)
    s_leaf, k_leaf = surf.detach().requires_grad_(True), kmat.detach().requires_grad_(True)
    loss, count = T.tracking_loss_by_segment(s_leaf, e, k_leaf, _on(tracks, dt), WEIGHT)
    ((surf * s_leaf.grad).sum() + (kmat * k_leaf.grad).sum()).backward()
    return dict(loss=loss, count=count, g_depth=d.grad[0].double().cpu(), g_ext=e.grad.double().cpu(),
                g_k4=k.grad[0].double().cpu())


def _kernel_count(d, e, k, pk, shared):
    """The valid count at the head of the tracking workspace (as test_gpu_round2's sharded sweep reads it)."""
    from flowmap_b200 import ops
    from flowmap_b200._lib import check as lib_check, lib
    L = lib()
    f, h, w = d.shape[1:]
    ws = torch.zeros(L.fm_track_workspace_bytes(f, pk.total), dtype=torch.uint8, device=DEV)
    P = lambda t: t.data_ptr()  # noqa: E731
    lib_check(L.fm_track_loss_fwd_sharded(P(d), P(k), P(e), P(pk.seg), pk.num_segments, pk.max_rows, pk.max_points,
                                          P(pk.xy), P(pk.vis), pk.total, ops.MAPPINGS["huber"], 0.01, WEIGHT, None,
                                          P(ws), f, h, w, 0, 0, f, int(shared), torch.cuda.current_stream().cuda_stream),
              "fm_track_loss_fwd_sharded")
    torch.cuda.synchronize()
    return int(ws[:16].view(torch.float64)[1])


def _kernel(depth, ext, k4, tracks, shared):
    from flowmap_b200 import ops
    pk = _packed(tracks)
    d, e, k = (t.float().to(DEV).contiguous().requires_grad_(True) for t in (depth, ext, k4))
    loss = ops.track_loss(d, e, k, pk, "huber", 0.01, WEIGHT, shared)
    loss.backward()
    return dict(loss=float(loss.detach()), count=_kernel_count(d.detach(), e.detach(), k.detach(), pk, shared),
                g_depth=d.grad[0].double().cpu(), g_ext=e.grad.double().cpu(), g_k4=k.grad[0].double().cpu())


def _op_errors(out, ref, out_rot, ref_twist, shared):
    """Loss; depth gradient whole, on the border band and per frame; pose twist per frame (out's at its own
    rotations out_rot, against ref_twist); intrinsics gradient per frame, or its sum over frames (shared)."""
    gd, rd = out["g_depth"], ref["g_depth"]
    band = border_band(*rd.shape[-2:])
    tw = twist(out_rot, out["g_ext"])
    e = dict(loss=abs(out["loss"] - ref["loss"]) / abs(ref["loss"]), pose=0.0, depth=rel_l2(gd, rd),
             depth_border=rel_l2(gd[:, band], rd[:, band]),
             depth_frame=[rel_l2(gd[i], rd[i]) for i in range(rd.shape[0])],
             twist_frame=[rel_l2(tw[i], ref_twist[i]) for i in range(rd.shape[0])])
    if shared:
        e["k4_sum"] = rel_l2(out["g_k4"].sum(0), ref["g_k4"].sum(0))
    else:
        e["k4_frame"] = [rel_l2(out["g_k4"][i], ref["g_k4"][i]) for i in range(rd.shape[0])]
    return e


def _noise(noise, kind):
    """The float32 oracle's errors as the bar's noise.  In Huber's quadratic branch ("consistent") the per-frame
    pose twist and intrinsics gradient are sums of terms of both signs that cancel to 1e-3 - 1e-2 of their size,
    and which frame a float32 summation order happens to get right varies: two orders (the kernel's per-lane
    and per-warp sums, torch's reductions) differ per frame by more than 3x while their worst frames agree.
    There every frame of those two metrics is held to 3x the float32 oracle's worst frame; the loss, count and
    depth gradient keep the per-frame bar."""
    if kind == "consistent":
        for key in ("twist_frame", "k4_frame"):
            if key in noise:
                noise[key] = [max(noise[key])] * len(noise[key])
    return noise


def _assert_reaches_purpose(label, ext, tracks, crossings, cleared, min_crossings):
    f = ext.shape[1]
    travel = float(ext[0, -1, :3, 3].norm())
    assert travel >= _min_travel(f), (label, "last camera's |t|", travel)
    assert max(t.xy.shape[1] for t in tracks) == 41, (label, "segment rows")
    assert crossings > min_crossings, (label, "border crossings", crossings)
    assert cleared > 0, (label, "the guard cleared nothing")


@pytest.mark.parametrize("kind", ["consistent", "uniform"])
@pytest.mark.parametrize("f,h,w", SHAPES, ids=[f"{f}x{h}x{w}" for f, h, w in SHAPES])
def test_track_loss_op_on_travelling_cameras(f, h, w, kind):
    """ops.track_loss in both shared_k modes against the float64 oracle, with the float32 oracle as the noise
    estimate, and the valid count exactly.  Without the guard the count mismatch is printed (not asserted):
    the flips it counts are what the guard removes."""
    depth, ext, k4, tracks = _op_inputs(f, h, w, kind, seed=f)
    label = f"track_loss {kind} {f}x{h}x{w}"
    guarded, count_unguarded, cleared, crossings = _guard(depth, ext, [ext], k4, tracks, label)
    _assert_reaches_purpose(label, ext, tracks, crossings, cleared, min_crossings=50_000)
    for shared in (False, True):
        raw = _kernel_count(*(t.float().to(DEV).contiguous() for t in (depth, ext, k4)),
                            _packed(tracks), shared)
        print(label, f"shared_k={shared} without the guard: valid count {raw} vs float64 {count_unguarded} "
                     f"({raw - count_unguarded:+d})")
    ref, ref32 = _oracle(depth, ext, k4, guarded, torch.float64), _oracle(depth, ext, k4, guarded, torch.float32)
    rot = ext[0, :, :3, :3]
    ref_twist = twist(rot, ref["g_ext"])
    for shared in (False, True):
        out = _kernel(depth, ext, k4, guarded, shared)
        lab = f"{label} shared_k={shared}"
        assert out["count"] == ref["count"], (lab, "valid count", out["count"], ref["count"])
        check(_op_errors(out, ref, rot, ref_twist, shared), _noise(_op_errors(ref32, ref, rot, ref_twist, shared), kind), lab,
              loss_tol=1e-4, pose_tol=0.0, floor=1e-4)


def _packed(tracks):
    from flowmap_b200 import ops
    from flowmap_b200.types import Tracks
    return ops.PackedTracks([Tracks(t.xy.float().to(DEV), t.visibility.to(DEV), t.start_frame) for t in tracks], DEV)


def _rigid(travel, seed):
    """A rigid motion (4, 4) with a random rotation of about 0.5 rad and |t| = travel."""
    g = torch.Generator().manual_seed(seed)
    a = 0.3 * torch.randn(3, generator=g, dtype=torch.float64)
    k = torch.zeros(3, 3, dtype=torch.float64)
    k[0, 1], k[0, 2], k[1, 2] = -a[2], a[1], -a[0]
    m = torch.eye(4, dtype=torch.float64)
    m[:3, :3] = torch.linalg.matrix_exp(k - k.T)
    d = torch.randn(3, generator=g, dtype=torch.float64)
    m[:3, 3] = travel * d / d.norm()
    return m


@pytest.mark.parametrize("kind", ["consistent", "uniform"])
def test_track_loss_gauge_invariance(kind):
    """The kernel on W ext (float32-rounded) for |W.t| in {0, 10, 100}, against the float64 oracle at W = I:
    the same loss, valid count and depth gradient, and twists turned by W's rotation.  The bar at each W is
    3x the float32 oracle's error under that W."""
    f, h, w = 42, 96, 128
    depth, ext, k4, tracks = _op_inputs(f, h, w, kind, seed=7)
    gauges = {travel: _rigid(travel, seed=int(travel) + 1) for travel in (0.0, 10.0, 100.0)}
    ext_w = {travel: (m @ ext).float().double() for travel, m in gauges.items()}
    label = f"gauge {kind} {f}x{h}x{w}"
    guarded, _, cleared, crossings = _guard(depth, ext, list(ext_w.values()), k4, tracks, label)
    _assert_reaches_purpose(label, ext, tracks, crossings, cleared, min_crossings=50_000)
    ref = _oracle(depth, ext, k4, guarded, torch.float64)
    ref_twist = twist(ext[0, :, :3, :3], ref["g_ext"])
    for travel, m in gauges.items():
        e = ext_w[travel]
        rot, wr = e[0, :, :3, :3], m[:3, :3]
        turned = torch.cat((ref_twist[:, :3] @ wr.T, ref_twist[:, 3:] @ wr.T), dim=-1)
        ref32 = _oracle(depth, e, k4, guarded, torch.float32)
        out = _kernel(depth, e, k4, guarded, False)
        lab = f"{label} |W.t| = {travel:g}"
        assert out["count"] == ref["count"], (lab, "valid count", out["count"], ref["count"])
        check(_op_errors(out, ref, rot, turned, False), _noise(_op_errors(ref32, ref, rot, turned, False), kind), lab,
              loss_tol=1e-4, pose_tol=0.0, floor=1e-4)


# ------------------------------------------------------------------------------------ fused one-video step
def _fused_video(case):
    """Float64 inputs of one video at its start point: depth (f,h,w), wparam (f-1,h,w), Flows, focal, tracks."""
    if case == "shift-42x176x224":
        # the 42-frame `shift` video of test_gpu_packed_videos_at_scale.py's LLFF cases (seed 5)
        from test_gpu_packed_videos_at_scale import _regime_video
        v = _regime_video("shift", 42, 176, 224, seed=5, focal_scale=1.1)
        tracks = O.synthetic_tracks(42, n_points=300, interval=5, radius=20, seed=5, dtype=torch.float64)
        return v["depth"], v["wparam"], v["flows"], v["focal"], tracks, None
    f, h, w = 150, 36, 64
    depth, fl, focal, ext = T.travel_scene(f, h, w, seed=3)
    tracks = O.scene_tracks(depth, ext, focal, T.reference_segments(f), n_points=1225, seed=3)
    wparam = 0.01 * torch.randn(f - 1, h, w, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    depth, focal = start_point(depth[None], focal, seed=5)
    return depth[0], wparam, fl, focal, tracks, ext


def _oracle_forward(depth, wparam, fl, focal, dt):
    """OverfitOracle (regressed focal length, tracking on) at step 0 in dtype dt: the model's forward."""
    f, h, w = depth.shape
    st = O.OverfitOracle(O.OverfitConfig(intrinsics="regressed", initial_focal=focal, use_tracking=True,
                                         tracking_enable_after=0), f, h, w, dtype=dt)
    with torch.no_grad():
        st.depth.copy_(depth.to(dt))
        st.weights.copy_(wparam.to(dt))
    flows = O.Flows(*(t.to(dt) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))
    return st, flows, st.forward(flows, 0)


def _oracle_step(st, flows, out, tracks):
    """The rest of OverfitOracle.training_step's gradients, with the tracking loss one segment at a time."""
    c = st.cfg
    flow = c.flow_weight * O.flow_loss(out.surfaces, out.extrinsics, out.intrinsics, flows, c.mapping, c.delta)
    leaves = [t.detach().to(DEV).requires_grad_(True) for t in (out.surfaces, out.extrinsics, out.intrinsics)]
    track, count = T.tracking_loss_by_segment(*leaves, _on(tracks, st.dtype), c.tracking_weight, c.mapping, c.delta)
    total = flow + sum((t * leaf.grad.cpu()).sum() for t, leaf in zip((out.surfaces, out.extrinsics, out.intrinsics),
                                                                        leaves))
    total.backward()
    return dict(loss=float(flow) + track, ext=out.extrinsics.detach().double()[0], g_depth=st.depth.grad.double(),
                g_w=st.weights.grad.double(), g_focal=float(st.focal.grad), track=track, count=count)


FUSED = ["shift-42x176x224", "travel-150x36x64"]


@pytest.mark.parametrize("case", FUSED)
def test_fused_step_tracking_on_travelling_cameras(case):
    """Step 0 of the fused one-video step against the float64 OverfitOracle, on tracks guarded with the float64
    oracle's own poses: loss, poses, gradients per frame / pair / border band, focal gradient, tracking loss,
    and the sweep's valid count (the head of the step's tracking workspace) exactly.  Loss and poses within 3x
    the float32 oracle's error where float32 itself misses the fixed tolerances (camera positions chained out
    to |t| ~ 10 - 40)."""
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows, Tracks
    depth, wparam, fl, focal, tracks, scene_ext = _fused_video(case)
    f, h, w = depth.shape
    tracks = [O.Tracks(t.xy.float().double(), t.visibility, t.start_frame) for t in tracks]
    fw64, fw32 = _oracle_forward(depth, wparam, fl, focal, torch.float64), \
        _oracle_forward(depth, wparam, fl, focal, torch.float32)
    label = f"fused {case}"
    with torch.no_grad():
        k64 = fw64[2].intrinsics.to(DEV)
        t64 = T.track_triples(fw64[2].surfaces.to(DEV), fw64[2].extrinsics.to(DEV), k64, _on(tracks, torch.float64))
        t32 = T.track_triples(fw32[2].surfaces.to(DEV), fw32[2].extrinsics.to(DEV), fw32[2].intrinsics.to(DEV),
                              _on(tracks, torch.float32))
        tr64 = _on(tracks, torch.float64)
        band = T.position_band(t64, t32, tr64)
        crossings = T.border_crossings(tr64, t64)
        guarded, cleared = T.clear_track_kinks(tr64, t64, band)
        flips = sum(int((a != b).sum()) for (_, a), (_, b) in zip(t64, t32))
        del t32
    guarded = [O.Tracks(t.xy.cpu(), t.visibility.cpu(), t.start_frame) for t in guarded]
    samples = sum(int(t.visibility.sum()) for t in tracks)
    print(label, f"band {band:.1e}, {crossings} border crossings, {flips} float32 / float64 validity flips "
                 f"unguarded, guard cleared {cleared} of {samples} samples")
    assert cleared <= MAX_CLEARED * samples, (label, "guard cleared", cleared, samples)
    ext = fw64[2].extrinsics.detach()
    if scene_ext is not None:
        ext = scene_ext  # the scene's cameras; the poses the step recovers are the same up to the fit
    _assert_reaches_purpose(label, ext, tracks, crossings, cleared, min_crossings=20_000)
    ref, ref32 = _oracle_step(*fw64, guarded), _oracle_step(*fw32, guarded)

    batch = Batch(torch.zeros(1, 1, 1, 1, 1).expand(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    o = FusedOverfitter(OverfitCfg(intrinsics="regressed", initial_focal=focal, use_tracking=True,
                                   tracking_enable_after=0), batch,
                        Flows(*(t.float() for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask))),
                        [Tracks(t.xy.float(), t.visibility, t.start_frame) for t in guarded])
    with torch.no_grad():
        o.model.backbone.depth.copy_(depth.float())
        o.model.backbone.weights.copy_(wparam.float())
    loss, _ = o.training_step(update=False)
    gr = o.gradients()
    out = dict(loss=float(loss), ext=o.extrinsics().cpu(), g_depth=gr["depth"].cpu(), g_w=gr["weights"].cpu(),
               g_focal=float(gr["focal"]))
    count = int(o._tws[:16].view(torch.float64)[1])
    assert count == ref["count"], (label, "valid count", count, ref["count"])
    track_err = abs(float(o._track_loss) - ref["track"]) / abs(ref["track"])
    print(label, f"tracking loss {ref['track']:.4e}: error {track_err:.1e}, float32 oracle "
                 f"{abs(ref32['track'] - ref['track']) / abs(ref['track']):.1e}")
    assert ref["track"] > 0 and track_err <= 1e-4, (label, "tracking loss", track_err)
    noise = errors(ref32, ref)
    relative = noise["pose"] > 2e-5
    if relative:
        print(label, f"float32 oracle's pose error {noise['pose']:.1e} > 2e-5: loss and poses within 3x it")
    check(errors(out, ref), noise, label, loss_tol=1e-4, pose_tol=2e-5, floor=1e-4, relative_fixed=relative)
