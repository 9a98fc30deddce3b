"""The constant-intrinsics step (FusedOverfitter with cfg.intrinsics "ground_truth": fm_overfit_step with focal =
g_k4 = track_g_k4 = NULL) against the float64 OverfitOracle(intrinsics="ground_truth") in the flow regimes, at
partial tiles and odd widths, on the index path, at the reference's 41-row track segments and on packed layouts.

The mode runs its own kernel instantiations, compiled separately from the K-carrying ones the per-op tests check
and reached only from the fused step: k_distribute_window<false>, k_distribute_dense<false> and k_distribute<1,
false> (the Procrustes backward's all-pixel W % 4 == 0, all-pixel W % 4 != 0 and index paths), k_track_src<true,
false> and k_track_finalize<TL, false> (the tracking sweep), each for one video and for packed videos.  Every case
here runs the step once against the float64 oracle, and also with scratch g_k4 / track_g_k4 buffers (the
K-carrying kernels, whose intrinsics gradient is thrown away) against its own run-to-run noise.  Packed videos are
held to each video's own float64 run, not to their solo runs, so a fault both layouts share does not pass.
test_every_k_free_instantiation_runs checks by name that the intended kernels ran and no K-carrying one did.

Bars as in the rest of the suite: loss 1e-4 relative; poses 2e-5 absolute (3x the float32 oracle's error where
float32 itself misses that: far-travelling cameras); every gradient metric max(1e-4, 3x the float32 oracle's
error), per frame, per pair and on the border band (flow_regime_checks.errors / check); tracking loss 1e-4
relative; the sweep's valid count equal to the oracle's.  Tracks are guarded (track_travel_checks.clear_track_kinks
with the float32 oracle's position error as the band) and the guard may clear at most 1 % of the samples.  Every
input is float32-rounded before it reaches either side."""
import pytest
import torch

import test_gpu_fused_ground_truth_intrinsics as GT
import test_gpu_per_frame_intrinsics as PF
import track_travel_checks as T
from conftest import rel_l2
from flow_regime_checks import check, errors, k4_regime, k4_scene, kmat, start_point
from oracle import flowmap_oracle as O
from test_gpu_tracking_travel import _fused_video, _on

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
MAX_CLEARED = 0.01


@pytest.fixture(autouse=True)
def _threads():
    torch.set_num_threads(min(16, torch.get_num_threads()))


def _r(t):
    return t.float().double().contiguous()


def _cfg(**kw):
    return GT._cfg(use_tracking=True, tracking_enable_after=0, **kw)


def _tracks(f, seed, interval=3, radius=2, n_points=300):
    return [O.Tracks(_r(t.xy), t.visibility, t.start_frame)
            for t in O.synthetic_tracks(f, n_points=n_points, interval=interval, radius=radius, seed=seed,
                                        dtype=torch.float64)]


def _video(kregime, flows, f, h, w, seed, k4=None):
    """Float32-rounded depth (f, h, w), weight logits (f-1, h, w), Flows (1, f-1, ...) and K (1, f, 3, 3) of one
    video: PF._inputs for the flow regimes and k4_scene ("scene"), oracle.depth_regime for "depth_<kind>"."""
    if flows.startswith("depth_"):
        depth, fl, _, wparam = O.depth_regime(flows[6:], f, h, w, seed=seed)
        k4 = k4_regime(kregime, 1, f, h, w) if k4 is None else k4
        fl = O.Flows(*(_r(t) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))
        depth, wparam, k4 = _r(depth), _r(wparam), _r(k4)
    elif k4 is not None:  # a given K (one video of the `videos` regime)
        depth, fl, _, _ = O.flow_regime(flows, f, h, w, seed=seed)
        depth, _ = start_point(depth, 1.0, seed=seed + 1)
        wparam = 0.01 * torch.randn(1, f - 1, h, w, generator=torch.Generator().manual_seed(seed + 2),
                                    dtype=torch.float64)
        fl = O.Flows(*(_r(t) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))
        depth, wparam, k4 = _r(depth), _r(wparam), _r(k4)
    else:
        depth, wparam, fl, k4 = PF._inputs(kregime, flows, 1, f, h, w, seed=seed)
    return depth[0], wparam[0], fl, kmat(k4)


# ------------------------------------------------------------------------------------------------ oracle
def _oracle_forward(depth, wparam, fl, kmat64, dt, idx=None, **kw):
    f, h, w = depth.shape
    st = O.OverfitOracle(O.OverfitConfig(intrinsics="ground_truth", use_tracking=True, tracking_enable_after=0, **kw),
                         f, h, w, dtype=dt, intrinsics=kmat64)
    with torch.no_grad():
        st.depth.copy_(depth.to(dt))
        st.weights.copy_(wparam.to(dt))
    flows = O.Flows(*(t.to(dt) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))
    return st, flows, st.forward(flows, 0, procrustes_idx=idx)


def _oracle_step(st, flows, out, tracks):
    """Loss, poses and gradients of step 0, the tracking loss one segment at a time (on the device)."""
    c = st.cfg
    flow = c.flow_weight * O.flow_loss(out.surfaces, out.extrinsics, out.intrinsics, flows, c.mapping, c.delta)
    leaves = [t.detach().to(DEV).requires_grad_(True) for t in (out.surfaces, out.extrinsics)]
    track, count = T.tracking_loss_by_segment(*leaves, out.intrinsics.detach().to(DEV), _on(tracks, st.dtype),
                                              c.tracking_weight, c.mapping, c.delta)
    total = flow + sum((t * leaf.grad.cpu()).sum() for t, leaf in zip((out.surfaces, out.extrinsics), leaves))
    total.backward()
    g_w = st.weights.grad
    return dict(loss=float(flow) + track, ext=out.extrinsics.detach().double()[0], g_depth=st.depth.grad.double(),
                g_w=torch.zeros_like(st.weights, dtype=torch.float64) if g_w is None else g_w.double(), g_focal=None,
                track=track, count=count)


def _reference(depth, wparam, fl, kmat64, tracks, label, idx=None, **kw):
    """(guarded tracks, float64 result, float32 result) of step 0.  The guard's band is the float32 oracle's
    predicted-target error (track_travel_checks.position_band)."""
    fw = [_oracle_forward(depth, wparam, fl, kmat64, dt, idx, **kw) for dt in (torch.float64, torch.float32)]
    with torch.no_grad():
        trip = [T.track_triples(o.surfaces.to(DEV), o.extrinsics.to(DEV), o.intrinsics.to(DEV), _on(tracks, st.dtype))
                for st, _, o in fw]
        tr64 = _on(tracks, torch.float64)
        band = T.position_band(trip[0], trip[1], tr64)
        guarded, cleared = T.clear_track_kinks(tr64, trip[0], band)
        del trip
    samples = sum(int(t.visibility.sum()) for t in tracks)
    print(label, f"band {band:.1e}, guard cleared {cleared} of {samples} samples")
    assert cleared <= MAX_CLEARED * samples, (label, "guard cleared", cleared, samples)
    guarded = [O.Tracks(t.xy.cpu(), t.visibility.cpu(), t.start_frame) for t in guarded]
    return guarded, _oracle_step(*fw[0], guarded), _oracle_step(*fw[1], guarded)


def _check(out, ref, ref32, label, relative=False):
    noise = errors(ref32, ref)
    relative = relative or noise["pose"] > 2e-5
    check(errors(out, ref), noise, label, loss_tol=1e-4, pose_tol=2e-5, floor=1e-4, relative_fixed=relative)
    err = abs(out["track"] - ref["track"]) / abs(ref["track"])
    print(label, f"tracking loss {ref['track']:.4e}: error {err:.1e} (float32 oracle "
                 f"{abs(ref32['track'] - ref['track']) / abs(ref['track']):.1e})")
    assert ref["track"] > 0 and err <= 1e-4, (label, "tracking loss", err)
    if "count" in out:
        assert out["count"] == ref["count"], (label, "valid count", out["count"], ref["count"])


# ------------------------------------------------------------------------------------------------ fused
def _one(cfg, depth, wparam, fl, kmat64, tracks):
    o = GT._fused(cfg, GT._batch(*depth.shape, kmat64.float().to(DEV)), GT._flows(fl), GT._device_tracks(tracks),
                  depth, wparam)
    assert o._args.g_k4 is None and o._args.track_g_k4 is None
    return o


def _result(o, i=None):
    """Step-0 result of the last training_step(update=False): the one video's, or video i's of packed videos
    (whose valid count is not kept at the head of the tracking workspace)."""
    g = o.gradients()
    if i is None:
        return dict(loss=float(o._total), ext=o.extrinsics().cpu(), g_depth=g["depth"].cpu(), g_w=g["weights"].cpu(),
                    g_focal=None, track=float(o._track_loss), count=int(o._tws[:16].view(torch.float64)[1]))
    return dict(loss=float(o._total[i]), ext=o.extrinsics()[i].cpu(), g_depth=g["depth"][i].cpu(),
                g_w=g["weights"][i].cpu(), g_focal=None, track=float(o._track_loss[i]))


def _k_carrying_agrees(o, label):
    """The same step with scratch g_k4 / track_g_k4 (the K-carrying kernels) against the K-free step: loss, rt,
    the depth gradient per frame and the weight gradient per pair within 3x the K-free step's own run-to-run
    difference (floors: loss 1e-6 relative, rt 1e-6, gradients 1e-5)."""
    h, w = o._hw
    weights = o._args.weight_logits is not None

    def run():
        o.training_step(update=False)
        return (o._total.double().cpu().reshape(-1), o.rt.cpu().reshape(-1, 12), o._g_depth.cpu().reshape(-1, h, w),
                o._g_w.cpu().reshape(-1, h, w) if weights else None)

    def diffs(x, y):
        d = [float(((x[0] - y[0]).abs() / y[0].abs()).max()), float((x[1] - y[1]).abs().max()),
             max(rel_l2(a, b) for a, b in zip(x[2], y[2]))]
        if weights:
            d.append(max(rel_l2(a, b) for a, b in zip(x[3], y[3])))
        return d

    a, b = run(), run()
    k4, tk4 = torch.empty(o.T, 4, device=DEV), torch.empty(o.T, 4, device=DEV)
    o._args.g_k4, o._args.track_g_k4 = k4.data_ptr(), tk4.data_ptr()
    try:
        c = run()
    finally:
        o._args.g_k4 = o._args.track_g_k4 = None
    assert bool(torch.isfinite(k4).all()) and float(k4.abs().sum()) > 0, label  # the K path ran
    noise, err = diffs(b, a), diffs(c, a)
    print(label, "K-carrying vs constant K (loss, rt, g_depth frame, g_weights pair):", [f"{e:.1e}" for e in err],
          "run to run:", [f"{e:.1e}" for e in noise])
    for name, e, n, floor in zip(("loss", "rt", "g_depth", "g_weights"), err, noise, (1e-6, 1e-6, 1e-5, 1e-5)):
        assert e <= max(floor, 3 * n), (label, name, e, n)


def _run_one(kregime, flows, shape, seed, label, **kw):
    f, h, w = shape
    depth, wparam, fl, kmat64 = _video(kregime, flows, f, h, w, seed)
    tracks, ref, ref32 = _reference(depth, wparam, fl, kmat64, _tracks(f, seed + 5), label, **kw)
    o = _one(_cfg(**kw), depth, wparam, fl, kmat64, tracks)
    o.training_step(update=False)
    out = _result(o)
    if not kw.get("use_correspondence_weights", True):
        out["g_w"] = ref["g_w"] = ref32["g_w"]  # no weights: no weight gradient
    _check(out, ref, ref32, label)
    _k_carrying_agrees(o, label)


# ------------------------------------------------------------------------------ A. one video, all pixels
WIN, PART, DENSE, DENSE_H = (6, 96, 192), (6, 72, 136), (6, 72, 133), (5, 38, 63)
CASES = ([("zoom", fl, WIN) for fl in ("iid", "shift", "leave", "outliers", "zoom", "scene")] +
         [(k, fl, WIN) for k in ("offcentre", "corner") for fl in ("shift", "scene")] +
         [("zoom", fl, PART) for fl in ("shift", "outliers")] +
         [("zoom", fl, s) for s in (DENSE, DENSE_H) for fl in ("shift", "outliers", "scene")] +
         [("zoom", fl, WIN) for fl in ("depth_centre_far", "depth_horizon")])


@pytest.mark.parametrize("kregime,flows,shape", CASES, ids=[f"{k}-{fl}-{'x'.join(map(str, s))}" for k, fl, s in CASES])
def test_one_video_step0_vs_float64_oracle(kregime, flows, shape):
    """Step 0 on every pixel: 6 x 96 x 192 takes k_distribute_window<false> (3 x 3 tiles, the zoom flows' taps in
    the last column leave the window), 72 x 136 partial tiles, W = 133 and 5 x 38 x 63 (H % 4 != 0 too)
    k_distribute_dense<false>; `scene` is k4_scene (the induced flows at the true per-frame K); the depth regimes
    set the fixed-point quantum through the conditioning depth z0."""
    _run_one(kregime, flows, shape, seed=shape[2] + len(flows), label=f"{kregime} {flows} {'x'.join(map(str, shape))}")


@pytest.mark.parametrize("shape", [WIN, DENSE], ids=["window", "dense"])
def test_one_video_without_correspondence_weights(shape):
    """use_correspondence_weights=False: the step's weight_logits == NULL path, every weight 1."""
    _run_one("zoom", "shift", shape, seed=17, label=f"no weights {'x'.join(map(str, shape))}",
             use_correspondence_weights=False)


# ----------------------------------------------------------------------------------------- B. index path
@pytest.mark.parametrize("shape", [(6, 96, 192), (6, 72, 133)], ids=["96x192", "72x133"])
def test_index_path_linspace_vs_float64_oracle(shape):
    """procrustes_points=1000 (k_distribute<1, false>), the oracle on the device's own index tensor (CUDA's
    linspace can round differently from the CPU's)."""
    f, h, w = shape
    label = f"linspace 1000 {f}x{h}x{w}"
    depth, wparam, fl, kmat64 = _video("zoom", "shift", f, h, w, seed=23)
    cfg = _cfg(procrustes_points=1000)
    probe = _one(cfg, depth, wparam, fl, kmat64, _tracks(f, 24))
    idx = probe._indices.cpu()
    assert idx.numel() == 1000
    tracks, ref, ref32 = _reference(depth, wparam, fl, kmat64, _tracks(f, 24), label, idx=idx)
    o = _one(cfg, depth, wparam, fl, kmat64, tracks)
    assert torch.equal(o._indices.cpu(), idx)
    o.training_step(update=False)
    _check(_result(o), ref, ref32, label)
    _k_carrying_agrees(o, label)


def test_index_path_randint_with_duplicates_vs_float64_oracle():
    """1000 randint points (some pixels repeat) substituted for the step's indices."""
    f, h, w = 6, 96, 192
    label = "randint 1000 6x96x192"
    depth, wparam, fl, kmat64 = _video("corner", "scene", f, h, w, seed=29)
    idx = torch.randint(0, h * w, (1000,), generator=torch.Generator().manual_seed(30))
    assert idx.unique().numel() < idx.numel()
    tracks, ref, ref32 = _reference(depth, wparam, fl, kmat64, _tracks(f, 31), label, idx=idx,
                                    procrustes_points=1000)
    o = _one(_cfg(procrustes_points=1000), depth, wparam, fl, kmat64, tracks)
    o._indices = idx.to(DEV)
    o.training_step(update=False)
    _check(_result(o), ref, ref32, label)
    _k_carrying_agrees(o, label)


def test_index_path_randomized_adam_steps_vs_float64_oracle():
    """procrustes_randomize=True for 3 eager update steps, each step's randint points (with duplicates) handed to
    the oracle: step 0 in full, every step's loss, and the depth and weight updates over the 3 steps (bar
    max(1e-3, 3x float32)).  The tracks are guarded at the step-0 parameters under each of the three point sets."""
    f, h, w = 6, 72, 136
    steps, label = 3, "randomize 6x72x136"
    depth, wparam, fl, kmat64 = _video("zoom", "scene", f, h, w, seed=37)
    g = torch.Generator().manual_seed(38)
    sets = [torch.randint(0, h * w, (1000,), generator=g) for _ in range(steps)]
    assert all(s.unique().numel() < s.numel() for s in sets)
    tracks = _tracks(f, 39)
    kw = dict(procrustes_points=1000, procrustes_randomize=True)
    with torch.no_grad():
        tr64 = _on(tracks, torch.float64)
        trip = []
        for s in sets:
            for dt in (torch.float64, torch.float32):
                _, _, out = _oracle_forward(depth, wparam, fl, kmat64, dt, s, **kw)
                trip.append(T.track_triples(out.surfaces.to(DEV), out.extrinsics.to(DEV), out.intrinsics.to(DEV),
                                            _on(tracks, dt)))
        band = max(T.position_band(trip[i], trip[i + 1], tr64) for i in range(0, len(trip), 2))
        cleared = 0
        for t64 in trip[::2]:
            tr64, n = T.clear_track_kinks(tr64, t64, band)
            cleared += n
        del trip
    samples = sum(int(t.visibility.sum()) for t in tracks)
    print(label, f"band {band:.1e}, guard cleared {cleared} of {samples} samples")
    assert cleared <= MAX_CLEARED * samples, (label, cleared, samples)
    tracks = [O.Tracks(t.xy.cpu(), t.visibility.cpu(), t.start_frame) for t in tr64]

    def oracle(dt):
        st = O.OverfitOracle(O.OverfitConfig(intrinsics="ground_truth", use_tracking=True, tracking_enable_after=0,
                                             **kw), f, h, w, dtype=dt, intrinsics=kmat64)
        with torch.no_grad():
            st.depth.copy_(depth.to(dt))
            st.weights.copy_(wparam.to(dt))
        flows = O.Flows(*(t.to(dt) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))
        trk = [O.Tracks(t.xy.to(dt), t.visibility, t.start_frame) for t in tracks]
        return [st.training_step(flows, trk, procrustes_idx=s) for s in sets], st

    (r64, st64), (r32, st32) = oracle(torch.float64), oracle(torch.float32)
    o = _one(_cfg(**kw), depth, wparam, fl, kmat64, tracks)
    queue = [s.to(DEV) for s in sets]
    o.model.extrinsics.select_indices = lambda *_: queue.pop(0)
    for step in range(steps):
        total, _ = o.training_step()
        assert torch.equal(o._indices.cpu(), sets[step])
        err = abs(float(total) - r64[step]["loss"]) / abs(r64[step]["loss"])
        n = abs(r32[step]["loss"] - r64[step]["loss"]) / abs(r64[step]["loss"])
        print(f"{label} step {step}: loss error {err:.1e} (float32 oracle {n:.1e})")
        assert err <= 1e-4, (label, step, err)
        if step == 0:
            gr = o.gradients()
            red = lambda r: dict(loss=r["loss"], ext=r["extrinsics"].double()[0], g_depth=r["grads"]["depth"].double(),  # noqa: E731
                                 g_w=r["grads"]["weights"].double(), g_focal=None)
            out = dict(loss=float(total), ext=o.extrinsics().cpu(), g_depth=gr["depth"].cpu(), g_w=gr["weights"].cpu(),
                       g_focal=None)
            check(errors(out, red(r64[0])), errors(red(r32[0]), red(r64[0])), f"{label} step 0", loss_tol=1e-4,
                  pose_tol=2e-5, floor=1e-4)
    _updates(label, [(o.model.backbone.depth, st64.depth, st32.depth, depth),
                     (o.model.backbone.weights, st64.weights, st32.weights, wparam)])


def _updates(label, params):
    for name, (p, p64, p32, start) in zip(("depth", "weights"), params):
        e = rel_l2(p.detach().double().cpu() - start, p64.detach() - start)
        n = rel_l2(p32.detach().double() - start, p64.detach() - start)
        print(f"{label}: {name} update error {e:.1e} (float32 oracle {n:.1e})")
        assert e <= max(1e-3, 3 * n), (label, name, e, n)


# ---------------------------------------------------------------------- C. tracking at 41-row segments
@pytest.mark.parametrize("case", ["travel-150x36x64", "scene-42x48x64"])
def test_reference_segments_vs_float64_oracle(case):
    """Interval 5, radius 20 (41-row segments: the sweep's fold crosses 32 rows).  travel_scene's 150 frames with
    1225 consistent tracks under the scene's own K (cameras to |t| ~ 37: loss and poses within 3x float32), and a
    42-frame k4_scene under the `zoom` K with uniform tracks."""
    if case.startswith("travel"):
        depth, wparam, fl, focal, tracks, _ = _fused_video(case)
        f, h, w = depth.shape
        # start_point's 1.05 undone: the scene's own focal length
        kmat64 = O.intrinsics_from_focal(torch.tensor(focal / 1.05, dtype=torch.float64), h, w).expand(1, f, 3, 3)
        depth, wparam, kmat64 = _r(depth), _r(wparam), _r(kmat64)
        fl = O.Flows(*(_r(t) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))
        tracks = [O.Tracks(_r(t.xy), t.visibility, t.start_frame) for t in tracks]
    else:
        f, h, w = 42, 48, 64
        # k4_scene at a third of its default motion: over 42 frames the default's float32 poses drift so far that
        # the guard would clear more than 1 % of the samples
        k4 = k4_regime("zoom", 1, f, h, w)
        depth, fl = k4_scene(k4, h, w, seed=43, rotation=0.03, translation=0.1)
        depth, _ = start_point(depth, 1.0, seed=44)
        wparam = 0.01 * torch.randn(f - 1, h, w, generator=torch.Generator().manual_seed(45), dtype=torch.float64)
        depth, wparam, kmat64 = _r(depth[0]), _r(wparam), _r(kmat(k4))
        fl = O.Flows(*(_r(t) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))
        tracks = _tracks(f, 44, interval=5, radius=20)
    assert max(t.xy.shape[1] for t in tracks) == 41
    tracks, ref, ref32 = _reference(depth, wparam, fl, kmat64, tracks, case)
    o = _one(_cfg(), depth, wparam, fl, kmat64, tracks)
    o.training_step(update=False)
    _check(_result(o), ref, ref32, case, relative=case.startswith("travel"))
    _k_carrying_agrees(o, case)


# ------------------------------------------------------------------------- D. packed videos vs the oracle
def _packed_video(i, f, h, w, seed):
    """Video i of a packed case: its own K from the `videos` regime, `shift` flows, its own tracks."""
    k4 = k4_regime("videos", 2, f, h, w)[i % 2][None]
    depth, wparam, fl, kmat64 = _video("videos", "shift", f, h, w, seed + 10 * i, k4=k4)
    return depth, wparam, fl, kmat64, _tracks(f, seed + 10 * i + 5)


def _packed(cfg, vids, tensor_batch, graph=False):
    from flowmap_b200.overfit import FusedOverfitter
    from flowmap_b200.types import Flows
    f, h, w = vids[0][0].shape
    trk = [GT._device_tracks(v[4]) for v in vids]
    if tensor_batch:
        batch = GT._batch(f, h, w, torch.cat([v[3] for v in vids]).float().to(DEV), b=len(vids))
        flows = Flows(*(torch.cat([getattr(v[2], n) for v in vids]).float().to(DEV)
                        for n in ("forward", "backward", "forward_mask", "backward_mask")))
    else:
        batch = [GT._batch(v[0].shape[0], h, w, v[3].float().to(DEV)) for v in vids]
        flows = [GT._flows(v[2]) for v in vids]
    o = FusedOverfitter(cfg, batch, flows, trk, device=DEV)
    o._clock.base_seed = GT.SEED
    with torch.no_grad():
        for m, v in zip(o.models, vids):
            m.backbone.depth.copy_(v[0].float())
            m.backbone.weights.copy_(v[1].float())
    o.use_cuda_graph = graph
    assert o._args.g_k4 is None and o._args.track_g_k4 is None
    return o


PACKED = [("tensor", (6, 96, 192)), ("tensor", (6, 72, 133)), ("list", 96), ("list", 133)]


@pytest.mark.parametrize("layout,shape", PACKED, ids=["tensor-6x96x192", "tensor-6x72x133", "list-w96", "list-w133"])
def test_packed_videos_step0_vs_float64_oracle(layout, shape):
    """A (2, F) tensor batch, and a list of Batches of 5, 2 and 7 frames (H = 40): every video against its own
    float64 run with its own per-frame K and tracks.  W = 96 / 192 takes k_distribute_window<false, packed>,
    W = 133 k_distribute_dense<false, packed>."""
    if layout == "tensor":
        vids = [_packed_video(i, *shape, seed=51) for i in range(2)]
    else:
        vids = [_packed_video(i, f, 40, shape, seed=53) for i, f in enumerate((5, 2, 7))]
    label = f"{layout} {shape}"
    refs = []
    for i, v in enumerate(vids):
        guarded, r64, r32 = _reference(*v, f"{label} video {i}")
        vids[i] = v[:4] + (guarded,)
        refs.append((r64, r32))
    o = _packed(_cfg(), vids, layout == "tensor")
    o.training_step(update=False)
    for i, (r64, r32) in enumerate(refs):
        _check(_result(o, i), r64, r32, f"{label} video {i}")
    _k_carrying_agrees(o, label)


def test_packed_index_path_vs_float64_oracle():
    """procrustes_points=1000 on a (2, F) tensor batch: k_distribute<1, false, packed>."""
    f, h, w = 6, 96, 192
    vids = [_packed_video(i, f, h, w, seed=57) for i in range(2)]
    cfg = _cfg(procrustes_points=1000)
    idx = _packed(cfg, vids, True)._indices.cpu()
    refs = []
    for i, v in enumerate(vids):
        guarded, r64, r32 = _reference(*v, f"packed linspace video {i}", idx=idx)
        vids[i] = v[:4] + (guarded,)
        refs.append((r64, r32))
    o = _packed(cfg, vids, True)
    o.training_step(update=False)
    for i, (r64, r32) in enumerate(refs):
        _check(_result(o, i), r64, r32, f"packed linspace video {i}")
    _k_carrying_agrees(o, "packed linspace")


# --------------------------------------------------------------------------------------- E. Adam steps
@pytest.mark.parametrize("layout", ["dense-one", "window-packed"])
def test_graph_replayed_adam_steps_vs_float64_oracle(layout):
    """5 graph-replayed update steps: one video at 6 x 72 x 133 (k_distribute_dense<false>, separate logit Adam)
    and a (2, F) tensor batch at 6 x 48 x 96 (k_distribute_window<false, packed> with the logit Adam fused into
    it).  Every step's loss, and the depth and weight updates over the run within max(1e-3, 3x float32)."""
    steps = 5
    if layout == "dense-one":
        depth, wparam, fl, kmat64 = _video("zoom", "scene", 6, 72, 133, seed=61)
        vids = [(depth, wparam, fl, kmat64, PF._guarded_tracks(depth, wparam, fl, kmat64, _tracks(6, 62)))]
        o = _one(_cfg(), *vids[0])
        o.use_cuda_graph = True
    else:
        vids = [_packed_video(i, 6, 48, 96, seed=63) for i in range(2)]
        vids = [v[:4] + (PF._guarded_tracks(*v),) for v in vids]
        o = _packed(_cfg(), vids, True, graph=True)
    refs = [(PF._dropin_oracle(*v, steps, torch.float64), PF._dropin_oracle(*v, steps, torch.float32)) for v in vids]
    losses = [o.training_step()[0].double().cpu().reshape(-1) for _ in range(steps)]
    assert len(o._graphs) == 1
    for i, ((r64, st64), (r32, st32)) in enumerate(refs):
        for step in range(steps):
            ref = r64[step]["loss"]
            err, n = abs(float(losses[step][i]) - ref) / abs(ref), abs(r32[step]["loss"] - ref) / abs(ref)
            print(f"{layout} video {i} step {step}: loss error {err:.1e} (float32 oracle {n:.1e})")
            assert err <= max(1e-4, 3 * n), (layout, i, step, err, n)
        _updates(f"{layout} video {i}", [(o.models[i].backbone.depth, st64.depth, st32.depth, vids[i][0]),
                                          (o.models[i].backbone.weights, st64.weights, st32.weights, vids[i][1])])


# ------------------------------------------------------------------------------------------- G. reach
def test_every_k_free_instantiation_runs():
    """One profiled step of each path: the intended K-free Procrustes and tracking kernels run, by their demangled
    names, and no K-carrying k_distribute* / k_track_src / k_track_finalize, nor k_k4_finalize."""
    import re
    from torch.profiler import ProfilerActivity, profile
    paths = {"window": (6, 48, 96, {}), "dense": (6, 40, 63, {}), "index": (6, 48, 96, {"procrustes_points": 1000})}
    seen = set()
    for name, (f, h, w, kw) in paths.items():
        depth, wparam, fl, kmat64 = _video("zoom", "shift", f, h, w, seed=71)
        tracks = _tracks(f, 72)
        runs = {"one": _one(_cfg(**kw), depth, wparam, fl, kmat64, tracks),
                "packed": _packed(_cfg(**kw), [_packed_video(i, f, h, w, seed=73) for i in range(2)], True)}
        for layout, o in runs.items():
            o.training_step(update=False)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                o.training_step(update=False)
                torch.cuda.synchronize()
            names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
            lay, tl = ("PairLayout", "TrackOneVideo") if layout == "one" else ("RaggedPairs", "TrackVideos")
            kern = {"window": "k_distribute_window<false, ", "dense": "k_distribute_dense<false, ",
                    "index": "k_distribute<1, false, "}[name]
            want = [(kern, lay), ("k_track_src<true, false, ", tl), ("k_track_finalize<", f"{tl}, false>")]
            for prefix, suffix in want:
                hits = [n for n in names if re.search(re.escape(prefix) + r"[^<>]*" + re.escape(suffix), n)]
                assert hits, (name, layout, prefix, suffix, sorted(names))
                seen.update(hits)
            bad = [n for n in names if re.search(r"k_distribute\w*<(1, )?true|k_track_src<\w+, true|k_k4_finalize|"
                                                 r"k_track_finalize<[^<>]*, true>", n)]
            assert not bad, (name, layout, bad)
    print("K-free kernels seen:", *sorted(seen), sep="\n  ")
    assert len(seen) == 10, sorted(seen)
