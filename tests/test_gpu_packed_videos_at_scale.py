"""The packed multi-video step (FusedOverfitter on a list of videos: fm_overfit_step_videos and its kernels on
the packed layout) at the shapes where its persistent grids cross pairs and videos.

A persistent ragged kernel hands every block a contiguous range of items (pixel chunks or window tiles of
one pair or frame).  Where a range runs into the next pair, the block restages that pair's constants
(PairAdjoint, PairGeom, fixed-point scale, conditioning shift) and, at the first pair of the next video,
that video's normaliser and frame count.  Whether any range of a launch does so depends on the shape, on
the frame counts and on the SM count, so the geometry is restated here (launch_geometry) and asserted: on
the CPU at 132 and 114 SMs, and in every GPU test with the device's own SM count and L2 size.

- The fused packed step against the float64 OverfitOracle on each video alone, with the float32 oracle as
  the noise estimate (flow_regime_checks): neighbouring videos in different flow and depth regimes and with
  different focal lengths, so that a constant that is stale after a crossing is a large error.
- Packed against solo runs over graph-replayed update steps, at LLFF's frame counts and at 360 x 640.
- The ragged pose chain and its adjoint through the C ABI, with videos of more than 256 pairs (chunked
  scan) next to videos of two frames."""
import ctypes

import pytest
import torch

from conftest import max_abs, rel_l2
from flow_regime_checks import check, errors, start_point
from test_gpu_ragged_overfit import _assert_matches_solo, _batch, _cfgs, _videos

gpu = pytest.mark.gpu
LLFF = (20, 25, 26, 34, 41, 42, 55, 62)  # frame counts of the eight LLFF scenes
FOUR = (20, 62, 25, 41)
L2_BYTES = 50 << 20  # H100 SXM and PCIe


@pytest.fixture(autouse=True)
def _threads():
    torch.set_num_threads(min(16, torch.get_num_threads()))


# ---------------------------------------------------------------------------------------- launch geometry
def _item_span(total, rounds, rnd, block, grid):
    """item_span (fm_math.cuh): the [i0, i1) items of `block` in round `rnd`."""
    length = (total + rounds - 1) // rounds
    s0, s1 = min(length * rnd, total), min(length * rnd + length, total)
    first = (rnd * (length % grid)) % grid
    part = (block - first + grid) % grid
    q, extra = (s1 - s0) // grid, (s1 - s0) % grid
    i0 = s0 + part * q + min(part, extra)
    return i0, i0 + q + (1 if part < extra else 0)


def _persistent_grid(ctas_per_sm, items, sms):
    """persistent_grid (fm_kernels.cu)."""
    return max(1, min(items, sms * ctas_per_sm))


def _procrustes_rounds(h, w, items, grid, gathers_only, l2_bytes):
    """procrustes_rounds (fm_kernels.cu): one round while the row bands of a gathers-only pass fit in L2,
    else runs of about 8 chunks per block and round."""
    if gathers_only and grid * (0.07 * h + 6.0) * w * 4.0 <= 0.35 * l2_bytes:
        return 1
    return max(1, -(-items // grid) // 8)


def _walk(units, per_unit, grid, rounds, video):
    """(rounds, ranges that span two or more units, ranges that span a video boundary) of a launch over
    units x per_unit items; video[u] is unit u's video."""
    multi = cross = 0
    for rnd in range(rounds):
        for block in range(grid):
            i0, i1 = _item_span(units * per_unit, rounds, rnd, block, grid)
            if i1 > i0:
                u0, u1 = i0 // per_unit, (i1 - 1) // per_unit
                multi += u1 > u0
                cross += video[u0] != video[u1]
    return rounds, multi, cross


def launch_geometry(frames, h, w, sms, l2_bytes=L2_BYTES):
    """{kernel: (rounds, multi, cross)} of the persistent launches of procrustes_fwd<RaggedPairs>
    (k_moments_dense<..., RaggedPairs>), launch_flow<Videos> (k_flow_lean_ragged) and procrustes_bwd<RaggedPairs>
    (k_distribute_window<RaggedPairs> for W % 4 == 0, else k_distribute_dense<RaggedPairs>) in fm_kernels.cu:
    256-thread chunks of 4 pixels (W % 4 == 0) or 1, 64 x 32 window tiles, 3 / 2 / 3 blocks per SM."""
    pair_video = [b for b, f in enumerate(frames) for _ in range(f - 1)]
    frame_video = [b for b, f in enumerate(frames) for _ in range(f)]
    pairs, n = len(pair_video), h * w
    vec = 4 if w % 4 == 0 else 1
    chunks = -(-n // (256 * vec))
    items = pairs * chunks
    grid = _persistent_grid(3, items, sms)
    rounds = _procrustes_rounds(h, w, items if vec == 4 else items // 4, grid, True, l2_bytes)
    geo = {"moments": _walk(pairs, chunks, grid, rounds, pair_video)}
    grid = _persistent_grid(2, len(frame_video) * chunks, sms)
    geo["flow"] = _walk(len(frame_video), chunks, grid, 1, frame_video)
    if w % 4 == 0:
        tiles = -(-w // 64) * -(-h // 32)
        grid = _persistent_grid(3, pairs * tiles, sms)
        rounds = _procrustes_rounds(h, w, pairs * tiles * 2048 // 1024, grid, False, l2_bytes)
        geo["window"] = _walk(pairs, tiles, grid, rounds, pair_video)
    else:
        grid = _persistent_grid(3, items, sms)
        rounds = _procrustes_rounds(h, w, items // 4, grid, False, l2_bytes)
        geo["dense"] = _walk(pairs, chunks, grid, rounds, pair_video)
    return geo


# id: (frame counts, H, W, kernels with ranges across units and videos, kernels that must run in rounds)
GEOMETRY = {
    "llff-176x224": (LLFF, 176, 224, ("moments", "flow", "window"), ("window",)),
    "four-176x228": (FOUR, 176, 228, ("moments", "flow", "window"), ()),   # vector strips: W % 32 != 0
    "four-176x222": (FOUR, 176, 222, ("moments", "flow", "dense"), ()),    # scalar: W % 4 != 0
    "two-360x640": ((19, 18), 360, 640, ("moments", "flow"), ("moments",)),
}


def _assert_geometry(case, sms, l2_bytes):
    frames, h, w, crossing, in_rounds = GEOMETRY[case]
    geo = launch_geometry(frames, h, w, sms, l2_bytes)
    print(f"{case} at {sms} SMs, L2 {l2_bytes >> 20} MiB: (rounds, multi-unit ranges, cross-video ranges)", geo)
    for k in crossing:
        assert geo[k][1] > 0 and geo[k][2] > 0, (case, sms, k, geo[k], "no range crosses a unit and a video")
    for k in in_rounds:
        assert geo[k][0] >= 2, (case, sms, k, geo[k], "one round")
    return geo


def _device_geometry(case):
    """_assert_geometry with this device's SM count and L2 size: what the kernels about to run will do."""
    p = torch.cuda.get_device_properties(0)
    return _assert_geometry(case, p.multi_processor_count, p.L2_cache_size)


@pytest.mark.parametrize("sms", [132, 114], ids=["132sm", "114sm"])
@pytest.mark.parametrize("case", list(GEOMETRY))
def test_cases_reach_their_launch_geometry(case, sms):
    """Each case below crosses pairs / frames and videos in the kernels it exists for, on a 132-SM H100
    SXM and on a 114-SM H100 PCIe."""
    _assert_geometry(case, sms, L2_BYTES)


def test_geometry_restatement_on_the_small_shapes():
    """The restatement on the shapes of test_gpu_ragged_overfit.py: at 72 x 96 no range crosses anything;
    at 72 x 133 only the flow kernel's do (14 ranges, 2 across a video, at 132 SMs)."""
    assert launch_geometry((4, 10, 7), 72, 96, 132) == {"moments": (1, 0, 0), "flow": (1, 0, 0),
                                                        "window": (1, 0, 0)}
    assert launch_geometry((4, 10, 7), 72, 133, 132) == {"moments": (1, 0, 0), "flow": (1, 14, 2),
                                                         "dense": (1, 0, 0)}


# ------------------------------------------------------------------- fused packed step vs float64 oracle
# Neighbouring videos in different regimes.  `scene` goes first: its camera walk leaves the scene's sphere
# (non-finite depth) beyond about 20 frames, and video 0 is the shortest of every case.
# Not in the LLFF cases: `scale_small` / `scale_large` on the 42-frame video (seed 5).  There one pair's weight
# gradient misses max(1e-4, 3x float32) by a few 1e-5, for the one-video step exactly as for the packed one, and
# at x 1e2 the softmin stage's absolute pose error (4.5e-4) sits just past 3x float32's (1.4e-4).
KINDS = ("scene", "scale_small", "iid", "horizon", "centre_far", "shift", "outliers", "zoom")
ORACLE_CASES = {
    "llff-176x224-regressed": ("llff-176x224", KINDS, {}),
    "llff-176x224-pts1000": ("llff-176x224", KINDS, {"procrustes_points": 1000}),  # index-mode kernels
    "four-176x228-regressed": ("four-176x228", ("scene", "outliers", "scale_small", "zoom"), {}),
    "four-176x222-regressed": ("four-176x222", ("scene", "shift", "horizon", "scale_large"), {}),
    "two-360x640-regressed": ("two-360x640", ("scene", "scale_small"), {}),
}
_FLOW_NAMES = ("forward", "backward", "forward_mask", "backward_mask")
# Regimes whose 41-row segments the float32 oracle cannot place: its own position error (on the 200- and
# 1000-deep pixels, and under the divergent `zoom` flow) sets a guard band that clears more than 1 % of their
# samples on the LLFF cases -- `horizon` 1.4 % (all pixels) to 22 % (1000 Procrustes points), `zoom` 3 %,
# `centre_far` 5.3 % (1000 points).  They keep 9 rows.
SHORT_SEGMENT_KINDS = ("horizon", "zoom", "centre_far")


def _regime_video(kind, f, h, w, seed, focal_scale):
    """Float64 inputs of one video at a start point (flow_regime_checks.start_point) in a flow or depth
    regime, with tracks (scene_tracks for `scene`, else synthetic_tracks) and its focal length x focal_scale."""
    from oracle import flowmap_oracle as O
    if kind in O.DEPTH_REGIMES:
        depth, fl, focal, wparam = O.depth_regime(kind, f, h, w, seed=seed)
        ext = None
    else:
        depth, fl, focal, ext = O.flow_regime(kind, f, h, w, seed=seed)
        wparam = 0.01 * torch.randn(1, f - 1, h, w, generator=torch.Generator().manual_seed(seed + 2),
                                    dtype=torch.float64)
    assert bool(torch.isfinite(depth).all()), (kind, f, seed)
    if ext is not None:
        tracks = O.scene_tracks(depth[0], ext, focal, [(0, f), (2, 3), (f - 2, 2)], n_points=600, seed=seed)
    else:  # the reference's segments, 41 rows, guarded by the tests (_guard_video); 9 rows in SHORT_SEGMENT_KINDS
        tracks = O.synthetic_tracks(f, n_points=300, interval=5, radius=4 if kind in SHORT_SEGMENT_KINDS else 20,
                                    seed=seed, dtype=torch.float64)
    depth, focal = start_point(depth, focal, seed=seed + 1)
    return dict(kind=kind, depth=depth[0], wparam=wparam[0], flows=fl, focal=focal * focal_scale, tracks=tracks,
                depth_regime=kind in O.DEPTH_REGIMES)


def _regime_videos(geometry_case, kinds):
    frames, h, w = GEOMETRY[geometry_case][:3]
    return [_regime_video(kinds[i % len(kinds)], f, h, w, seed=i, focal_scale=1.0 + 0.02 * i)
            for i, f in enumerate(frames)]


def _packed_optimiser(cfg, videos):
    """One FusedOverfitter on all videos, at each video's start point and focal length."""
    from flowmap_b200.overfit import FusedOverfitter
    from flowmap_b200.types import Flows, Tracks
    dev = torch.device("cuda:0")
    h, w = videos[0]["depth"].shape[-2:]
    o = FusedOverfitter(cfg, [_batch(v["depth"].shape[0], h, w, dev) for v in videos],
                        [Flows(*(getattr(v["flows"], n).float() for n in _FLOW_NAMES)) for v in videos],
                        [[Tracks(t.xy.float(), t.visibility, t.start_frame) for t in v["tracks"]] for v in videos]
                        if cfg.use_tracking else None, device=dev)
    with torch.no_grad():
        for m, v in zip(o.models, videos):
            m.backbone.depth.copy_(v["depth"].float())
            m.backbone.weights.copy_(v["wparam"].float())
        if cfg.intrinsics == "regressed":
            o._focal.copy_(torch.tensor([v["focal"] for v in videos]))
    return o


def _oracle_model(v, kw, dt):
    """OverfitOracle on video v alone in dtype dt, at v's start point, and v's flows in dt."""
    from oracle import flowmap_oracle as O
    f, h, w = v["depth"].shape
    st = O.OverfitOracle(O.OverfitConfig(initial_focal=v["focal"], **kw), f, h, w, dtype=dt)
    with torch.no_grad():
        st.depth.copy_(v["depth"].to(dt))
        st.weights.copy_(v["wparam"].to(dt))
    return st, O.Flows(*(getattr(v["flows"], n).to(dt) for n in _FLOW_NAMES))


def _guard_video(v, kw, **forward_kw):
    """v with its tracks guarded by track_travel_checks.clear_track_kinks at the poses and intrinsics of step 0 of
    its float64 oracle, the band from the float32 oracle's position error.  Under a long coherent motion the
    41-row segments cross the [0,1)^2 border ~1e5 times, and a target within rounding of it is valid in one
    precision and not in the other: a whole saturated Huber term at four depth taps of one frame."""
    import track_travel_checks as T
    from oracle import flowmap_oracle as O
    if v["kind"] in SHORT_SEGMENT_KINDS:
        return v  # 9-row segments, as before the guard: the float32 oracle's band there is the problem
    triples = {}
    for dt in (torch.float64, torch.float32):
        st, flows = _oracle_model(v, kw, dt)
        with torch.no_grad():
            m = st.forward(flows, 0, **forward_kw)
            triples[dt] = T.track_triples(m.surfaces, m.extrinsics, m.intrinsics,
                                          [O.Tracks(t.xy.to(dt), t.visibility, t.start_frame) for t in v["tracks"]])
    band = T.position_band(triples[torch.float64], triples[torch.float32], v["tracks"])
    tracks, cleared = T.clear_track_kinks(v["tracks"], triples[torch.float64], band)
    samples = sum(int(t.visibility.sum()) for t in v["tracks"])
    assert cleared <= 0.01 * samples, (v["kind"], "guard cleared", cleared, samples)
    return dict(v, tracks=tracks)


def _oracle(v, kw, dt, steps=1, **step_kw):
    """OverfitOracle on video v alone in dtype dt: the oracle and its first `steps` training steps."""
    from oracle import flowmap_oracle as O
    st, flows = _oracle_model(v, kw, dt)
    tracks = [O.Tracks(t.xy.to(dt), t.visibility, t.start_frame) for t in v["tracks"]] \
        if kw.get("use_tracking") else None
    out = []
    for _ in range(steps):
        r = st.training_step(flows, tracks, **step_kw)
        gf = r["grads"]["focal"]
        out.append(dict(loss=r["loss"], ext=r["extrinsics"].double(), g_depth=r["grads"]["depth"].double(),
                        g_w=r["grads"]["weights"].double(), g_focal=None if gf is None else float(gf),
                        track=r["parts"].get("tracking"), fx=float(r["intrinsics"][0, 0, 0, 0])))
    return st, out


class _Largest:
    """The largest error per metric over the videos of a case, and the float32 oracle's in brackets."""

    def __init__(self):
        self.got, self.noise = {}, {}

    def add(self, errs, noise):
        for k, v in errs.items():
            n = noise.get(k, 0.0)
            v, n = (max(v), max(n)) if isinstance(v, list) else (v, n)
            self.got[k], self.noise[k] = max(self.got.get(k, 0.0), v), max(self.noise.get(k, 0.0), n)

    def report(self, label):
        print(label, "largest errors vs float64 oracle [float32 oracle]:",
              ", ".join(f"{k} {v:.1e} [{self.noise[k]:.1e}]" for k, v in self.got.items()))


def _check_step0(o, total, videos, refs, label, largest):
    """Step 0 of every video against its own float64 oracle: loss, poses, tracking loss, gradients per frame,
    pair and border band, focal gradient.  Loss and poses are held to the fixed tolerances, or to 3x the
    float32 oracle's error in the depth regimes (as in test_gpu_depth_conditioning.py) and where float32
    itself misses the fixed pose tolerance: a long coherent motion chains its camera positions out to
    |t| ~ 10 - 20, where float32 rounding alone is ~2e-5."""
    gr, ext = o.gradients(), o.extrinsics()
    for i, (v, (r64, r32)) in enumerate(zip(videos, refs)):
        out = dict(loss=float(total[i]), ext=ext[i].cpu(), g_depth=gr["depth"][i].cpu(), g_w=gr["weights"][i].cpu(),
                   g_focal=None if r64["g_focal"] is None else float(gr["focal"][i]))
        e, noise = errors(out, r64), errors(r32, r64)
        lab = f"{label} video {i} ({v['depth'].shape[0]} frames, {v['kind']})"
        relative = v["depth_regime"] or noise["pose"] > 2e-5
        if relative and not v["depth_regime"]:
            print(lab, f"float32 oracle's pose error {noise['pose']:.1e} > 2e-5: loss and poses within 3x it")
        check(e, noise, lab, loss_tol=1e-4, pose_tol=2e-5, floor=1e-4, relative_fixed=relative)
        largest.add(e, noise)
        if r64["track"] is not None:
            t_err = abs(float(o._track_loss[i]) - r64["track"]) / abs(r64["track"])
            print(lab, f"tracking loss {r64['track']:.4e}: error {t_err:.1e}")
            assert r64["track"] > 0 and t_err <= 1e-4, (lab, "tracking loss", t_err)
            largest.add({"track": t_err}, {"track": abs(r32["track"] - r64["track"]) / abs(r64["track"])})


@gpu
@pytest.mark.parametrize("case", list(ORACLE_CASES))
def test_packed_step_vs_float64_oracle_per_video(case):
    """Step 0 (training_step(update=False)) of the packed step, regressed focal lengths, tracking on, against
    each video's own float64 OverfitOracle."""
    from flowmap_b200.overfit import OverfitCfg
    geometry_case, kinds, extra = ORACLE_CASES[case]
    if "procrustes_points" not in extra:
        _device_geometry(geometry_case)
    from oracle import flowmap_oracle as O
    kw = dict(intrinsics="regressed", use_tracking=True, tracking_enable_after=0, **extra)
    h, w = GEOMETRY[geometry_case][1:3]
    idx = None if "procrustes_points" not in extra else \
        O.procrustes_indices(h, w, extra["procrustes_points"], False, device="cuda").cpu()
    videos = [_guard_video(v, kw, procrustes_idx=idx) for v in _regime_videos(geometry_case, kinds)]
    o = _packed_optimiser(OverfitCfg(**kw), videos)
    pts = None if o._indices is None else o._indices.cpu()  # the oracle gets the device's point set
    total, _ = o.training_step(update=False)
    refs = [tuple(_oracle(v, kw, dt, procrustes_idx=pts)[1][0] for dt in (torch.float64, torch.float32))
            for v in videos]
    largest = _Largest()
    _check_step0(o, total, videos, refs, case, largest)
    largest.report(case)


@gpu
def test_packed_softmin_stage_vs_float64_oracle_per_video():
    """The softmin stage (regression_after=None) with 8192 injected sweep points and tracking at LLFF x 176 x
    224: step 0 and every video's f_hat, then 3 Adam steps against each oracle's trajectory (loss and fx per
    step, depth and weight update at the end).  The update steps run what step 0 does not: the early moment
    pass at the candidate-0 intrinsics (fm_procrustes_moments_videos, rescaled in the step's solve), the
    ragged sweep's forward and backward, and the per-video frame Adam."""
    from flowmap_b200.overfit import OverfitCfg
    _device_geometry("llff-176x224")
    h, w = GEOMETRY["llff-176x224"][1:3]
    kw = dict(intrinsics="softmin", regression_after=None, use_tracking=True, tracking_enable_after=0)
    sweep_idx = torch.randperm(h * w, generator=torch.Generator().manual_seed(35))[:8192].cuda()
    videos = [_guard_video(v, kw, softmin_indices=sweep_idx.cpu()) for v in _regime_videos("llff-176x224", KINDS)]
    o = _packed_optimiser(OverfitCfg(**kw), videos)
    o.injected_indices = sweep_idx
    label = "packed softmin llff-176x224"
    total, _ = o.training_step(update=False)
    fx = [float(k[0, 0]) for k in o.intrinsics_k4()]
    runs = [(_oracle(v, kw, torch.float64, steps=3, softmin_indices=sweep_idx.cpu()),
             _oracle(v, kw, torch.float32, steps=3, softmin_indices=sweep_idx.cpu())) for v in videos]
    largest = _Largest()
    _check_step0(o, total, videos, [(r64[0], r32[0]) for (_, r64), (_, r32) in runs], label, largest)
    for i, ((_, r64), (_, r32)) in enumerate(runs):
        fx_err, fx_noise = abs(fx[i] - r64[0]["fx"]), abs(r32[0]["fx"] - r64[0]["fx"])
        print(label, f"video {i} f_hat {r64[0]['fx']:.6f}: error {fx_err:.1e} | float32 oracle {fx_noise:.1e}")
        assert fx_err <= max(1e-5, 3 * fx_noise), (label, i, "f_hat", fx_err, fx_noise)
        largest.add({"f_hat": fx_err}, {"f_hat": fx_noise})
    for s in range(3):
        total, _ = o.training_step()
        fx = [float(k[0, 0]) for k in o.intrinsics_k4()]
        for i, ((_, r64), (_, r32)) in enumerate(runs):
            l_err = abs(float(total[i]) - r64[s]["loss"]) / abs(r64[s]["loss"])
            fx_err, fx_noise = abs(fx[i] - r64[s]["fx"]), abs(r32[s]["fx"] - r64[s]["fx"])
            print(label, f"Adam step {s} video {i}: loss error {l_err:.1e}, fx error {fx_err:.1e} "
                  f"| float32 oracle {fx_noise:.1e}")
            assert l_err <= 1e-4 and fx_err <= max(1e-5, 3 * fx_noise), (label, s, i, l_err, fx_err, fx_noise)
    for i, (v, ((st64, _), (st32, _))) in enumerate(zip(videos, runs)):
        d_err = rel_l2(o.models[i].backbone.depth.detach().cpu(), st64.depth.detach())
        d_noise = rel_l2(st32.depth.detach(), st64.depth.detach())
        upd = o.models[i].backbone.weights.detach().cpu().double() - v["wparam"]
        w_err = rel_l2(upd, st64.weights.detach() - v["wparam"])
        print(label, f"video {i} after 3 Adam steps: depth {d_err:.1e} | float32 oracle {d_noise:.1e}, "
                     f"weight update {w_err:.1e}")
        # the depth within 1e-5, or 3x the float32 oracle's own trajectory where the sweep's gradient on frames
        # 0 and 1 is that noisy (scale_small)
        assert d_err <= max(1e-5, 3 * d_noise) and w_err <= 2e-2, (label, i, d_err, d_noise, w_err)
        largest.add({"depth_after_3": d_err, "weight_update_after_3": w_err}, {"depth_after_3": d_noise})
    largest.report(label)


# ------------------------------------------------------------- packed vs solo runs, graph-replayed steps
SOLO_CASES = {  # id: (geometry case or None, frame counts, H, W, configuration of test_gpu_ragged_overfit._cfgs)
    "llff-176x224-regressed": ("llff-176x224", LLFF, 176, 224, "regressed"),
    "llff-176x224-handover-tracking": ("llff-176x224", LLFF, 176, 224, "softmin_tracking"),
    "two-360x640-regressed": ("two-360x640", (19, 18), 360, 640, "regressed"),
    "llff-160x224-handover-tracking": (None, LLFF, 160, 224, "softmin_tracking"),  # the throughput workload
}


@gpu
@pytest.mark.parametrize("case", list(SOLO_CASES))
def test_packed_graph_replayed_steps_equal_solo_runs(case):
    """8 update steps replayed from CUDA graphs (the fused logit Adam, the clock-driven frame Adam and, with
    softmin_tracking, the hand-over at step 4) follow each video's one-video run step by step, to the
    tolerances of test_gpu_ragged_overfit.py.  LLFF x 160 x 224 is the shape of DESIGN's throughput table;
    on a 132-SM card its window ranges line up with the pairs.

    Except the focal length after the hand-over, which is held to a quarter of one Adam step (lr).  At these
    shapes the packed and the one-video launches split the pixels into different block ranges, so their
    float32 per-thread partial sums round differently, and the focal gradient, a sum of per-frame terms that
    cancel, differs deterministically: by 2e-3 of itself at step 0 of LLFF x 160 x 224's 20-frame video.
    The hand-over seeds the focal length at the softmin estimate, close to the loss's optimum, where that
    gradient crosses zero (+4.0e-6, +1.1e-6, -1.9e-6 at steps 4 - 6) and its relative difference reaches 6 %.
    Adam normalises each update to about lr, so those percent become percent of lr in the focal length, a few
    1e-6 of it.  A wrong video's window, seed or Adam state moves the focal length by 1e-3 or by a whole lr."""
    geometry_case, frames, h, w, config = SOLO_CASES[case]
    if geometry_case is not None:
        _device_geometry(geometry_case)
    cfg, loss_tol = _cfgs()[config]
    focal_tol = 0.25 * cfg.lr if cfg.intrinsics == "softmin" else None
    _assert_matches_solo(cfg, _videos("synthetic", w, frames=frames, h=h), True, loss_tol, focal_tol=focal_tol)


# ------------------------------------------------------------------------ ragged pose chain, C ABI
CHAIN_LAYOUTS = {
    "2-3-2": (2, 3, 2),
    "257-2-300-258": (257, 2, 300, 258),  # chunked scans (> 256 pairs) next to a two-frame video
    "llff": LLFF,
    "40-videos-of-2-to-9": tuple(2 + (5 * i) % 8 for i in range(40)),
}


def _rigid_motions(n, gen):
    """n small random rigid motions (n, 4, 4), float64 (as test_gpu_parity's chain test)."""
    w = 0.05 * torch.randn(n, 3, generator=gen, dtype=torch.float64)
    k = torch.zeros(n, 3, 3, dtype=torch.float64)
    k[:, 0, 1], k[:, 0, 2], k[:, 1, 0] = -w[:, 2], w[:, 1], w[:, 2]
    k[:, 1, 2], k[:, 2, 0], k[:, 2, 1] = -w[:, 0], -w[:, 1], w[:, 0]
    t = torch.eye(4, dtype=torch.float64).repeat(n, 1, 1)
    t[:, :3, :3] = torch.linalg.matrix_exp(k)
    t[:, :3, 3] = 0.1 * torch.randn(n, 3, generator=gen, dtype=torch.float64)
    return t


@gpu
@pytest.mark.parametrize("layout", list(CHAIN_LAYOUTS))
def test_ragged_pose_chain_vs_float64_oracle(layout):
    """fm_pose_chain_videos and fm_pose_chain_bwd_videos on a layout built by overfit.video_tables (as
    FusedOverfitter builds it): every video's chain from its own frame 0, and its adjoint under a random
    cotangent with a zero bottom row, against oracle.pose_chain in float64, to the tolerances of
    test_gpu_parity.test_pose_chain_scan_vs_sequential_float64."""
    from oracle import flowmap_oracle as O
    from flowmap_b200._lib import VideoLayout, check as lib_check, lib
    from flowmap_b200.overfit import video_tables
    frames = CHAIN_LAYOUTS[layout]
    B, T = len(frames), sum(frames)
    gen = torch.Generator().manual_seed(T)
    rel = [_rigid_motions(f - 1, gen).requires_grad_(True) for f in frames]
    gout = [torch.randn(f, 4, 4, generator=gen, dtype=torch.float64) for f in frames]
    for g in gout:
        g[:, 3, :] = 0
    refs = []
    for r, g in zip(rel, gout):
        ext = O.pose_chain(r[None])[0]
        ext.backward(g)
        refs.append(ext.detach())
    dev = torch.device("cuda:0")
    tables = video_tables(list(frames), dev)
    lay = VideoLayout(B, T, *(t.data_ptr() for t in tables))
    rt = torch.cat([r.detach()[:, :3, :] for r in rel]).float().to(dev).contiguous()
    g_ext = torch.cat(gout).float().to(dev).contiguous()
    ext = torch.full((T, 4, 4), float("nan"), device=dev)
    g_rt = torch.full((T - B, 3, 4), float("nan"), device=dev)
    st = torch.cuda.current_stream().cuda_stream
    lib_check(lib().fm_pose_chain_videos(rt.data_ptr(), ext.data_ptr(), ctypes.byref(lay), st), "fm_pose_chain_videos")
    lib_check(lib().fm_pose_chain_bwd_videos(rt.data_ptr(), ext.data_ptr(), g_ext.data_ptr(), g_rt.data_ptr(),
                                             ctypes.byref(lay), st), "fm_pose_chain_bwd_videos")
    ext, g_rt = ext.cpu(), g_rt.cpu()
    f0 = 0
    for b, (f, r, ref) in enumerate(zip(frames, rel, refs)):
        scale = float(ref.abs().max())
        e = max_abs(ext[f0:f0 + f], ref)
        g = rel_l2(g_rt[f0 - b:f0 - b + f - 1], r.grad[:, :3, :])
        assert e <= 2e-6 * max(1.0, scale) * (1 + f / 150), (layout, b, f, "chain", e)
        assert g <= 1e-5, (layout, b, f, "adjoint", g)
        f0 += f
