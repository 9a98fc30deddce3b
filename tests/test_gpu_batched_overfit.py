"""Several same-shape videos optimised as one fused step (FusedOverfitter with B > 1).

The batched step is B independent overfits: video b must follow a one-video FusedOverfitter on video b
(same cfg, same step-clock seed) to the noise of the float atomics.  The one-video optimiser is the
reference here; it is pinned to the float64 oracle and the goldens by the other suites."""
import re

import pytest
import torch

from conftest import ROOT

gpu = pytest.mark.gpu
F, H, STEPS, SEED = 10, 72, 8, 1234


# ---------------------------------------------------------------------------------------------- CPU
def _header_struct_fields(name):
    text = (ROOT / "include" / "flowmap_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    body = re.search(r"typedef struct \{([^}]*)\}\s*" + name + ";", text).group(1)
    fields = []
    for decl in body.split(";"):
        for part in decl.split(","):
            ids = re.findall(r"[A-Za-z_]\w*", part)
            if ids:
                fields.append(ids[-1])
    return fields


def test_overfit_step_args_field_order_matches_the_header():
    from flowmap_b200._lib import OverfitStepArgs
    assert [f[0] for f in OverfitStepArgs._fields_] == _header_struct_fields("fm_overfit_step_args")
    # appended: every existing caller keeps its layout
    assert [f[0] for f in OverfitStepArgs._fields_[-2:]] == ["B", "gt_fxfy"]


def _cpu_inputs(b, f=4, h=8, w=8):
    from flowmap_b200.types import Batch, Flows, Tracks
    batch = Batch(torch.zeros(b, f, 3, h, w), torch.arange(f)[None].expand(b, f), ["s"] * b, ["d"] * b)
    flows = Flows(torch.zeros(b, f - 1, h, w, 2), torch.zeros(b, f - 1, h, w, 2), torch.ones(b, f - 1, h, w),
                  torch.ones(b, f - 1, h, w))
    tracks = [Tracks(torch.rand(1, 2, 5, 2), torch.ones(1, 2, 5, dtype=torch.bool), 0)]
    return batch, flows, tracks


def test_batched_step_validates_its_inputs():
    """Refused before anything reaches the device: a track list that is not one list per video, a bound
    Model, flows whose batch does not match the videos, and pair sharding of several videos."""
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg, ShardedFusedOverfitter
    batch, flows, tracks = _cpu_inputs(2)
    with pytest.raises(ValueError, match="one segment list per video"):
        FusedOverfitter(OverfitCfg(use_tracking=True), batch, flows, [tracks])
    with pytest.raises(ValueError, match="Model"):
        FusedOverfitter(OverfitCfg(), batch, flows, model=object())
    _, flows3, _ = _cpu_inputs(3)
    with pytest.raises(ValueError, match="pairs"):
        FusedOverfitter(OverfitCfg(), batch, flows3)
    with pytest.raises(ValueError, match="one video"):
        ShardedFusedOverfitter(OverfitCfg(), batch, flows, plan=None)


def test_packed_tracks_of_several_videos():
    """Segment s of video b is packed with start frame b * F + s.start_frame, samples in order; a
    segment that leaves its video is refused."""
    from flowmap_b200 import ops
    from flowmap_b200.types import Tracks
    g = torch.Generator().manual_seed(0)
    seg = lambda rows, n, start: Tracks(torch.rand(1, rows, n, 2, generator=g),  # noqa: E731
                                        torch.rand(1, rows, n, generator=g) < 0.5, start)
    videos = [[seg(3, 5, 0), seg(2, 4, 3)], [], [seg(4, 6, 1)]]
    pk = ops.PackedTracks(videos, "cpu", video_frames=5)
    assert pk.seg.tolist() == [[0, 3, 5, 0], [15, 2, 4, 3], [23, 4, 6, 2 * 5 + 1]]
    assert pk.total == 47 and pk.num_segments == 3 and pk.max_rows == 4 and pk.max_points == 6
    flat = [t for v in videos for t in v]
    assert torch.equal(pk.xy, torch.cat([t.xy[0].reshape(-1, 2) for t in flat]))
    assert torch.equal(pk.vis, torch.cat([t.visibility[0].reshape(-1) for t in flat]).to(torch.uint8))
    one = ops.PackedTracks(videos[0], "cpu")  # one video: the layout it always had
    assert one.seg.tolist() == [[0, 3, 5, 0], [15, 2, 4, 3]]
    with pytest.raises(ValueError, match="leaves"):
        ops.PackedTracks([[seg(3, 5, 3)]], "cpu", video_frames=5)


# ---------------------------------------------------------------------------------------------- GPU
def _videos(kind, w):
    """Three videos with different content: (depth (F,H,W), weight logits (F-1,H,W), Flows (1, ...))."""
    import bench
    from oracle.flowmap_oracle import flow_regime
    from flowmap_b200.types import Flows, Tracks
    out = []
    for i in range(3):
        if kind == "synthetic":
            inp = bench.synthetic_inputs(F, H, w, seed=i)
            depth, wl = 1.0 + inp["depth"], inp["wparam"]
            flows = Flows(inp["fwd"], inp["bwd"], inp["fmask"], inp["bmask"])
        else:
            depth, fl, _, _ = flow_regime(("shift", "outliers", "scene")[i], F, H, w, seed=i)
            depth = depth[0].float()
            wl = 0.01 * torch.randn(F - 1, H, w, generator=torch.Generator().manual_seed(i))
            flows = Flows(*(getattr(fl, n).float() for n in ("forward", "backward", "forward_mask", "backward_mask")))
        tracks = [Tracks(xy, vis, st) for xy, vis, st in
                  bench.synthetic_track_arrays(F, n_points=48 + 40 * i, interval=3 + i, radius=2, seed=i)]
        out.append((depth, wl, flows, tracks))
    return out


def _run(cfg, videos, graph, steps=STEPS, extrinsics=None, intrinsics=None, log=0):
    """Optimise `videos` as one batched FusedOverfitter (or one video alone when len == 1): per step the
    losses (B,) and rt; at the end depth (B,F,H,W), logits (B,F-1,H,W), focal (B,)."""
    from flowmap_b200.overfit import FusedOverfitter
    from flowmap_b200.types import Batch, Flows
    dev = torch.device("cuda:0")
    b, w = len(videos), videos[0][0].shape[-1]
    batch = Batch(torch.zeros(b, F, 3, H, w, device=dev), torch.arange(F, device=dev)[None].expand(b, F), ["s"] * b,
                  ["d"] * b, extrinsics=extrinsics, intrinsics=intrinsics)
    flows = Flows(*(torch.cat([getattr(v[2], n) for v in videos]).to(dev)
                    for n in ("forward", "backward", "forward_mask", "backward_mask")))
    tracks = None if not cfg.use_tracking else (videos[0][3] if b == 1 else [v[3] for v in videos])
    o = FusedOverfitter(cfg, batch, flows, tracks, device=dev)
    o._clock.base_seed = SEED  # one softmin point sample per step, the same for batched and solo runs
    assert len(o.models) == b and o.models[0] is o.model
    with torch.no_grad():
        for m, (depth, wl, _, _) in zip(o.models, videos):
            m.backbone.depth.copy_(depth)
            m.backbone.weights.copy_(wl)
    o.use_cuda_graph = graph
    if log:
        o.enable_metrics_log(log)
    losses, rts = [], []
    for _ in range(steps):
        total, rt = o.training_step()
        losses.append(total.reshape(b).clone())
        rts.append(rt.clone())
    torch.cuda.synchronize()
    depth = torch.stack([m.backbone.depth.detach() for m in o.models])
    logits = torch.stack([m.backbone.weights.detach() for m in o.models])
    # the batched buffers are the models' parameters (views, no copies)
    assert o.models[-1].backbone.depth.data_ptr() == o._depth.reshape(b, -1)[-1].data_ptr()
    return torch.stack(losses), torch.stack(rts), depth, logits, o._focal.reshape(b).clone(), o


def _rel_l2(a, b):
    return float((a - b).norm() / b.norm())


def _assert_matches_solo(cfg, videos, graph, loss_tol):
    lb, rb, db, wb, fb, o = _run(cfg, videos, graph)
    if graph:
        assert len(o._graphs) >= 1
    for i, v in enumerate(videos):
        ls, rs, ds, ws, fs, _ = _run(cfg, [v], graph)
        assert float(((lb[:, i] - ls[:, 0]).abs() / ls[:, 0].abs().clamp_min(1e-30)).max()) <= loss_tol, i
        assert _rel_l2(db[i], ds[0]) <= 1e-5, i
        assert float((wb[i] - ws[0]).abs().max()) <= 1e-5, i
        assert abs(float(fb[i]) - float(fs[0])) <= 1e-6 * abs(float(fs[0])), i
        assert float((rb[:, i] - rs[:, 0]).abs().max()) <= 2e-6, i
    return lb


def _cfgs():
    from flowmap_b200.overfit import OverfitCfg
    return {
        "regressed": (OverfitCfg(), 1e-6),
        "softmin_handover": (OverfitCfg(intrinsics="softmin", regression_after=4, regression_window=2,
                                        softmin_points=500), 1e-5),
        "softmin_tracking": (OverfitCfg(intrinsics="softmin", regression_after=4, regression_window=2,
                                        softmin_points=500, use_tracking=True, tracking_enable_after=0), 1e-5),
        "softmin_no_regression": (OverfitCfg(intrinsics="softmin", regression_after=None, softmin_points=500), 1e-5),
        "procrustes_points": (OverfitCfg(procrustes_points=1000), 1e-5),
        "no_weights": (OverfitCfg(use_correspondence_weights=False), 1e-6),
    }


@gpu
@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("config", ["regressed", "softmin_handover", "softmin_tracking", "softmin_no_regression",
                                    "procrustes_points", "no_weights"])
@pytest.mark.parametrize("w", [96, 133])
@pytest.mark.parametrize("kind", ["synthetic", "regimes"])
def test_batched_step_equals_solo_runs(kind, w, config, graph):
    """Three different videos in one step follow three one-video runs, step by step: loss, poses, and at
    the end depth, weight logits and focal length.  W = 133 takes the scalar kernels (no fused logit
    Adam); the softmin configs cross the hand-over to the regressed focal length within the 8 steps, one
    with the tracking loss from step 0 (each video has a track set of its own size)."""
    cfg, loss_tol = _cfgs()[config]
    _assert_matches_solo(cfg, _videos(kind, w), graph, loss_tol)


@gpu
def test_each_video_has_its_own_flow_normaliser():
    """Video 1 without any valid flow: its mask sum is 0 and "or 1" applies to it alone (its loss is 0),
    while videos 0 and 2 still follow their solo runs."""
    from flowmap_b200.overfit import OverfitCfg
    videos = _videos("synthetic", 96)
    fl = videos[1][2]
    fl.forward_mask.zero_()
    fl.backward_mask.zero_()
    lb = _assert_matches_solo(OverfitCfg(), videos, False, 1e-6)
    assert float(lb[:, 1].abs().max()) == 0.0 and float(lb[:, 0].min()) > 0.0


@gpu
def test_each_video_has_its_own_tracking_normaliser():
    """Track sets of different sizes: every video's tracking loss is its solo tracking loss (its own
    valid count), and so are the totals, flow loss and parameters."""
    from flowmap_b200.overfit import OverfitCfg
    cfg = OverfitCfg(use_tracking=True, tracking_enable_after=0)
    videos = _videos("synthetic", 96)
    _, _, _, _, _, o = _run(cfg, videos, False, steps=2)
    for i, v in enumerate(videos):
        _, _, _, _, _, s = _run(cfg, [v], False, steps=2)
        assert abs(float(o._track_loss[i]) - float(s._track_loss)) <= 1e-5 * abs(float(s._track_loss)), i
        assert float(s._track_loss) > 0.0
    _assert_matches_solo(cfg, videos, False, 1e-5)


@gpu
@pytest.mark.parametrize("config", ["regressed", "softmin_tracking"])
def test_batched_metrics_rows_equal_solo_rows(config):
    """The (steps, B) metrics log holds every video's solo rows; videos 0 and 2 have ground truth
    (a consistent scene's camera centres and intrinsics), video 1 has none: its columns are NaN."""
    from oracle.flowmap_oracle import flow_regime
    cfg = _cfgs()[config][0]
    videos = _videos("synthetic", 96)
    ext = torch.stack([flow_regime("scene", F, H, 96, seed=i)[3][0].float() for i in range(3)])
    k = torch.eye(3).expand(3, F, 3, 3).clone()
    k[:, :, 0, 0], k[:, :, 1, 1] = 0.8, 0.9
    k[:, :, :2, 2] = 0.5
    ext[1], k[1] = float("nan"), float("nan")
    *_, o = _run(cfg, videos, True, extrinsics=ext, intrinsics=k, log=16)
    log = o.metrics_log()
    assert all(t.shape == (STEPS, 3) for t in log.values())
    for i, v in enumerate(videos):
        gt = (None, None) if i == 1 else (ext[i:i + 1], k[i:i + 1])
        *_, s = _run(cfg, [v], True, extrinsics=gt[0], intrinsics=gt[1], log=16)
        solo = s.metrics_log()
        for name in log:
            a, b = log[name][:, i], solo[name]
            assert torch.equal(a.isnan(), b.isnan()), (i, name)
            a, b = a[~b.isnan()].double(), b[~b.isnan()].double()
            if b.numel():
                assert float((a - b).abs().max()) <= 1e-5 * max(1.0, float(b.abs().max())), (i, name)
        if i == 1:
            assert bool(log["metrics/ate"][:, 1].isnan().all()) and bool(log["train/intrinsics/fx_error"][:, 1].isnan().all())
        else:
            assert not bool(log["metrics/ate"][:, i].isnan().any())


@gpu
def test_batched_step_surface():
    """Shapes of what the batched optimiser hands out, and set_flows with per-video mask sums."""
    from flowmap_b200.overfit import OverfitCfg
    from flowmap_b200.types import Flows
    videos = _videos("synthetic", 96)
    _, _, _, _, _, o = _run(OverfitCfg(), videos, False, steps=1)
    assert o.intrinsics_k4().shape == (3, F, 4) and o.extrinsics().shape == (3, F, 4, 4)
    assert o.gradients()["depth"].shape == (3, F, H, 96) and o.gradients()["focal"].shape == (3,)
    assert all(m.state_dict()["backbone.depth"].shape == (F, H, 96) for m in o.models)
    dev = o.rt.device
    flows = Flows(*(torch.cat([getattr(v[2], n) for v in videos[::-1]]).to(dev)
                    for n in ("forward", "backward", "forward_mask", "backward_mask")))
    o.set_flows(flows)
    expect = torch.stack([(v[2].forward_mask.double().sum() + v[2].backward_mask.double().sum()) for v in videos[::-1]])
    assert torch.allclose(o._msum.cpu(), expect, rtol=1e-7)  # k_mask_sum adds float pairs before float64
