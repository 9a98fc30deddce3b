"""Videos of different lengths optimised as one fused step (FusedOverfitter with lists of one-video inputs).

Video b must follow a one-video FusedOverfitter on video b at its own frame count F_b (same cfg, same
step-clock seed) to the noise of the float atomics, with the tolerances of test_gpu_batched_overfit.py."""
import re

import pytest
import torch

from conftest import ROOT

gpu = pytest.mark.gpu
H, STEPS, SEED = 72, 8, 1234
FRAMES = (4, 10, 7)


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


def test_video_layout_field_order_matches_the_header():
    from flowmap_b200._lib import VideoLayout
    assert [f[0] for f in VideoLayout._fields_] == _header_struct_fields("fm_video_layout")


def _cpu_video(f, h=8, w=8):
    from flowmap_b200.types import Batch, Flows
    batch = Batch(torch.zeros(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    flows = Flows(torch.zeros(1, f - 1, h, w, 2), torch.zeros(1, f - 1, h, w, 2), torch.ones(1, f - 1, h, w),
                  torch.ones(1, f - 1, h, w))
    return batch, flows


def test_ragged_step_validates_its_inputs():
    """Refused before anything reaches the device: videos of different H x W, a video of one frame, Flows
    that are not (1, F_b - 1, H, W, ...), a bound Model, and pair sharding."""
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg, ShardedFusedOverfitter
    (b4, f4), (b6, f6) = _cpu_video(4), _cpu_video(6)
    cfg = OverfitCfg()
    with pytest.raises(ValueError, match="same H x W"):
        FusedOverfitter(cfg, [b4, _cpu_video(6, w=12)[0]], [f4, _cpu_video(6, w=12)[1]])
    b1, _ = _cpu_video(1)
    with pytest.raises(ValueError, match="frame"):
        FusedOverfitter(cfg, [b4, b1], [f4, f4])
    with pytest.raises(ValueError, match=r"\(1, F_b-1, H, W\)"):
        FusedOverfitter(cfg, [b4, b6], [f4, f4])
    with pytest.raises(ValueError, match="one Flows per Batch"):
        FusedOverfitter(cfg, [b4, b6], [f4])
    with pytest.raises(ValueError, match="Model"):
        FusedOverfitter(cfg, [b4, b6], [f4, f6], model=object())
    with pytest.raises(ValueError, match="one segment list per video"):
        FusedOverfitter(OverfitCfg(use_tracking=True), [b4, b6], [f4, f6], [[]])
    with pytest.raises(ValueError, match="one video"):
        ShardedFusedOverfitter(cfg, [b4, b6], [f4, f6], plan=None)


def test_packed_tracks_of_videos_of_different_lengths():
    """Segment s of video b is packed with start frame fo_b + s.start_frame (fo_b = frames of the videos
    before it); a segment that leaves its own video is refused."""
    from flowmap_b200 import ops
    from flowmap_b200.types import Tracks
    g = torch.Generator().manual_seed(0)
    seg = lambda rows, n, start: Tracks(torch.rand(1, rows, n, 2, generator=g),  # noqa: E731
                                        torch.rand(1, rows, n, generator=g) < 0.5, start)
    videos = [[seg(3, 5, 0), seg(2, 4, 2)], [], [seg(4, 6, 1)]]
    pk = ops.PackedTracks(videos, "cpu", video_frames=[4, 2, 6])
    assert pk.seg.tolist() == [[0, 3, 5, 0], [15, 2, 4, 2], [23, 4, 6, 4 + 2 + 1]]
    flat = [t for v in videos for t in v]
    assert torch.equal(pk.xy, torch.cat([t.xy[0].reshape(-1, 2) for t in flat]))
    with pytest.raises(ValueError, match="leaves its 4 frames"):
        ops.PackedTracks([[seg(3, 5, 2)], []], "cpu", video_frames=[4, 6])
    with pytest.raises(ValueError, match="one frame count per video"):
        ops.PackedTracks([[seg(3, 5, 0)]], "cpu", video_frames=[4, 6])


# ---------------------------------------------------------------------------------------------- GPU
def _videos(kind, w, frames=FRAMES, h=H):
    """One video per frame count: (depth (F,h,w), weight logits (F-1,h,w), Flows (1, ...), tracks)."""
    import bench
    from oracle.flowmap_oracle import flow_regime
    from flowmap_b200.types import Flows, Tracks
    out = []
    for i, f in enumerate(frames):
        if kind == "synthetic":
            inp = bench.synthetic_inputs(f, h, w, seed=i)
            depth, wl = 1.0 + inp["depth"], inp["wparam"]
            flows = Flows(inp["fwd"], inp["bwd"], inp["fmask"], inp["bmask"])
        else:
            depth, fl, _, _ = flow_regime(("shift", "outliers", "scene")[i % 3], f, h, w, seed=i)
            depth = depth[0].float()
            wl = 0.01 * torch.randn(f - 1, h, w, generator=torch.Generator().manual_seed(i))
            flows = Flows(*(getattr(fl, n).float() for n in ("forward", "backward", "forward_mask", "backward_mask")))
        tracks = [Tracks(xy, vis, st) for xy, vis, st in
                  bench.synthetic_track_arrays(f, n_points=48 + 40 * i, interval=3 + i % 3, radius=2, seed=i)] \
            if f >= 4 else []
        out.append((depth, wl, flows, tracks))
    return out


def _batch(f, h, w, dev, extrinsics=None, intrinsics=None):
    from flowmap_b200.types import Batch
    return Batch(torch.zeros(1, f, 3, h, w, device=dev), torch.arange(f, device=dev)[None], ["s"], ["d"],
                 extrinsics=extrinsics, intrinsics=intrinsics)


def _run(cfg, videos, graph, ragged=True, steps=STEPS, gt=None, log=0):
    """Optimise `videos` as one ragged FusedOverfitter (or one video alone through the tensor path when
    ragged is False): per step the losses (B,) and each video's rt; at the end depth, logits, focal."""
    from flowmap_b200.overfit import FusedOverfitter
    from flowmap_b200.types import Flows
    dev = torch.device("cuda:0")
    h, w = videos[0][0].shape[-2:]
    gt = gt or [(None, None)] * len(videos)
    flows = [Flows(*(getattr(v[2], n).to(dev) for n in ("forward", "backward", "forward_mask", "backward_mask")))
             for v in videos]
    batches = [_batch(v[0].shape[0], h, w, dev, *g) for v, g in zip(videos, gt)]
    if ragged:
        tracks = [v[3] for v in videos] if cfg.use_tracking else None
        o = FusedOverfitter(cfg, batches, flows, tracks, device=dev)
    else:
        assert len(videos) == 1
        o = FusedOverfitter(cfg, batches[0], flows[0], videos[0][3] if cfg.use_tracking else None, device=dev)
    o._clock.base_seed = SEED
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
        losses.append(total.reshape(-1).clone())
        rts.append([r.clone() for r in rt] if ragged else [rt[0].clone()])
    torch.cuda.synchronize()
    depth = [m.backbone.depth.detach().clone() for m in o.models]
    logits = [m.backbone.weights.detach().clone() for m in o.models]
    return torch.stack(losses), rts, depth, logits, o._focal.reshape(-1).clone(), o


def _rel_l2(a, b):
    return float((a - b).norm() / b.norm())


def _assert_matches_solo(cfg, videos, graph, loss_tol, steps=STEPS, focal_tol=None):
    """Each video of one packed run against its solo run, step by step (videos of any H, W and lengths).
    focal_tol: an absolute tolerance for the final focal length instead of 1e-6 of it."""
    lb, rb, db, wb, fb, o = _run(cfg, videos, graph, steps=steps)
    if graph:
        assert len(o._graphs) >= 1
    for i, v in enumerate(videos):
        ls, rs, ds, ws, fs, _ = _run(cfg, [v], graph, ragged=False, steps=steps)
        assert float(((lb[:, i] - ls[:, 0]).abs() / ls[:, 0].abs().clamp_min(1e-30)).max()) <= loss_tol, i
        assert _rel_l2(db[i], ds[0]) <= 1e-5, i
        assert float((wb[i] - ws[0]).abs().max()) <= 1e-5, i
        f_tol = 1e-6 * abs(float(fs[0])) if focal_tol is None else focal_tol
        assert abs(float(fb[i]) - float(fs[0])) <= f_tol, (i, float(fb[i]), float(fs[0]))
        for k in range(steps):
            assert float((rb[k][i] - rs[k][0]).abs().max()) <= 2e-6, (i, k)
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
def test_ragged_step_equals_solo_runs(kind, w, config, graph):
    """Videos of 4, 10 and 7 frames in one step follow three one-video runs at their own frame counts,
    step by step: loss, poses, and at the end depth, weight logits and focal length."""
    cfg, loss_tol = _cfgs()[config]
    _assert_matches_solo(cfg, _videos(kind, w), graph, loss_tol)


@gpu
@pytest.mark.parametrize("config", ["regressed", "softmin_handover"])
def test_a_two_frame_video_among_longer_ones(config):
    """A video of 2 frames has only pair 0: the softmin stage's "frames >= 2" Adam pass skips it."""
    cfg, loss_tol = _cfgs()[config]
    _assert_matches_solo(cfg, _videos("synthetic", 96, frames=(5, 2, 7)), True, loss_tol)


@gpu
def test_equal_lengths_equal_the_tensor_path():
    """A list of equal-length videos gives what the (B, F) tensor batch gives."""
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows
    cfg = OverfitCfg(intrinsics="softmin", regression_after=4, regression_window=2, softmin_points=500)
    videos = _videos("synthetic", 96, frames=(6, 6, 6))
    lr, rr, dr, wr, fr, _ = _run(cfg, videos, True)
    dev = torch.device("cuda:0")
    batch = Batch(torch.zeros(3, 6, 3, H, 96, device=dev), torch.arange(6, device=dev)[None].expand(3, 6), ["s"] * 3,
                  ["d"] * 3)
    flows = Flows(*(torch.cat([getattr(v[2], n) for v in videos]).to(dev)
                    for n in ("forward", "backward", "forward_mask", "backward_mask")))
    o = FusedOverfitter(cfg, batch, flows, device=dev)
    o._clock.base_seed = SEED
    with torch.no_grad():
        for m, (depth, wl, _, _) in zip(o.models, videos):
            m.backbone.depth.copy_(depth)
            m.backbone.weights.copy_(wl)
    o.use_cuda_graph = True
    for k in range(STEPS):
        total, rt = o.training_step()
        assert float(((lr[k] - total).abs() / total.abs()).max()) <= 1e-5, k
        for i in range(3):
            assert float((rr[k][i] - rt[i]).abs().max()) <= 2e-6, (k, i)
    for i in range(3):
        assert _rel_l2(dr[i], o._depth[i]) <= 1e-5 and float((wr[i] - o._wlog[i]).abs().max()) <= 1e-5
    assert torch.allclose(fr, o._focal, rtol=1e-6)


@gpu
def test_each_video_has_its_own_normalisers():
    """Video 1 without any valid flow has loss 0 ("or 1" applies to it alone) and the others follow their
    solo runs; with track sets of different sizes every video's tracking loss is its solo one."""
    from flowmap_b200.overfit import OverfitCfg
    videos = _videos("synthetic", 96)
    videos[1][2].forward_mask.zero_()
    videos[1][2].backward_mask.zero_()
    lb = _assert_matches_solo(OverfitCfg(), videos, False, 1e-6)
    assert float(lb[:, 1].abs().max()) == 0.0 and float(lb[:, 0].min()) > 0.0
    cfg = OverfitCfg(use_tracking=True, tracking_enable_after=0)
    videos = _videos("synthetic", 96)
    *_, o = _run(cfg, videos, False, steps=2)
    for i, v in enumerate(videos):
        *_, s = _run(cfg, [v], False, ragged=False, steps=2)
        assert abs(float(o._track_loss[i]) - float(s._track_loss)) <= 1e-5 * abs(float(s._track_loss)), i
        assert float(s._track_loss) > 0.0


@gpu
@pytest.mark.parametrize("config", ["regressed", "softmin_tracking"])
def test_ragged_metrics_rows_equal_solo_rows(config):
    """The (steps, B) metrics log holds every video's solo rows, the ATE over its own F_b camera centres;
    video 1 has no ground truth: its columns are NaN."""
    from oracle.flowmap_oracle import flow_regime
    cfg = _cfgs()[config][0]
    videos = _videos("synthetic", 96)
    gt = []
    for i, f in enumerate(FRAMES):
        ext = flow_regime("scene", f, H, 96, seed=i)[3][0].float()[None]
        k = torch.eye(3).expand(1, f, 3, 3).clone()
        k[..., 0, 0], k[..., 1, 1] = 0.8, 0.9
        k[..., :2, 2] = 0.5
        gt.append((None, None) if i == 1 else (ext, k))
    *_, o = _run(cfg, videos, True, gt=gt, log=16)
    log = o.metrics_log()
    assert all(t.shape == (STEPS, 3) for t in log.values())
    for i, v in enumerate(videos):
        *_, s = _run(cfg, [v], True, ragged=False, gt=[gt[i]], log=16)
        solo = s.metrics_log()
        for name in log:
            a, b = log[name][:, i], solo[name]
            assert torch.equal(a.isnan(), b.isnan()), (i, name)
            a, b = a[~b.isnan()].double(), b[~b.isnan()].double()
            if b.numel():
                assert float((a - b).abs().max()) <= 1e-5 * max(1.0, float(b.abs().max())), (i, name)
        assert bool(log["metrics/ate"][:, i].isnan().all()) == (i == 1)


@gpu
def test_ragged_step_surface():
    """Per-video shapes of what the optimiser hands out, parameters as views into the packed buffers,
    and set_flows with a list."""
    from flowmap_b200.overfit import OverfitCfg
    from flowmap_b200.types import Flows
    videos = _videos("synthetic", 96)
    _, rts, _, _, _, o = _run(OverfitCfg(), videos, False, steps=1)
    assert [r.shape for r in rts[0]] == [(f - 1, 3, 4) for f in FRAMES]
    assert [k.shape for k in o.intrinsics_k4()] == [(f, 4) for f in FRAMES]
    assert [e.shape for e in o.extrinsics()] == [(f, 4, 4) for f in FRAMES]
    g = o.gradients()
    assert [t.shape for t in g["depth"]] == [(f, H, 96) for f in FRAMES]
    assert [t.shape for t in g["weights"]] == [(f - 1, H, 96) for f in FRAMES]
    assert len(g["focal"]) == 3
    assert o._depth.shape == (sum(FRAMES), H, 96) and o._wlog.shape == (sum(FRAMES) - 3, H, 96)
    first = 0
    for m, f in zip(o.models, FRAMES):
        assert m.state_dict()["backbone.depth"].shape == (f, H, 96)
        assert m.backbone.depth.data_ptr() == o._depth[first].data_ptr()
        assert m.backbone.weights.data_ptr() == o._wlog[first - o.models.index(m)].data_ptr()
        first += f
    dev = o.rt.device
    new = [Flows(*(getattr(v[2], n).flip(-2).contiguous().to(dev)
                   for n in ("forward", "backward", "forward_mask", "backward_mask"))) for v in videos]
    for fl in new:
        fl.forward_mask.mul_(0.5)
    o.set_flows(new)
    expect = torch.stack([(f.forward_mask.double().sum() + f.backward_mask.double().sum()).cpu() for f in new])
    assert torch.allclose(o._msum.cpu(), expect, rtol=1e-7)
    with pytest.raises(ValueError, match="one Flows per video"):
        o.set_flows(new[:2])
    with pytest.raises(ValueError, match="split-step"):
        o.forward_phase(0)
