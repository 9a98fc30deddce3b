"""Inputs and fixture layout of the whole-schedule comparison (tests/golden/make_golden_schedule.py writes the
fixtures from the unmodified reference, test_gpu_full_schedule.py replays the run on the GPU): one overfit run of
the reference's default schedule -- 2000 Adam steps, the tracking loss from step 50, the softmin sweep's focal
estimates collected from step 900 and the focal length regressed from step 1000 -- on a scene whose flows and
tracks are exact, so the run converges towards a known camera path and focal length.

Both sides build their inputs here, from seeds; the fixtures hold no inputs."""
import torch

from flow_regime_checks import start_point
from oracle import flowmap_oracle as O
from track_travel_checks import reference_segments

SEED = 0
FRAMES, HEIGHT, WIDTH = 12, 64, 96
STEPS = 2000
TRACK_POINTS = 300
TRACK_MARGIN = 0.05  # a kept track point's true projection stays this far inside [0,1)^2 in every frame
STRIDE = 7  # the strided subsample of a parameter update: prime to the row length and the frame size
# the parameters these steps evaluate (before their own update); STEPS: the final ones, after the last update
CHECKPOINTS = (50, 900, 1000, 1999, STEPS)
POSE_STEPS = sorted(set(range(0, STEPS, 10)) | set(range(48, 53)) | set(range(898, 903)) | set(range(998, 1004)))
BORDER_STEPS = tuple(range(0, STEPS, 10))
BORDER_MIN = 1e-3  # the float64 run's predicted targets of visible triples stay this far from the border


def _f32(t):
    """The float32 value of t, held in float64: both precisions of a run then start from the same numbers."""
    return t.to(torch.float32).to(torch.float64)


def schedule_inputs(seed=SEED):
    """The scene of the whole-schedule run, float32-representable values in float64 tensors.

    oracle.consistent_scene(12, 64, 96): 64 x 96 is 2 x 2 window tiles of the Procrustes backward, W = 96 takes
    its fused logit Adam, and 6144 pixels are fewer than the sweep's 8192 softmin points, so the sweep samples
    every pixel and any sampling order gives the same focal estimate up to summation order.  The start depth
    is flow_regime_checks.start_point's (depth x (1 + N(0, 0.02^2))), the weight logits start at 0.  The tracks
    are oracle.scene_tracks on the reference's segment layout, 300 points per segment, of which only the
    points whose true projections stay inside [0.05, 0.95]^2 in every frame of their segment are kept: no
    predicted target comes near the border over the run, where validity could differ between precisions.

    Returns a dict: depth (start, (F, H, W)), flows (oracle.Flows), tracks (list of oracle.Tracks),
    gt_extrinsics (1, F, 4, 4), gt_intrinsics (1, F, 3, 3), focal (the true one)."""
    f, h, w = FRAMES, HEIGHT, WIDTH
    depth, flows, focal, ext = O.consistent_scene(f, h, w, seed=seed)
    start, _ = start_point(depth, focal, seed + 1)
    tracks = []
    for seg in O.scene_tracks(depth, ext, focal, reference_segments(f), TRACK_POINTS, seed=seed):
        keep = ((seg.xy[0] >= TRACK_MARGIN) & (seg.xy[0] <= 1 - TRACK_MARGIN)).all(dim=-1).all(dim=0)
        tracks.append(O.Tracks(_f32(seg.xy[:, :, keep]), seg.visibility[:, :, keep].clone(), seg.start_frame))
    k = O.intrinsics_from_focal(torch.tensor(focal, dtype=torch.float64), h, w).expand(1, f, 3, 3)
    return dict(depth=_f32(start), flows=O.Flows(*(_f32(getattr(flows, n)) for n in
                                                   ("forward", "backward", "forward_mask", "backward_mask"))),
                tracks=tracks, gt_extrinsics=_f32(ext), gt_intrinsics=_f32(k).contiguous(), focal=focal)


def reduced_update(name, value, start):
    """What a fixture keeps of a parameter at a checkpoint: the per-frame L2 norms of the value and of the
    update (value - start), float64, and every STRIDE-th element of the update, float32."""
    value, upd = value.detach().double(), value.detach().double() - start.double()
    return {f"{name}_norms": value.flatten(1).norm(dim=1).numpy(),
            f"{name}_upd_norms": upd.flatten(1).norm(dim=1).numpy(),
            f"{name}_upd_sub": upd.flatten()[::STRIDE].float().numpy()}


def border_distance(surfaces, ext, k, tracks):
    """The smallest distance from the border of [0,1)^2 of any predicted target (oracle.track_positions) of a
    triple whose two ends are visible and whose source lies inside."""
    best = float("inf")
    for seg in tracks:
        s, n_f = seg.start_frame, seg.xy.shape[1]
        target, _ = O.track_positions(surfaces[:, s:s + n_f], ext[:, s:s + n_f], k[:, s:s + n_f], seg)
        vis = seg.visibility[0]
        cand = (vis & ((seg.xy[0] >= 0) & (seg.xy[0] < 1)).all(dim=-1))[:, None] & vis[None]
        t = target[0][cand]
        if t.numel():
            best = min(best, float(torch.minimum(t.abs(), (1 - t).abs()).min()))
    return best
