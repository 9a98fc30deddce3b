"""Inputs and float64 reference computations for the tracking loss on videos whose cameras travel far from
frame 0 (test_gpu_tracking_travel.py; pinned on the CPU by test_track_travel_checks.py).

A (source row, target row, point) triple of a track segment counts only while its PREDICTED target lies in
[0,1)^2 (oracle.track_positions).  Once the cameras move far, many targets cross that border inside one
41-row segment, and a target within rounding of it is valid for one precision and invalid for another: a
whole saturated Huber term appears or vanishes at four taps of one frame's depth gradient.  The float64
result is then not a sharper version of the float32 one, and no rounding-level bar can hold.  So the
comparisons run on tracks from which `clear_track_kinks` has removed every target sample that takes part in
such a triple, with the band set by the float32 oracle's own position error (`position_band`)."""
import torch

from oracle import flowmap_oracle as O


def travel_scene(f, h, w, step=0.25, rotation=0.02, seed=0, focal=0.85, radius=3.0, dtype=torch.float64):
    """A video whose cameras travel far while its depths stay bounded: the surface is the inside of the
    x-aligned cylinder y^2 + z^2 = radius^2; camera i sits on the axis at x = step * i and looks along +z
    with a small random rotation (axis-angle ~ N(0, rotation^2) per component, independent per frame).
    Depths are the exact ray/cylinder roots and flows the exact induced correspondences, as in
    oracle.consistent_scene.  Returns (depth (f,h,w), Flows, focal, camera-to-world extrinsics (1,f,4,4))."""
    g = torch.Generator().manual_seed(seed)
    ang = rotation * torch.randn(f, 3, generator=g, dtype=torch.float64)
    skew = torch.zeros(f, 3, 3, dtype=torch.float64)
    skew[:, 0, 1], skew[:, 0, 2], skew[:, 1, 2] = -ang[:, 2], ang[:, 1], -ang[:, 0]
    ext = torch.eye(4, dtype=torch.float64).repeat(1, f, 1, 1)
    ext[0, :, :3, :3] = torch.linalg.matrix_exp(skew - skew.transpose(-1, -2))
    ext[0, :, 0, 3] = step * torch.arange(f, dtype=torch.float64)
    k = O.intrinsics_from_focal(torch.tensor(focal, dtype=torch.float64), h, w).expand(1, f, 3, 3)
    xy = O.pixel_grid(h, w, torch.float64)
    rays = O.unproject(xy, torch.ones(1, f, h, w, dtype=torch.float64), k[:, :, None, None])
    # ray/cylinder: |(o + z d)_yz|^2 = radius^2 with o, d the camera centre / ray (z = 1) in world space
    d = O.matvec(ext[:, :, None, None, :3, :3], rays)[..., 1:]
    o = ext[:, :, None, None, 1:3, 3]
    a_ = (d * d).sum(-1)
    b_ = 2 * (d * o).sum(-1)
    c_ = (o * o).sum(-1) - radius ** 2
    depth = ((-b_ + torch.sqrt(b_ * b_ - 4 * a_ * c_)) / (2 * a_))[0]
    surf = O.unproject(xy, depth[None], k[:, :, None, None])
    fwd = O.forward_flow_positions(surf, ext, k) - xy
    bwd = O.backward_flow_positions(surf, ext, k) - xy
    u = lambda *s: 0.5 + 0.5 * torch.rand(*s, generator=g, dtype=torch.float64)  # noqa: E731
    flows = O.Flows(fwd.to(dtype), bwd.to(dtype), u(1, f - 1, h, w).to(dtype), u(1, f - 1, h, w).to(dtype))
    return depth.to(dtype), flows, focal, ext


def reference_segments(f, interval=5, radius=20):
    """(start frame, rows) of the segments of oracle.synthetic_tracks (tracking/__init__.py:80-110)."""
    return [(max(0, mid - radius), min(f, mid + radius + 1) - max(0, mid - radius)) for mid in range(0, f, interval)]


def track_triples(surfaces, ext, k, tracks):
    """For every segment, oracle.track_positions' predicted targets (rows, rows, n, 2) (source row, target row,
    point) and validity mask (rows, rows, n), of batch item 0."""
    out = []
    for seg in tracks:
        s, n_f = seg.start_frame, seg.xy.shape[1]
        target, valid = O.track_positions(surfaces[:, s:s + n_f], ext[:, s:s + n_f], k[:, s:s + n_f], seg)
        out.append((target[0], valid[0]))
    return out


def _candidates(seg):
    """(rows, rows, n): both ends visible and the source inside [0,1)^2 -- valid but for the target test."""
    vis = seg.visibility[0]
    src = ((seg.xy[0] >= 0) & (seg.xy[0] < 1)).all(dim=-1)
    return (vis & src)[:, None] & vis[None]


def position_band(triples64, triples32, tracks, margin=10.0, floor=1e-5):
    """max(floor, margin x the largest |float32 - float64| predicted-target coordinate over the triples that
    could be valid and whose float64 target lies in [-1, 2]^2 (points near or behind a camera project to
    anywhere and decide nothing))."""
    err = 0.0
    for seg, (t64, _), (t32, _) in zip(tracks, triples64, triples32):
        near = _candidates(seg) & ((t64 > -1) & (t64 < 2)).all(dim=-1)
        if bool(near.any()):
            err = max(err, float((t32.double() - t64)[near].abs().max()))
    return max(floor, margin * err)


def border_crossings(tracks, triples):
    """Number of times a predicted target track crosses the border of [0,1)^2: over every (source row, point)
    whose source sample is visible and inside, the target rows t where inside(target_t) != inside(target_t+1)."""
    n = 0
    for seg, (t64, _) in zip(tracks, triples):
        vis = seg.visibility[0]
        src = vis & ((seg.xy[0] >= 0) & (seg.xy[0] < 1)).all(dim=-1)
        inside = ((t64 >= 0) & (t64 < 1)).all(dim=-1)  # (rows_s, rows_t, n)
        n += int(((inside[:, 1:] != inside[:, :-1]) & src[:, None]).sum())
    return n


def clear_track_kinks(tracks, triples, band):
    """Tracks without the target samples that take part in a near-border triple: every (source row, target
    row, point) whose two ends are visible, whose source is inside [0,1)^2 and whose float64 predicted target
    (triples: track_triples in float64) lies within `band` of 0 or 1 in either coordinate loses the
    visibility of its target sample; repeated until no such triple is left.  Returns (tracks, number of
    samples cleared)."""
    out, cleared = [], 0
    for seg, (t64, _) in zip(tracks, triples):
        near = ((t64.abs() < band) | ((t64 - 1).abs() < band)).any(dim=-1)
        seg = O.Tracks(seg.xy, seg.visibility.clone(), seg.start_frame)
        while True:
            kill = (_candidates(seg) & near).any(dim=0)  # (target row, point)
            n = int(kill.sum())
            if n == 0:
                break
            seg.visibility[0] &= ~kill
            cleared += n
        out.append(seg)
    return out, cleared


def near_border_triples(tracks, triples, band):
    """Number of triples clear_track_kinks would still act on."""
    return sum(int((_candidates(seg) & ((t64.abs() < band) | ((t64 - 1).abs() < band)).any(dim=-1)).sum())
               for seg, (t64, _) in zip(tracks, triples))


def tracking_loss_by_segment(surfaces, ext, k, tracks, weight=1.0, mapping="huber", delta=0.01):
    """weight x oracle.tracking_loss(surfaces, ext, k, tracks), with the gradient accumulated into whichever of
    surfaces, ext, k are leaves that require it, one segment's graph at a time: the valid count in a no-grad
    pass, then each segment's sum / count backward.  The graph of all 41 x 41 x 1225-triple segments of a long
    video at once does not fit in memory.  Returns (loss, valid count)."""
    h, w = surfaces.shape[2:4]
    with torch.no_grad():
        count = sum(int(track_triples(surfaces, ext, k, [seg])[0][1].sum()) for seg in tracks)
    scale = weight / (count if count else 1)
    total = 0.0
    for seg in tracks:
        s, n_f = seg.start_frame, seg.xy.shape[1]
        target, vis = O.track_positions(surfaces[:, s:s + n_f], ext[:, s:s + n_f], k[:, s:s + n_f], seg)
        part = scale * (O.robust_map(target, seg.xy[:, None], h, w, mapping, delta) * vis).sum()
        if part.requires_grad:
            part.backward()
        total += float(part.detach())
    return total, count
