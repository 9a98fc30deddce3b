"""CPU checks of the inputs and reference computations of test_gpu_tracking_travel.py (track_travel_checks):
the travelling scene is what it claims to be, the border guard does what it claims with little loss of
data, and the segment-at-a-time oracle loss is the oracle's tracking loss."""
import pytest
import torch

import track_travel_checks as T
from conftest import max_abs, rel_l2
from oracle import flowmap_oracle as O


@pytest.mark.parametrize("f,h,w", [(42, 24, 32), (150, 12, 16)])
def test_travel_scene_depths_and_travel(f, h, w):
    """Depths are finite and within the cylinder's 3 (rays at most ~0.5 off its cross-section plane), and
    the last camera is 0.25 (f - 1) from frame 0's."""
    depth, _, _, ext = T.travel_scene(f, h, w, seed=1)
    assert bool(torch.isfinite(depth).all())
    assert 2.5 <= float(depth.min()) and float(depth.max()) <= 3.2
    assert abs(float(ext[0, -1, :3, 3].norm()) - 0.25 * (f - 1)) < 1e-12
    assert float(ext[0, -1, :3, 3].norm()) >= {42: 10.0, 150: 37.0}[f]
    r = ext[0, :, :3, :3]
    assert max_abs(r @ r.transpose(-1, -2), torch.eye(3, dtype=torch.float64).expand_as(r)) < 1e-12


def test_travel_scene_flows_round_trip():
    """The backward flow of frame i+1, sampled where the forward flow takes frame i's pixels, brings them back
    (the exact induced flows of one static surface), wherever the forward target is inside the frame."""
    f, h, w = 6, 48, 64
    _, fl, _, _ = T.travel_scene(f, h, w, seed=2)
    xy = O.pixel_grid(h, w, torch.float64)
    target = xy + fl.forward[0]  # (f-1, h, w, 2) in frame i+1
    img = fl.backward[0].permute(0, 3, 1, 2)
    back = target + O.bilinear_border(img, target.reshape(f - 1, -1, 2)).reshape(f - 1, h, w, 2)
    margin = 1.0 / min(h, w)
    inside = ((target > margin) & (target < 1 - margin)).all(dim=-1)
    assert float(inside.float().mean()) > 0.5  # the cameras move a fifth of the frame or less per step
    assert float((back - xy)[inside].abs().max()) < 1e-3  # bilinear interpolation of a smooth flow


def test_reference_segments_are_synthetic_tracks_layout():
    for f in (6, 42, 150):
        got = [(t.start_frame, t.xy.shape[1]) for t in O.synthetic_tracks(f, n_points=3)]
        assert T.reference_segments(f) == got
        assert max(r for _, r in got) == min(f, 41)


@pytest.mark.parametrize("kind", ["consistent", "uniform"])
def test_guard_clears_every_near_border_triple(kind):
    """On a 42-frame travelling video with 41-row segments: many predicted targets cross the border, the guard
    leaves no triple within the band of it, clears fewer than 0.5 % of the visible samples, and clears
    nothing it need not (every cleared sample was the target of a near-border triple)."""
    f, h, w = 42, 24, 32
    depth, _, focal, ext = T.travel_scene(f, h, w, seed=3)
    if kind == "consistent":
        tracks = O.scene_tracks(depth, ext, focal, T.reference_segments(f), n_points=300, seed=3)
    else:
        tracks = O.synthetic_tracks(f, n_points=300, seed=3, dtype=torch.float64)
    k = O.intrinsics_from_focal(torch.tensor(focal, dtype=torch.float64), h, w).expand(1, f, 3, 3)
    surf = O.unproject(O.pixel_grid(h, w, torch.float64), depth[None], k[:, :, None, None])
    t64 = T.track_triples(surf, ext, k, tracks)
    t32 = T.track_triples(surf.float(), ext.float(), k.float(),
                          [O.Tracks(t.xy.float(), t.visibility, t.start_frame) for t in tracks])
    band = T.position_band(t64, t32, tracks)
    assert 1e-5 <= band < 1e-3
    assert T.border_crossings(tracks, t64) > 5000
    before = T.near_border_triples(tracks, t64, band)
    guarded, cleared = T.clear_track_kinks(tracks, t64, band)
    samples = sum(int(t.visibility.sum()) for t in tracks)
    assert before > 0 and 0 < cleared < 5e-3 * samples
    assert T.near_border_triples(guarded, t64, band) == 0
    assert sum(int(t.visibility.sum()) for t in guarded) == samples - cleared
    # a wider band only clears more
    assert T.clear_track_kinks(tracks, t64, 4 * band)[1] >= cleared


def test_tracking_loss_by_segment_is_the_oracle_loss():
    """Loss, count and gradients (surfaces, extrinsics, intrinsics) of the segment-at-a-time float64 loss
    equal oracle.tracking_loss's, with overlapping segments."""
    f, h, w = 9, 12, 16
    depth, _, focal, ext = T.travel_scene(f, h, w, seed=4)
    tracks = O.synthetic_tracks(f, n_points=40, interval=3, radius=3, seed=4, dtype=torch.float64)
    k = O.intrinsics_from_focal(torch.tensor(focal, dtype=torch.float64), h, w).expand(1, f, 3, 3).contiguous()
    surf = O.unproject(O.pixel_grid(h, w, torch.float64), depth[None], k[:, :, None, None])
    leaves = [[t.clone().requires_grad_(True) for t in (surf, ext, k)] for _ in range(2)]
    ref = 100.0 * O.tracking_loss(*leaves[0], tracks)
    ref.backward()
    loss, count = T.tracking_loss_by_segment(*leaves[1], tracks, weight=100.0)
    assert count == sum(int(v.sum()) for _, v in T.track_triples(surf, ext, k, tracks)) > 0
    assert abs(loss - float(ref)) <= 1e-12 * abs(float(ref))
    for a, b in zip(leaves[1], leaves[0]):
        assert rel_l2(a.grad, b.grad) <= 1e-12
