"""The tracking sweep works on items of (segment, source row, half of the row's points): an item's
usable source points are compacted once and spread over the warps of a block in passes, in rounds of
at most 2048 points.  These cases check the fused step with tracking against the float64 oracle where
that layout has edges: a segment of >= 1000 points over >= 30 rows (several passes per warp), rows
of 4500 points (halves that need two compaction rounds), segments of different lengths down to one
row, and rows with no usable source point (all invisible, or all outside the image)."""
import pytest
import torch

from conftest import rel_l2
from test_gpu_parity import _tracking_case

pytestmark = pytest.mark.gpu


def _segments():
    from oracle import flowmap_oracle as O
    gen = torch.Generator().manual_seed(17)

    def mk(rows, n, start, vis_p=0.7):
        xy = torch.rand(1, rows, n, 2, generator=gen, dtype=torch.float64)
        vis = torch.rand(1, rows, n, generator=gen) < vis_p
        return xy, vis, start

    long_xy, long_vis, _ = mk(32, 1100, 0)
    long_xy[0, 7] += 2.0        # row 7: every source point outside [0,1)^2
    long_vis[0, 9] = False      # row 9: nothing visible
    mid_xy, mid_vis, _ = mk(17, 300, 10)
    mid_vis[0, 4] = False
    wide = mk(2, 4500, 20)      # half a row is more than one compaction round holds
    return [O.Tracks(long_xy, long_vis, 0), O.Tracks(mid_xy, mid_vis, 10), O.Tracks(*wide),
            O.Tracks(*mk(5, 70, 3)), O.Tracks(*mk(1, 10, 25))]


def test_whole_row_tracking_sweep_vs_oracle():
    segs = _segments()
    loss, gr, track_loss, ref = _tracking_case(segs, f=32, h=12, w=16)
    assert track_loss > 0.0
    ref_track = float(ref["parts"]["tracking"])
    assert abs(track_loss - ref_track) <= 1e-4 * abs(ref_track)
    assert abs(loss - ref["loss"]) <= 1e-4 * abs(ref["loss"])
    assert rel_l2(gr["depth"].cpu(), ref["grads"]["depth"]) <= 3e-4
    assert rel_l2(gr["weights"].cpu(), ref["grads"]["weights"]) <= 3e-4
