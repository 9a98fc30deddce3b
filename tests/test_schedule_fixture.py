"""The inputs and fixtures of the whole-schedule comparison (test_gpu_full_schedule.py), on the CPU: the inputs keep
their promises, and the fixtures match the layout schedule_checks describes and the schedule the reference runs."""
import numpy as np
import pytest
import torch

import schedule_checks as S
from conftest import GOLDEN


def _load(f64):
    with np.load(GOLDEN / f"schedule{'_f64' if f64 else ''}.npz") as z:
        return {k: z[k] for k in z.files}


def test_schedule_inputs_are_float32_values_and_keep_their_tracks_inside_the_margin():
    inp = S.schedule_inputs(S.SEED)
    fl = inp["flows"]
    for t in (inp["depth"], fl.forward, fl.backward, fl.forward_mask, fl.backward_mask, inp["gt_extrinsics"],
              *(seg.xy for seg in inp["tracks"])):
        assert t.dtype == torch.float64 and torch.equal(t, t.float().double())
    assert inp["depth"].shape == (S.FRAMES, S.HEIGHT, S.WIDTH)
    assert [(seg.start_frame, seg.xy.shape[1]) for seg in inp["tracks"]] == [(0, S.FRAMES)] * 3
    for seg in inp["tracks"]:
        n = seg.xy.shape[2]
        assert S.TRACK_POINTS // 3 <= n < S.TRACK_POINTS  # the margin drops some points, not most
        assert bool(((seg.xy >= S.TRACK_MARGIN) & (seg.xy <= 1 - S.TRACK_MARGIN)).all())
        assert 0.8 < float(seg.visibility.float().mean()) < 0.97  # only the random occlusions remain
    again = S.schedule_inputs(S.SEED)
    assert torch.equal(again["depth"], inp["depth"]) and torch.equal(again["tracks"][2].xy, inp["tracks"][2].xy)


@pytest.mark.parametrize("f64", [False, True], ids=["f32", "f64"])
def test_schedule_fixture_layout(f64):
    g = _load(f64)
    assert (int(g["frames"]), int(g["height"]), int(g["width"])) == (S.FRAMES, S.HEIGHT, S.WIDTH)
    assert int(g["seed"]) == S.SEED and int(g["steps"]) == S.STEPS and int(g["stride"]) == S.STRIDE
    assert g["checkpoints"].tolist() == list(S.CHECKPOINTS) and g["pose_steps"].tolist() == S.POSE_STEPS
    assert g["border_steps"].tolist() == list(S.BORDER_STEPS)
    for key in ("loss", "loss_flow", "loss_tracking", "fx"):
        assert g[key].shape == (S.STEPS,) and np.isfinite(g[key]).all()
    assert np.allclose(g["loss"], g["loss_flow"] + g["loss_tracking"], rtol=1e-6)
    assert (g["loss_tracking"][:50] == 0).all() and (g["loss_tracking"][50:] > 0).all()
    assert g["extrinsics"].shape == (len(S.POSE_STEPS), S.FRAMES, 3, 4)
    assert g["window"].shape == (100,) and abs(g["window"].mean() - float(g["handover"])) <= 1e-6
    # fx follows the sweep up to step 999 and is the regressed focal length from step 1000 on, seeded there
    assert abs(g["fx"][1000] - float(g["handover"]) * S.HEIGHT ** 0.5 / S.WIDTH ** 0.5) <= 1e-6
    assert g["extrinsics"].dtype == np.float32  # 6e-8 of storage rounding under a 5e-5 bar
    for s in S.CHECKPOINTS:
        assert g[f"depth_s{s}_upd_norms"].shape == (S.FRAMES,) and g[f"wlog_s{s}_upd_norms"].shape == (S.FRAMES - 1,)
        assert (g[f"depth_s{s}_upd_norms"] > 0).all() and (g[f"wlog_s{s}_upd_norms"] > 0).all()
    # reduced forms only (make_golden_schedule.py): each fixture stays well under a megabyte
    assert (GOLDEN / f"schedule{'_f64' if f64 else ''}.npz").stat().st_size <= 600_000
    if f64:  # the generator's self-check: no predicted target of a visible triple near the border
        assert g["border_distance"].min() >= S.BORDER_MIN


def test_schedule_fixtures_agree_to_float32_rounding():
    """The float32 run stays close to the float64 one over the whole schedule: the comparison is well posed."""
    g32, g64 = _load(False), _load(True)
    assert np.max(np.abs(g32["loss"] - g64["loss"]) / g64["loss"]) <= 1e-3
    assert np.max(np.abs(g32["fx"] - g64["fx"])) <= 1e-4
    assert np.max(np.abs(g32["extrinsics"] - g64["extrinsics"])) <= 1e-4
    assert np.max(np.abs(g32["window"] - g64["window"])) <= 1e-4
