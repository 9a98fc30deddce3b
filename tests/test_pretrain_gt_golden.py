"""Pins the oracle's pretraining step with ground-truth intrinsics (tests/pretrain_gt_checks.py: one video at a
time under the pooled mask sum, K per video and per frame) against the unmodified reference's
`Model(IntrinsicsGroundTruth)` + `LossFlow` at B > 1 (tests/golden/pretrain_gt*.npz, produced by
tests/golden/make_golden_pretrain_gt.py).  CPU only."""
import pytest
import torch

from conftest import load_golden, max_abs, rel_l2
from pretrain_gt_checks import pretrain_gt_oracle

T = torch.as_tensor


def _run(g, dtype):
    from oracle import flowmap_oracle as O
    b, f, h, w = g["in_depths"].shape
    flows = O.Flows(*(T(g[k]) for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    pidx = torch.linspace(0, h * w - 1, int(g["procrustes_points"]), dtype=torch.int64)
    return pretrain_gt_oracle(T(g["in_depths"]), T(g["in_weights"]), flows, T(g["in_intrinsics"]), pidx, dtype=dtype)


@pytest.mark.parametrize("f64", [False, True])
def test_oracle_ground_truth_pretraining_step_matches_the_reference(f64):
    """Loss, each video's extrinsics, d loss / d depths and d loss / d weights of every video."""
    g = load_golden("pretrain_gt", f64)
    r = _run(g, torch.float64 if f64 else torch.float32)
    assert g["in_depths"].shape[0] > 1
    tol = 1e-12 if f64 else 2e-5
    gtol = 1e-10 if f64 else 2e-4
    assert abs(r["loss"] - float(g["loss"])) <= tol * abs(float(g["loss"])), (r["loss"], float(g["loss"]))
    assert max_abs(r["ext"], g["extrinsics"]) <= (1e-10 if f64 else 2e-5)
    for v in range(g["in_depths"].shape[0]):
        assert rel_l2(r["g_depth"][v], g["g_depths"][v]) <= gtol, (v, rel_l2(r["g_depth"][v], g["g_depths"][v]))
        assert rel_l2(r["g_w"][v], g["g_weights"][v]) <= gtol, (v, rel_l2(r["g_w"][v], g["g_weights"][v]))


def test_golden_batch_has_per_video_per_frame_off_centre_intrinsics():
    """The fixture tells per-video, per-frame K from a shared or centred one: every frame's K differs, every
    principal point is off centre, and the mask sums are more than 2x apart from one video to the next."""
    g = load_golden("pretrain_gt", True)
    k = T(g["in_intrinsics"]).flatten(0, 1)
    assert len({tuple(x.tolist()) for x in k[:, :2].reshape(len(k), -1)}) == len(k)
    assert float((k[:, :2, 2] - 0.5).abs().min()) > 1e-3
    m = (T(g["in_fmask"]).sum(dim=(1, 2, 3)) + T(g["in_bmask"]).sum(dim=(1, 2, 3))).tolist()
    assert all(m[v] > 2.0 * m[v + 1] for v in range(len(m) - 1)), m
