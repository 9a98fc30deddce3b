"""Pins the oracle's pretraining step (tests/pretrain_checks.py: one video at a time under the pooled mask
sum) against the unmodified reference's `Model` + `LossFlow` at B > 1 (tests/golden/pretrain*.npz, produced
by tests/golden/make_golden_pretrain.py).  CPU only.

The golden batches' mask sums fall by more than 2x from one video to the next, so a per-video normaliser,
or the sum of the videos' own losses, is far off the reference's batch loss and gradients."""
import pytest
import torch

from conftest import load_golden, max_abs, rel_l2
from pretrain_checks import pretrain_oracle

T = torch.as_tensor


def _run(g, dtype):
    from oracle import flowmap_oracle as O
    b, f, h, w = g["in_depths"].shape
    flows = O.Flows(*(T(g[k]) for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    pts = int(g["procrustes_points"])
    pidx = None if pts < 0 else torch.linspace(0, h * w - 1, pts, dtype=torch.int64)
    return pretrain_oracle(T(g["in_depths"]), T(g["in_weights"]), flows, T(g["indices"]),
                           torch.linspace(0.5, 2.0, 60, dtype=torch.float64), pidx, dtype=dtype, use_weights=bool(g["use_weights"]))


@pytest.mark.parametrize("name", ["pretrain", "pretrain_noweights"])
@pytest.mark.parametrize("f64", [False, True])
def test_oracle_pretraining_step_matches_the_reference(name, f64):
    """Loss, each video's intrinsics and extrinsics, d loss / d depths and d loss / d weights of every video."""
    g = load_golden(name, f64)
    r = _run(g, torch.float64 if f64 else torch.float32)
    b, f = g["in_depths"].shape[:2]
    assert b > 1
    tol = 1e-12 if f64 else 2e-5
    gtol = 1e-10 if f64 else 2e-4
    assert abs(r["loss"] - float(g["loss"])) <= tol * abs(float(g["loss"])), (r["loss"], float(g["loss"]))
    assert max_abs(r["k"], T(g["intrinsics"])[:, 0]) <= tol * 10
    assert max_abs(r["k"][:, None].expand(b, f, 3, 3), g["intrinsics"]) <= tol * 10
    assert max_abs(r["ext"], g["extrinsics"]) <= (1e-10 if f64 else 2e-5)
    for v in range(b):
        assert rel_l2(r["g_depth"][v], g["g_depths"][v]) <= gtol, (v, rel_l2(r["g_depth"][v], g["g_depths"][v]))
        if r["g_w"] is not None:
            assert rel_l2(r["g_w"][v], g["g_weights"][v]) <= gtol, (v, rel_l2(r["g_w"][v], g["g_weights"][v]))
    assert ("g_weights" in g) == bool(g["use_weights"]) == (r["g_w"] is not None)


@pytest.mark.parametrize("name", ["pretrain", "pretrain_noweights"])
def test_golden_batches_separate_the_normalisers(name):
    """The fixtures tell the pooled normaliser from a per-video one and from the sum of the videos' own losses:
    the mask sums are more than 2x apart, and the sum of the videos' own-normalised losses misses the
    reference's batch loss by more than 10 %."""
    g = load_golden(name, True)
    m = (T(g["in_fmask"]).sum(dim=(1, 2, 3)) + T(g["in_bmask"]).sum(dim=(1, 2, 3))).tolist()
    assert all(m[v] > 2.0 * m[v + 1] for v in range(len(m) - 1)), m
    r = _run(g, torch.float64)
    loss = float(g["loss"])
    own = [s * r["mask_sum"] / mv for s, mv in zip(r["share"].tolist(), m)]  # video v normalised by its own sum
    assert abs(sum(own) - loss) > 0.1 * abs(loss), (sum(own), loss)
