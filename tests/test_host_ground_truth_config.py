"""OverfitCfg(intrinsics="ground_truth") builds the reference's IntrinsicsGroundTruth (no focal parameter, the
reference's state_dict names), on the host."""
from flowmap_b200.model import IntrinsicsGroundTruth
from flowmap_b200.overfit import OverfitCfg, build_model_and_losses


def test_ground_truth_cfg_builds_ground_truth_intrinsics():
    model, losses = build_model_and_losses(OverfitCfg(intrinsics="ground_truth", use_tracking=True), 4, (8, 12))
    assert type(model.intrinsics) is IntrinsicsGroundTruth
    assert sorted(model.state_dict()) == ["backbone.depth", "backbone.weights"]
    assert not any("focal" in name for name, _ in model.named_parameters())
    assert len(losses) == 2
    regressed, _ = build_model_and_losses(OverfitCfg(), 4, (8, 12))
    assert "intrinsics.focal_length" in regressed.state_dict()
