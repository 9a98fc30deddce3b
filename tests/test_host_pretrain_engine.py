"""The fused engine of a network backbone's batch of several videos (the pretraining step) refuses what the
packed split step does not serve before anything reaches the device: tracks, a regressed focal length and a
softmin regression stage.  CPU only."""
import pytest
import torch
from torch import nn


class _Net(nn.Module):
    def __init__(self, cfg, num_frames, image_shape):
        super().__init__()
        self.p = nn.Parameter(torch.zeros(()))

    def forward(self, batch, flows):  # not reached
        raise AssertionError


def _inputs(b=2, f=3, h=8, w=12):
    from flowmap_b200.model import BACKBONES, ExtrinsicsProcrustesCfg, IntrinsicsSoftminCfg, Model, ModelCfg
    from flowmap_b200.types import Batch, Flows, Tracks
    from dataclasses import make_dataclass
    BACKBONES["test_host_net"] = _Net
    cfg = make_dataclass("NetCfg", [("name", str)])("test_host_net")
    model = Model(ModelCfg(cfg, IntrinsicsSoftminCfg("softmin", 16, 0.5, 2.0, 4, None),
                           ExtrinsicsProcrustesCfg("procrustes", None, False), True), f, (h, w))
    batch = Batch(torch.zeros(b, f, 3, h, w), torch.arange(f)[None].expand(b, f), ["s"] * b, ["d"] * b)
    flows = Flows(torch.zeros(b, f - 1, h, w, 2), torch.zeros(b, f - 1, h, w, 2), torch.ones(b, f - 1, h, w),
                  torch.ones(b, f - 1, h, w))
    tracks = [Tracks(torch.rand(1, 2, 5, 2), torch.ones(1, 2, 5, dtype=torch.bool), 0)]
    return model, batch, flows, tracks


def test_network_batch_engine_refusals():
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    model, batch, flows, tracks = _inputs()
    soft = OverfitCfg(intrinsics="softmin", regression_after=None, weight_sensitivity=0.0)
    with pytest.raises(ValueError, match="no tracks"):
        FusedOverfitter(soft, batch, flows, tracks, device="cpu", model=model)
    with pytest.raises(ValueError, match="no tracks"):
        FusedOverfitter(OverfitCfg(intrinsics="softmin", regression_after=None, use_tracking=True), batch, flows,
                        device="cpu", model=model)
    for cfg in (OverfitCfg(intrinsics="regressed"), OverfitCfg(intrinsics="softmin", regression_after=1000),
                OverfitCfg(intrinsics="ground_truth")):
        with pytest.raises(ValueError, match="softmin intrinsics without a regression stage"):
            FusedOverfitter(cfg, batch, flows, device="cpu", model=model)


def test_network_batch_engine_takes_cuda_flows_only():
    """The engine reads the caller's Flows in place: they must be CUDA float32 tensors."""
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    model, batch, flows, _ = _inputs()
    with pytest.raises(ValueError, match="CUDA tensor"):
        FusedOverfitter(OverfitCfg(intrinsics="softmin", regression_after=None), batch, flows, device="cpu",
                        model=model)
