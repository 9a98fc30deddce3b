"""Generate golden vectors of the pretraining step with ground-truth intrinsics (pretrain.py with
model/intrinsics=ground_truth, calibrated data) from the UNMODIFIED reference: a batch of B > 1 videos through the
reference's `Model` (IntrinsicsGroundTruth, Procrustes extrinsics) and `LossFlow` (weight 1000, Huber), then
backward().

Run where a checkout of the reference is available (FLOWMAP_REFERENCE names its root):

    python tests/golden/make_golden_pretrain_gt.py          # float32 run of the reference
    python tests/golden/make_golden_pretrain_gt.py --f64    # float64 run (see make_golden.py)

As in make_golden_pretrain.py, the reference's backbone is replaced by `FixedBackbone`, whose parameters ARE the
per-video depths and correspondence weights it returns, and video v's masks are scaled by MASK_RATIO ** v.  K
comes with the batch: a different one for every video and every frame, with off-centre principal points.  No
sweep runs, so nothing is injected.

Inputs are stored as float32 values (the float64 run reads the same values), outputs in the run's dtype.
"""

from __future__ import annotations

import argparse
import os
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_golden_pretrain import F32, _inputs  # noqa: E402

REF = os.environ.get("FLOWMAP_REFERENCE", "reference")
OUT = Path(__file__).resolve().parent

# name: (B, F, H, W, Procrustes points, seed)
CASES = {"pretrain_gt": (4, 4, 24, 36, 600, 53)}


def _intrinsics(b, f, seed):
    """(B, F, 3, 3) normalised K: fx, fy in [0.6, 1.6] (fx != fy), principal points up to 0.12 off centre;
    float32 values held in float64."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)  # noqa: E731
    k = torch.zeros(b, f, 3, 3, dtype=torch.float64)
    k[..., 0, 0], k[..., 1, 1] = 0.6 + r(b, f), 0.6 + r(b, f)
    k[..., 0, 2], k[..., 1, 2] = 0.5 + 0.24 * (r(b, f) - 0.5), 0.5 + 0.24 * (r(b, f) - 0.5)
    k[..., 2, 2] = 1.0
    return k.to(F32).to(torch.float64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--f64", action="store_true")
    args = ap.parse_args()

    real_f32 = torch.float32
    if args.f64:
        torch.float32 = torch.float64  # rebinding the name only; see make_golden.py
        torch.set_default_dtype(torch.float64)
    dtype = torch.float64 if args.f64 else real_f32
    suffix = "_f64" if args.f64 else ""
    sys.path.insert(0, REF)
    os.environ["PYTHONDONTWRITEBYTECODE"] = "1"
    sys.dont_write_bytecode = True
    torch.set_num_threads(8)

    from torch import nn

    from flowmap.dataset.types import Batch
    from flowmap.flow.flow_predictor import Flows
    from flowmap.loss import get_losses
    from flowmap.loss.loss_flow import LossFlowCfg
    from flowmap.loss.mapping.mapping_huber import MappingHuberCfg
    from flowmap.model.backbone.backbone import BackboneOutput
    from flowmap.model.backbone.backbone_explicit_depth import BackboneExplicitDepthCfg
    from flowmap.model.extrinsics.extrinsics_procrustes import ExtrinsicsProcrustesCfg
    from flowmap.model.intrinsics.intrinsics_ground_truth import IntrinsicsGroundTruthCfg
    from flowmap.model.model import Model, ModelCfg

    class FixedBackbone(nn.Module):
        """Returns its parameters: fixed per-video depths and correspondence weights."""

        def __init__(self, depths, weights):
            super().__init__()
            self.depths = nn.Parameter(depths.to(dtype).clone())
            self.weights = nn.Parameter(weights.to(dtype).clone())

        def forward(self, batch, flows):
            return BackboneOutput(self.depths, self.weights)

    for name, (b, f, h, w, proc_pts, seed) in CASES.items():
        inp = _inputs(b, f, h, w, seed)
        inp["intrinsics"] = _intrinsics(b, f, seed + 7)
        # the backbone's cfg only serves Model's constructor; the backbone itself is replaced below
        mcfg = ModelCfg(BackboneExplicitDepthCfg("explicit_depth", 0.1, 100.0), IntrinsicsGroundTruthCfg("ground_truth"),
                        ExtrinsicsProcrustesCfg("procrustes", proc_pts, False), True)
        model = Model(mcfg, f, (h, w))
        model.backbone = FixedBackbone(inp["depths"], inp["weights"])
        losses = get_losses([LossFlowCfg(0, 1000.0, "flow", MappingHuberCfg("huber", 0.01))])
        batch = Batch(torch.zeros((b, f, 3, h, w), dtype=dtype), torch.arange(f)[None].expand(b, f),
                      ["s"] * b, ["d"] * b, intrinsics=inp["intrinsics"].to(dtype))
        flows = Flows(*(inp[k].to(dtype) for k in ("fwd", "bwd", "fmask", "bmask")))
        out = model(batch, flows, 0)
        total = sum(loss.forward(batch, flows, None, out, 0) for loss in losses)
        total.backward()
        bb = model.backbone
        arrays = {"in_" + k: v.to(real_f32).numpy() for k, v in inp.items()}
        arrays.update(procrustes_points=np.int64(proc_pts), loss=total.detach().numpy(),
                      extrinsics=out.extrinsics.detach().numpy(), g_depths=bb.depths.grad.numpy(),
                      g_weights=bb.weights.grad.numpy())
        path = OUT / f"{name}{suffix}.npz"
        np.savez_compressed(path, **arrays)
        print(f"wrote {path.name}: {path.stat().st_size / 1e3:.0f} kB on disk")


if __name__ == "__main__":
    main()
