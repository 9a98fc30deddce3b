"""Generate golden vectors of the pretraining step (pretrain.py, model_wrapper_pretrain.py) from the
UNMODIFIED reference: a batch of B > 1 videos through the reference's `Model` (softmin intrinsics without a
regression stage, Procrustes extrinsics) and `LossFlow` (weight 1000, Huber), then backward().

Run where a checkout of the reference is available (FLOWMAP_REFERENCE names its root):

    python tests/golden/make_golden_pretrain.py          # float32 run of the reference
    python tests/golden/make_golden_pretrain.py --f64    # float64 run (see make_golden.py)

The reference's network backbone is replaced, after the Model is built, by `FixedBackbone` below: its
parameters ARE the per-video depths (B, F, H, W) and correspondence weights (B, F-1, H, W) it returns, so
their gradients are d loss / d depths and d loss / d weights.  What these files pin is the B > 1 semantics
of the step: one mask sum pooled over the whole batch (loss_flow.py:31-70), one sweep sample shared by all
videos and one softmin focal length per video (intrinsics_softmin.py:84-131).  The sweep's sample is
injected by patching torch.randperm, as make_golden.py does.

Inputs are stored as float32 values (the float64 run reads the same values), outputs in the run's dtype.
"""

from __future__ import annotations

import argparse
import os
import sys
from pathlib import Path

import numpy as np
import torch

REF = os.environ.get("FLOWMAP_REFERENCE", "reference")
OUT = Path(__file__).resolve().parent
F32 = torch.float32  # bound before the --f64 run rebinds the name
MASK_RATIO = 0.45  # video v's masks are scaled by MASK_RATIO ** v: mask sums more than 2x apart

# name: (B, F, H, W, softmin points, Procrustes points, correspondence weights, seed)
CASES = {
    "pretrain": (4, 4, 24, 36, 300, 600, True, 51),
    "pretrain_noweights": (3, 3, 16, 24, 300, None, False, 52),
}


def _inputs(b, f, h, w, seed):
    """Per-video smooth depths of different scales, weights in (0, 1), few-pixel flows and masks whose
    sums fall by MASK_RATIO from one video to the next; float32 values held in float64 tensors."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)  # noqa: E731
    rn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)  # noqa: E731
    lo = r(b * f, 1, 3, 4)
    smooth = torch.nn.functional.interpolate(lo, size=(h, w), mode="bicubic", align_corners=True)
    scale = torch.tensor([1.0, 3.0, 0.5, 10.0][:b], dtype=torch.float64) if b <= 4 else torch.ones(b)
    depth = (1.0 + smooth.reshape(b, f, h, w) + 0.02 * r(b, f, h, w)) * scale[:, None, None, None]
    weights = torch.sigmoid(rn(b, f - 1, h, w))
    fwd, bwd = 0.01 * rn(b, f - 1, h, w, 2), 0.01 * rn(b, f - 1, h, w, 2)
    ms = torch.tensor([MASK_RATIO ** v for v in range(b)], dtype=torch.float64)[:, None, None, None]
    fm, bm = r(b, f - 1, h, w) * ms, r(b, f - 1, h, w) * ms
    out = dict(depths=depth, weights=weights, fwd=fwd, bwd=bwd, fmask=fm, bmask=bm)
    return {k: v.to(F32).to(torch.float64) for k, v in out.items()}


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
    from flowmap.model.intrinsics.intrinsics_softmin import IntrinsicsSoftminCfg
    from flowmap.model.model import Model, ModelCfg

    class FixedBackbone(nn.Module):
        """Returns its parameters: fixed per-video depths and correspondence weights."""

        def __init__(self, depths, weights):
            super().__init__()
            self.depths = nn.Parameter(depths.to(dtype).clone())
            self.weights = nn.Parameter(weights.to(dtype).clone())

        def forward(self, batch, flows):
            return BackboneOutput(self.depths, self.weights)

    for name, (b, f, h, w, sweep_pts, proc_pts, use_weights, seed) in CASES.items():
        inp = _inputs(b, f, h, w, seed)
        perm = torch.randperm(h * w, generator=torch.Generator().manual_seed(seed + 1))
        # the backbone's cfg only serves Model's constructor; the backbone itself is replaced below
        mcfg = ModelCfg(BackboneExplicitDepthCfg("explicit_depth", 0.1, 100.0),
                        IntrinsicsSoftminCfg("softmin", sweep_pts, 0.5, 2.0, 60, None),
                        ExtrinsicsProcrustesCfg("procrustes", proc_pts, False), use_weights)
        model = Model(mcfg, f, (h, w))
        model.backbone = FixedBackbone(inp["depths"], inp["weights"])
        losses = get_losses([LossFlowCfg(0, 1000.0, "flow", MappingHuberCfg("huber", 0.01))])
        batch = Batch(torch.zeros((b, f, 3, h, w), dtype=dtype), torch.arange(f)[None].expand(b, f),
                      ["s"] * b, ["d"] * b)
        flows = Flows(*(inp[k].to(dtype) for k in ("fwd", "bwd", "fmask", "bmask")))
        real_randperm = torch.randperm
        torch.randperm = lambda n, **kw: perm  # inject the sweep's sample (SURVEY A.8 item 1)
        try:
            out = model(batch, flows, 0)
            total = sum(loss.forward(batch, flows, None, out, 0) for loss in losses)
            total.backward()
        finally:
            torch.randperm = real_randperm
        bb = model.backbone
        arrays = {"in_" + k: v.to(real_f32).numpy() for k, v in inp.items()}
        arrays.update(indices=perm[:sweep_pts].numpy(), use_weights=np.bool_(use_weights),
                      procrustes_points=np.int64(-1 if proc_pts is None else proc_pts),
                      loss=total.detach().numpy(), intrinsics=out.intrinsics.detach().numpy(),
                      extrinsics=out.extrinsics.detach().numpy(), g_depths=bb.depths.grad.numpy())
        if use_weights:
            arrays["g_weights"] = bb.weights.grad.numpy()
        path = OUT / f"{name}{suffix}.npz"
        np.savez_compressed(path, **arrays)
        print(f"wrote {path.name}: {path.stat().st_size / 1e3:.0f} kB on disk")


if __name__ == "__main__":
    main()
