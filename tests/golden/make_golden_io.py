"""Golden vectors for the stages either side of the hot path (flow preprocessing, export),
generated from the UNMODIFIED reference (FLOWMAP_REFERENCE names the root of its checkout):

    python tests/golden/make_golden_io.py

Imports flowmap.flow.flow_predictor.FlowPredictor (its static rescale / consistency-mask
methods and compute_bidirectional_flow), flowmap.misc.cropping.center_crop_intrinsics and
flowmap.export.colmap (write_colmap_model, the point-cloud loop of export_to_colmap restated
call for call since the function itself also copies image files).  ``plyfile`` is not
installed here; colmap.py imports it at module level, so an empty stand-in module is
registered for the import only (write_ply is not exercised).
"""
from __future__ import annotations

import os
import sys
import tempfile
import types
from pathlib import Path

import numpy as np
import torch

REF = os.environ.get("FLOWMAP_REFERENCE", "reference")
OUT = Path(__file__).resolve().parent


def main():
    sys.path.insert(0, REF)
    os.environ["PYTHONDONTWRITEBYTECODE"] = "1"
    sys.dont_write_bytecode = True
    stub = types.ModuleType("plyfile")
    stub.PlyData = stub.PlyElement = object
    sys.modules.setdefault("plyfile", stub)

    from flowmap.dataset.types import Batch
    from flowmap.flow.flow_predictor import FlowPredictor
    from flowmap.misc.cropping import center_crop_intrinsics
    from flowmap.export import colmap as ref_colmap
    from flowmap.model.projection import homogenize_points, sample_image_grid, unproject
    from einops import einsum, rearrange

    class DiffPredictor(FlowPredictor):
        """A deterministic stand-in for RAFT: the flow is a fixed function of the two frames, so
        that reversing the video changes it the way a real predictor's output would change."""

        def forward(self, videos):
            d = videos[:, 1:, :2] - videos[:, :-1, :2] + 0.25 * videos[:, 1:, 2:3]
            return 0.08 * rearrange(d, "b f xy h w -> b f h w xy")

    g = torch.Generator().manual_seed(7)
    out = {}
    # -- consistency masks and rescaling ------------------------------------------------
    b, f, h, w = 2, 4, 20, 28
    lo = torch.rand(b * f, 3, 5, 7, generator=g)
    videos = torch.nn.functional.interpolate(lo, (h, w), mode="bicubic", align_corners=True).clamp(0, 1)
    videos = videos.reshape(b, f, 3, h, w)
    flow = 0.06 * torch.randn(b, f - 1, h, w, 2, generator=g)   # some samples leave the frame
    out["videos"], out["flow"] = videos, flow
    out["mask"] = FlowPredictor.compute_consistency_mask(videos, flow)
    for name, shape in (("down", (15, 18)), ("up", (33, 40)), ("same", (h, w)), ("odd", (7, 61))):
        out[f"flow_{name}"] = FlowPredictor.rescale_flow(flow, shape)
        out[f"mask_{name}"] = FlowPredictor.rescale_mask(out["mask"], shape)
    pred = DiffPredictor(None)
    batch = Batch(videos, torch.arange(f)[None].expand(b, f), ["s"] * b, ["d"] * b)
    flows = pred.compute_bidirectional_flow(batch, (16, 24))
    out["bi_forward"], out["bi_backward"] = flows.forward, flows.backward
    out["bi_forward_mask"], out["bi_backward_mask"] = flows.forward_mask, flows.backward_mask
    np.savez_compressed(OUT / "io_flow.npz", **{k: v.numpy() for k, v in out.items()})

    # -- export -------------------------------------------------------------------------
    from scipy.spatial.transform import Rotation
    f, h, w = 5, 12, 16
    rot = Rotation.from_rotvec(0.3 * torch.randn(f, 3, generator=g).numpy()).as_matrix()
    ext = torch.eye(4).repeat(f, 1, 1)
    ext[:, :3, :3] = torch.tensor(rot, dtype=torch.float32)
    ext[:, :3, 3] = torch.randn(f, 3, generator=g)
    k = torch.eye(3).repeat(f, 1, 1)
    k[:, 0, 0] = 0.9 + 0.1 * torch.rand(f, generator=g)
    k[:, 1, 1] = 1.2 + 0.1 * torch.rand(f, generator=g)
    k[:, :2, 2] = 0.5
    depths = 1 + torch.rand(f, h, w, generator=g)
    names = [f"frame_{i:03d}.png" for i in range(f)]
    cropped = center_crop_intrinsics(k[None], (h, w), (h + 4, w + 6))[0]
    with tempfile.TemporaryDirectory() as tmp:
        ref_colmap.write_colmap_model(Path(tmp), ext, cropped, names, (48, 64))
        cams = np.frombuffer((Path(tmp) / "cameras.bin").read_bytes(), dtype=np.uint8)
        imgs = np.frombuffer((Path(tmp) / "images.bin").read_bytes(), dtype=np.uint8)
        # the reference reader wants all three files; the writer is called with points3D=None
        (Path(tmp) / "points3D.bin").write_bytes((0).to_bytes(8, "little"))
        back_ext, back_k, back_names = ref_colmap.read_colmap_model(Path(tmp))
    # export_to_colmap's point-cloud loop (export/colmap.py:84-101)
    xy, _ = sample_image_grid((h, w), ext.device)
    points = []
    for e, kk, d in zip(ext, k, depths):
        xyz = homogenize_points(unproject(xy, d, kk))
        xyz = einsum(e, xyz, "i j, ... j -> ... i")[..., :3]
        points.append(rearrange(xyz, "h w xyz -> (h w) xyz").numpy())
    # checkpoint layout: parameter / buffer names and shapes of the reference Model (the Lightning
    # wrapper prefixes them with "model.", model_wrapper_overfit.py:40-49)
    from flowmap.model.backbone.backbone_explicit_depth import BackboneExplicitDepthCfg
    from flowmap.model.extrinsics.extrinsics_procrustes import ExtrinsicsProcrustesCfg
    from flowmap.model.intrinsics.intrinsics_regressed import IntrinsicsRegressedCfg
    from flowmap.model.intrinsics.intrinsics_softmin import IntrinsicsSoftminCfg, RegressionCfg
    from flowmap.model.model import Model, ModelCfg
    state = {}
    for tag, icfg in (("regressed", IntrinsicsRegressedCfg("regressed", 0.85)),
                      ("softmin", IntrinsicsSoftminCfg("softmin", 64, 0.5, 2.0, 60, RegressionCfg(1000, 100)))):
        model = Model(ModelCfg(BackboneExplicitDepthCfg("explicit_depth", 0.1, 100.0), icfg,
                               ExtrinsicsProcrustesCfg("procrustes", None, False), True), 5, (12, 16))
        sd = model.state_dict()
        state[f"state_{tag}_names"] = np.array(list(sd.keys()))
        state[f"state_{tag}_shapes"] = np.array([",".join(map(str, v.shape)) for v in sd.values()])
    np.savez_compressed(OUT / "io_export.npz", **state, extrinsics=ext.numpy(), intrinsics=k.numpy(),
                        depths=depths.numpy(), cropped=cropped.numpy(), cameras_bin=cams, images_bin=imgs,
                        points=np.concatenate(points), read_extrinsics=back_ext.numpy(),
                        read_intrinsics=back_k.numpy(), names=np.array(names), read_names=np.array(back_names))
    print("wrote io_flow.npz, io_export.npz")


if __name__ == "__main__":
    main()
