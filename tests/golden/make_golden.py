"""Generate golden input/output vectors from the UNMODIFIED reference.

Run where a checkout of the reference is available (FLOWMAP_REFERENCE names its root):

    python tests/golden/make_golden.py            # float32 run of the reference
    python tests/golden/make_golden.py --f64      # float64 run of the same modules
    python tests/golden/make_golden.py --only gt_intrinsics [--f64]   # write one case only

The reference ships no tests or golden vectors for this path (SURVEY.md section 4), so
these files are the pin for ``oracle/flowmap_oracle.py`` and, through it, for the CUDA
kernels.  The reference modules are imported from that checkout as they lie (nothing
is copied); only the Lightning shell is restated here (model_wrapper_overfit.py:51-73,
104-105) because lightning/hydra are not installed.

float64 run: the reference hard-codes torch.float32 in a dozen places (SURVEY A.8 item
13).  Rather than editing a copy, this script rebinds the *name* ``torch.float32`` to
``torch.float64`` in this process before importing the reference and sets the default
dtype to float64; every ``dtype=torch.float32`` in the reference then evaluates to
float64.  Outputs of that run are stored with the suffix ``_f64`` and are the arbiter
for gradient comparisons.
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


def _inputs(seed, f, h, w, sigma=0.01, smooth_depth=True):
    """Seeded float64 master copies of the inputs (cast per run)."""
    g = torch.Generator().manual_seed(seed)
    if smooth_depth:
        lo = torch.rand(f, 1, 3, 4, generator=g, dtype=torch.float64)
        depth = 1.0 + torch.nn.functional.interpolate(lo, size=(h, w), mode="bicubic",
                                                      align_corners=True)[:, 0]
        depth = depth + 0.02 * torch.rand(f, h, w, generator=g, dtype=torch.float64)
    else:
        depth = 0.1 + 0.05 * torch.rand(f, h, w, generator=g, dtype=torch.float64)
    wparam = 0.01 * torch.randn(f - 1, h, w, generator=g, dtype=torch.float64)
    fwd = sigma * torch.randn(1, f - 1, h, w, 2, generator=g, dtype=torch.float64)
    bwd = sigma * torch.randn(1, f - 1, h, w, 2, generator=g, dtype=torch.float64)
    fm = torch.rand(1, f - 1, h, w, generator=g, dtype=torch.float64)
    bm = torch.rand(1, f - 1, h, w, generator=g, dtype=torch.float64)
    return dict(depth=depth, wparam=wparam, fwd=fwd, bwd=bwd, fmask=fm, bmask=bm)


def _tracks(seed, segments, n_points, dtype):
    """segments: list of (start, length).  xy slightly outside [0,1) on purpose."""
    from flowmap.tracking.track_predictor import Tracks
    g = torch.Generator().manual_seed(seed)
    out, raw = [], []
    for s, n_f in segments:
        xy = (torch.rand(1, n_f, n_points, 2, generator=g, dtype=torch.float64) * 1.2 - 0.1)
        vis = torch.rand(1, n_f, n_points, generator=g) < 0.7
        out.append(Tracks(xy.to(dtype), vis, s))
        raw.append((xy, vis, s))
    return out, raw


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--f64", action="store_true")
    ap.add_argument("--only", help="write only this case (every case is still computed)")
    args = ap.parse_args()

    real_f32 = torch.float32
    if args.f64:
        torch.float32 = torch.float64  # rebinding the name only; see module docstring
        torch.set_default_dtype(torch.float64)
    dtype = torch.float64 if args.f64 else real_f32
    suffix = "_f64" if args.f64 else ""
    sys.path.insert(0, REF)
    os.environ["PYTHONDONTWRITEBYTECODE"] = "1"
    sys.dont_write_bytecode = True
    torch.set_num_threads(8)

    from flowmap.dataset.types import Batch
    from flowmap.flow.flow_predictor import Flows
    from flowmap.loss import get_losses
    from flowmap.loss.loss_flow import LossFlowCfg
    from flowmap.loss.loss_tracking import LossTrackingCfg
    from flowmap.loss.mapping import get_mapping
    from flowmap.loss.mapping.mapping import fix_aspect_ratio
    from flowmap.loss.mapping.mapping_huber import MappingHuberCfg
    from flowmap.loss.mapping.mapping_l1 import MappingL1Cfg
    from flowmap.loss.mapping.mapping_l2 import MappingL2Cfg
    from flowmap.model.backbone.backbone_explicit_depth import BackboneExplicitDepthCfg
    from flowmap.model.extrinsics.extrinsics_procrustes import ExtrinsicsProcrustesCfg
    from flowmap.model.intrinsics.common import focal_lengths_to_intrinsics
    from flowmap.model.intrinsics.intrinsics_ground_truth import IntrinsicsGroundTruthCfg
    from flowmap.model.intrinsics.intrinsics_regressed import IntrinsicsRegressedCfg
    from flowmap.model.intrinsics.intrinsics_softmin import (IntrinsicsSoftminCfg,
                                                             RegressionCfg)
    from flowmap.model.model import Model, ModelCfg
    from flowmap.model import projection as P
    from flowmap.model.procrustes import align_rigid

    def npy(t):
        return t.detach().cpu().numpy()

    def mapping_cfg(name, delta=0.01):
        return {"huber": MappingHuberCfg("huber", delta), "l1": MappingL1Cfg("l1"),
                "l2": MappingL2Cfg("l2")}[name]

    def build(f, h, w, inp, intr="regressed", focal=0.85, npts=None, mapping="huber",
              tracking=False, softmin_pts=300, regression=None, k=None):
        if intr == "regressed":
            icfg = IntrinsicsRegressedCfg("regressed", focal)
        elif intr == "ground_truth":  # K is the batch's (intrinsics_ground_truth.py)
            icfg = IntrinsicsGroundTruthCfg("ground_truth")
        else:
            icfg = IntrinsicsSoftminCfg("softmin", softmin_pts, 0.5, 2.0, 60, regression)
        mcfg = ModelCfg(BackboneExplicitDepthCfg("explicit_depth", 0.1, 100.0), icfg,
                        ExtrinsicsProcrustesCfg("procrustes", npts, False), True)
        model = Model(mcfg, f, (h, w))
        with torch.no_grad():
            model.backbone.depth.copy_(inp["depth"].to(dtype))
            model.backbone.weights.copy_(inp["wparam"].to(dtype))
        lcfgs = [LossFlowCfg(0, 1000.0, "flow", mapping_cfg(mapping))]
        if tracking:
            lcfgs.append(LossTrackingCfg(0, 100.0, "tracking", mapping_cfg(mapping)))
        losses = get_losses(lcfgs)
        batch = Batch(torch.zeros((1, f, 3, h, w), dtype=dtype),
                      torch.arange(f)[None], ["s"], ["d"],
                      intrinsics=None if k is None else k.to(dtype))
        flows = Flows(inp["fwd"].to(dtype), inp["bwd"].to(dtype), inp["fmask"].to(dtype),
                      inp["bmask"].to(dtype))
        return model, losses, batch, flows

    def step(model, losses, batch, flows, tracks, global_step):
        """model_wrapper_overfit.py:51-73 without the logging."""
        out = model(batch, flows, global_step)
        parts = [l.forward(batch, flows, tracks, out, global_step) for l in losses]
        return out, parts, sum(parts)

    def grads_of(model):
        d = {"g_depth": model.backbone.depth.grad, "g_wparam": model.backbone.weights.grad}
        intr = model.intrinsics
        fl = getattr(intr, "focal_length", None)
        if fl is None and hasattr(intr, "intrinsics_regressed"):
            fl = intr.intrinsics_regressed.focal_length
        if fl is not None and fl.grad is not None:
            d["g_focal"] = fl.grad
        return {k: npy(v) for k, v in d.items() if v is not None}

    def save(name, **arrays):
        if args.only and name != args.only:
            return
        path = OUT / f"{name}{suffix}.npz"
        arrays = {k: (np.asarray(v) if not isinstance(v, torch.Tensor) else npy(v))
                  for k, v in arrays.items()}
        np.savez_compressed(path, **arrays)
        print(f"wrote {path.name}: {sum(a.nbytes for a in arrays.values()) / 1e3:.0f} kB")

    def input_arrays(inp):
        return {"in_" + k: v.to(torch.float64).numpy() for k, v in inp.items()}

    # ------------------------------------------------------------------ unit vectors
    g = torch.Generator().manual_seed(7)
    rnd = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64).to(dtype)  # noqa
    rndn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64).to(dtype)  # noqa
    h, w = 6, 10
    xy, ij = P.sample_image_grid((h, w))
    foc = torch.tensor([0.5, 0.85, 2.0], dtype=dtype)
    k3 = focal_lengths_to_intrinsics(foc, (h, w))
    z = 0.5 + rnd(3, h, w)
    surf = P.unproject(xy, z, k3[:, None, None])
    pts = rndn(4, 50, 3)
    pts[0, 0, 2] = -1e-5  # exercises the nan_to_num branch (SURVEY A.2)
    pts[0, 1] = torch.tensor([0.0, 0.0, -1e-5], dtype=dtype)
    kk = focal_lengths_to_intrinsics(torch.tensor(0.9, dtype=dtype), (h, w))
    proj = P.project_camera_space(pts, kk)
    pa, qa, wa = rndn(3, 40, 3), rndn(3, 40, 3), rnd(3, 40)
    # One well-posed case (q is a rigid motion of p) and two generic ones.
    ang = torch.tensor([0.3, -0.2, 0.5], dtype=torch.float64)
    sk = torch.tensor([[0, -ang[2], ang[1]], [ang[2], 0, -ang[0]], [-ang[1], ang[0], 0]],
                      dtype=torch.float64)
    r0 = torch.linalg.matrix_exp(sk).to(dtype)
    qa[0] = pa[0] @ r0.T + torch.tensor([0.1, -0.3, 0.2], dtype=dtype)
    qa[2] = -qa[2]  # tends to produce the reflection (det < 0) branch
    rig = align_rigid(pa, qa, wa)
    rel = rig[None]
    chain = P.get_extrinsics(rel)
    a2, b2 = rndn(5, 7, 2) * 0.02, rndn(5, 7, 2) * 0.02
    a2[0, 0] = b2[0, 0]  # zero residual: norm subgradient
    maps = {}
    for mname in ("huber", "l1", "l2"):
        maps[f"map_{mname}"] = get_mapping(mapping_cfg(mname)).forward(a2, b2, (h, w))
    samp_img = rndn(2, 3, 5, 7)
    samp_xy = rnd(2, 11, 2) * 1.4 - 0.2
    samp = torch.nn.functional.grid_sample(samp_img, (samp_xy * 2 - 1)[:, :, None],
                                           mode="bilinear", padding_mode="border",
                                           align_corners=False)[..., 0].transpose(1, 2)
    save("units", grid_xy=xy, grid_ij=ij, focals=foc, k3=k3, z=z, surfaces=surf,
         proj_pts=pts, proj_k=kk, proj_xy=proj, rigid_p=pa, rigid_q=qa, rigid_w=wa,
         rigid_t=rig, chain=chain, map_a=a2, map_b=b2, aspect=fix_aspect_ratio(a2, (h, w)),
         samp_img=samp_img, samp_xy=samp_xy, samp_out=samp, **maps)

    # ------------------------------------------------------------------ flow loss cases
    def run_flow_case(name, f, h, w, seed, **kw):
        inp = _inputs(seed, f, h, w, smooth_depth=kw.pop("smooth", True))
        model, losses, batch, flows = build(f, h, w, inp, **kw)
        out, parts, total = step(model, losses, batch, flows, None, 0)
        total.backward()
        fwd_xy = P.compute_forward_flow(out.surfaces, out.extrinsics, out.intrinsics)
        bwd_xy = P.compute_backward_flow(out.surfaces, out.extrinsics, out.intrinsics)
        save(name, **input_arrays(inp), focal=np.float64(kw.get("focal", 0.85)),
             loss=total, extrinsics=out.extrinsics, intrinsics=out.intrinsics,
             weights=out.backward_correspondence_weights,
             fwd_xy=fwd_xy[:, :2], bwd_xy=bwd_xy[:, :2], **grads_of(model))

    run_flow_case("flow_huber", 5, 24, 32, seed=1)
    run_flow_case("flow_l1", 4, 16, 24, seed=2, mapping="l1")
    run_flow_case("flow_l2", 4, 16, 24, seed=3, mapping="l2")
    run_flow_case("flow_pts1000", 4, 36, 48, seed=4, npts=1000)
    run_flow_case("flow_rough", 6, 20, 28, seed=5, smooth=False, focal=1.3)

    # ------------------------------------------------------------------ softmin intrinsics
    f, h, w = 4, 24, 40
    inp = _inputs(11, f, h, w)
    perm = torch.randperm(h * w, generator=torch.Generator().manual_seed(3))
    real_randperm = torch.randperm
    torch.randperm = lambda n, **kw: perm  # inject the indices (SURVEY A.8 item 1)
    try:
        model, losses, batch, flows = build(f, h, w, inp, intr="softmin", softmin_pts=300)
        out, parts, total = step(model, losses, batch, flows, None, 0)
        total.backward()
    finally:
        torch.randperm = real_randperm
    save("softmin", **input_arrays(inp), indices=perm[:300].numpy(), loss=total,
         extrinsics=out.extrinsics, intrinsics=out.intrinsics, **grads_of(model))

    # ------------------------------------------------------------------ tracking loss
    f, h, w = 9, 20, 28
    inp = _inputs(21, f, h, w)
    model, losses, batch, flows = build(f, h, w, inp, tracking=True)
    tracks, raw = _tracks(5, [(0, 6), (3, 6)], 50, dtype)
    out, parts, total = step(model, losses, batch, flows, tracks, 0)
    total.backward()
    tr = {}
    for i, (txy, tvis, s) in enumerate(raw):
        tr[f"trk{i}_xy"], tr[f"trk{i}_vis"], tr[f"trk{i}_start"] = txy.numpy(), tvis.numpy(), s
    tgt0, vis0 = P.compute_track_flow(out.surfaces[:, :6], out.extrinsics[:, :6],
                                      out.intrinsics[:, :6], tracks[0])
    save("tracking", **input_arrays(inp), **tr, loss=total, loss_flow=parts[0],
         loss_tracking=parts[1], extrinsics=out.extrinsics, trk0_target=tgt0,
         trk0_valid=vis0, **grads_of(model))

    # ------------------------------------------------------------------ Adam trajectories
    def run_traj(name, f, h, w, seed, steps, from_init, intr="regressed"):
        inp = _inputs(seed, f, h, w)
        if from_init:  # the true start of an overfit run: planar depth 0.1, weight 0
            inp["depth"] = torch.full((f, h, w), 0.1, dtype=torch.float64)
            inp["wparam"] = torch.zeros(f - 1, h, w, dtype=torch.float64)
        model, losses, batch, flows = build(f, h, w, inp, intr=intr)
        opt = torch.optim.Adam(model.parameters(), lr=3e-5)  # model_wrapper_overfit.py:104
        rec = {"loss": [], "extrinsics": [], "focal": []}
        for s in range(steps):
            opt.zero_grad()
            out, parts, total = step(model, losses, batch, flows, None, s)
            total.backward()
            opt.step()
            rec["loss"].append(float(total))
            rec["extrinsics"].append(npy(out.extrinsics))
            rec["focal"].append(npy(out.intrinsics[0, 0, 0, 0]))
        save(name, **input_arrays(inp), loss=np.array(rec["loss"]),
             extrinsics=np.stack(rec["extrinsics"]), fx=np.stack(rec["focal"]),
             depth_final=model.backbone.depth, wparam_final=model.backbone.weights)

    run_traj("traj_generic", 5, 16, 24, seed=31, steps=6, from_init=False)
    run_traj("traj_init", 4, 16, 24, seed=32, steps=6, from_init=True)

    # ------------------------------------------------------------------ ground-truth intrinsics
    # model/intrinsics: ground_truth on calibrated data: a K per frame, off-centre and anisotropic.
    # fx grows 1.5x and fy 1.4x over the video (fx != fy H / W), the principal point drifts from
    # (0.3, 0.7) to (0.7, 0.3).  Flow + tracking (overlapping segments, tracks leaving the frame).
    f, h, w = 6, 20, 28
    inp = _inputs(41, f, h, w)
    s_ = (h * w) ** 0.5
    t_ = torch.linspace(0.0, 1.0, f, dtype=torch.float64)
    kgt = torch.zeros(1, f, 3, 3, dtype=torch.float64)
    kgt[0, :, 0, 0] = 0.8 * s_ / w * (1 + 0.5 * t_)
    kgt[0, :, 1, 1] = 0.95 * s_ / h * (1 + 0.4 * t_)
    kgt[0, :, 0, 2] = 0.3 + 0.4 * t_
    kgt[0, :, 1, 2] = 0.7 - 0.4 * t_
    kgt[0, :, 2, 2] = 1.0
    model, losses, batch, flows = build(f, h, w, inp, intr="ground_truth", tracking=True, k=kgt)
    tracks, raw = _tracks(42, [(0, 4), (2, 4)], 60, dtype)
    out, parts, total = step(model, losses, batch, flows, tracks, 0)
    total.backward()
    tr = {}
    for i, (txy, tvis, s) in enumerate(raw):
        tr[f"trk{i}_xy"], tr[f"trk{i}_vis"], tr[f"trk{i}_start"] = txy.numpy(), tvis.numpy(), s
    fwd_xy = P.compute_forward_flow(out.surfaces, out.extrinsics, out.intrinsics)
    bwd_xy = P.compute_backward_flow(out.surfaces, out.extrinsics, out.intrinsics)
    tgt1, vis1 = P.compute_track_flow(out.surfaces[:, 2:6], out.extrinsics[:, 2:6],
                                      out.intrinsics[:, 2:6], tracks[1])
    # projection unit under the same K: unproject, project (world points, incl. the nan_to_num
    # branch at z = -1e-5 in camera space) and reproject_points
    g = torch.Generator().manual_seed(43)
    kd = kgt.to(dtype)
    z = (0.5 + torch.rand(1, f, h, w, generator=g, dtype=torch.float64)).to(dtype)
    xy, _ = P.sample_image_grid((h, w))
    u_surf = P.unproject(xy.to(dtype), z, kd[:, :, None, None])
    cam = torch.randn(1, f, 40, 3, generator=g, dtype=torch.float64).to(dtype)
    cam[..., 2] = cam[..., 2].abs() + 0.3
    cam[0, :, :5, 2] = -cam[0, :, :5, 2]  # behind the camera
    cam[0, 0, 5, 2] = -1e-5
    cam[0, 1, 6] = torch.tensor([0.0, 0.0, -1e-5], dtype=dtype)
    eye = torch.eye(4, dtype=dtype).expand(1, f, 4, 4)
    p_xy, p_front = P.project(cam, eye[:, :, None], kd[:, :, None])
    rel_t = out.extrinsics.detach()
    r_xy = P.reproject_points(cam, rel_t[:, :, None], kd[:, :, None])
    save("gt_intrinsics", **input_arrays(inp), **tr, intrinsics=kgt, loss=total, loss_flow=parts[0],
         loss_tracking=parts[1], extrinsics=out.extrinsics, fwd_xy=fwd_xy[:, :2], bwd_xy=bwd_xy[:, :2],
         trk1_target=tgt1, trk1_valid=vis1, unit_z=z, unit_surfaces=u_surf, unit_cam=cam, unit_proj_xy=p_xy,
         unit_proj_front=p_front, unit_rel=rel_t, unit_reproj_xy=r_xy, **grads_of(model))


if __name__ == "__main__":
    main()
