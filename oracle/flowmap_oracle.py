"""CPU oracle for FlowMap's per-iteration optimisation hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``flowmap_b200/`` may import this file; only
``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference``
legs of ``bench.py`` do, and there only as the checker / the timed CPU baseline.

What it is: a plain-PyTorch (CPU, autograd) restatement of the algorithm the reference
runs every optimisation step (SURVEY.md section 8(a), rows a1-a17).  The reference is pure
Python on top of ATen, so the restatement is Python on top of ATen as well; it is
dtype-generic (the reference hard-codes float32, SURVEY A.8 item 13) so the same code
also serves as the float64 arbiter.  All citations are relative to the reference checkout.

Parity status: PINNED.  The reference ships no tests or golden vectors for this path
(SURVEY section 4), so the pin is against outputs of the reference itself: the script
``tests/golden/make_golden.py`` imports the unmodified reference modules in the build
container, runs them on seeded inputs and stores inputs+outputs under
``tests/golden/*.npz``; ``tests/test_oracle_golden.py`` checks every function here
against those files (float32 outputs of the reference and of a float64 run of it).

Third-party arithmetic: the numerics live in torch (reference pin torch==2.2.1,
requirements_exact.txt:75; this image has 2.11.0).  The call sites restated here are
linalg.svd (procrustes.py:35), det (:38), inverse (projection.py:46,86,154,176,288),
grid_sample (projection.py:235,266), nan_to_num (:56), huber_loss (mapping_huber.py:25),
softmin (intrinsics_softmin.py:129) and optim.Adam (model_wrapper_overfit.py:105).
"""

from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional, Sequence

import torch
import torch.nn.functional as F
from torch import Tensor

# --------------------------------------------------------------------------------------
# a1 / a2 / a3: pixel grid, intrinsics from a focal length, unprojection
# --------------------------------------------------------------------------------------


def pixel_grid(h: int, w: int, dtype=torch.float32, device="cpu") -> Tensor:
    """Pixel-centre coordinates, (h, w, 2) with last axis (x, y), both in (0, 1).

    flowmap/model/projection.py:93-113 (sample_image_grid): x = (col + .5) / w,
    y = (row + .5) / h.
    """
    ys = (torch.arange(h, dtype=dtype, device=device) + 0.5) / h
    xs = (torch.arange(w, dtype=dtype, device=device) + 0.5) / w
    return torch.stack((xs[None, :].expand(h, w), ys[:, None].expand(h, w)), dim=-1)


def intrinsics_from_focal(focal: Tensor, h: int, w: int) -> Tensor:
    """(...,) focal lengths -> (..., 3, 3) normalised intrinsics.

    flowmap/model/intrinsics/common.py:6-20: fx = f*sqrt(hw)/w, fy = f*sqrt(hw)/h,
    principal point at (.5, .5).
    """
    scaled = focal * (h * w) ** 0.5
    k = torch.zeros((*focal.shape, 3, 3), dtype=focal.dtype, device=focal.device)
    k[..., 0, 2] = 0.5
    k[..., 1, 2] = 0.5
    k[..., 2, 2] = 1.0
    fx = scaled / w
    fy = scaled / h
    # Assemble without in-place writes on a leaf-dependent tensor so autograd is clean.
    e00 = torch.zeros_like(k)
    e00[..., 0, 0] = 1.0
    e11 = torch.zeros_like(k)
    e11[..., 1, 1] = 1.0
    return k + fx[..., None, None] * e00 + fy[..., None, None] * e11


def to_homogeneous(v: Tensor, last: float = 1.0) -> Tensor:
    """projection.py:11-23 (homogenize_points / homogenize_vectors)."""
    pad = torch.full_like(v[..., :1], last)
    return torch.cat((v, pad), dim=-1)


def matvec(m: Tensor, v: Tensor) -> Tensor:
    """Broadcasting matrix-vector product ('... i j, ... j -> ... i'), projection.py:30."""
    return (m * v[..., None, :]).sum(dim=-1)


def unproject(xy: Tensor, z: Tensor, k: Tensor) -> Tensor:
    """projection.py:76-90: S = z * K^-1 [x, y, 1]^T (K inverted numerically)."""
    rays = matvec(torch.linalg.inv(k), to_homogeneous(xy))
    return rays * z[..., None]


# --------------------------------------------------------------------------------------
# a4: explicit-depth backbone
# --------------------------------------------------------------------------------------


def explicit_backbone(depth_param: Tensor, weight_param: Tensor, sensitivity: float):
    """backbone_explicit_depth.py:34-41: depths = depth[None]; weights = sigmoid(s*w)[None]."""
    return depth_param[None], torch.sigmoid(sensitivity * weight_param)[None]


# --------------------------------------------------------------------------------------
# a5: Procrustes point selection
# --------------------------------------------------------------------------------------


def procrustes_indices(h: int, w: int, num_points: Optional[int], randomize: bool,
                       device="cpu", generator: Optional[torch.Generator] = None) -> Tensor:
    """extrinsics_procrustes.py:33-51: all pixels / randint / linspace cast to int64."""
    n = h * w
    if num_points is None:
        return torch.arange(n, dtype=torch.int64, device=device)
    if randomize:
        return torch.randint(0, n, (num_points,), dtype=torch.int64, device=device,
                             generator=generator)
    return torch.linspace(0, n - 1, num_points, dtype=torch.int64, device=device)


# --------------------------------------------------------------------------------------
# a6 / a7 / a8: bilinear gather, weighted Procrustes, pose chain
# --------------------------------------------------------------------------------------


def bilinear_border(image: Tensor, xy: Tensor) -> Tensor:
    """Sample (n, c, h, w) at normalised (n, p, 2) -> (n, p, c).

    Same operator the reference uses (grid_sample, bilinear, border padding,
    align_corners=False; projection.py:235-241 and :266-272).
    """
    grid = (xy * 2 - 1)[:, :, None, :]
    out = F.grid_sample(image, grid, mode="bilinear", padding_mode="border",
                        align_corners=False)
    return out[..., 0].transpose(1, 2)


def bilinear_border_explicit(image: Tensor, xy: Tensor) -> Tensor:
    """Spelled-out twin of :func:`bilinear_border` (SURVEY A.3) used to pin the exact
    sampling rule the CUDA kernels implement: pixel coords px = x*w - .5 clamped to
    [0, w-1]; the four neighbours floor/floor+1 with out-of-range taps dropped."""
    n, c, h, w = image.shape
    px = (xy[..., 0] * w - 0.5).clamp(0, w - 1)
    py = (xy[..., 1] * h - 0.5).clamp(0, h - 1)
    x0 = px.floor()
    y0 = py.floor()
    tx = px - x0
    ty = py - y0
    x0 = x0.long()
    y0 = y0.long()
    flat = image.reshape(n, c, h * w)
    out = 0
    for dy, wy in ((0, 1 - ty), (1, ty)):
        for dx, wx in ((0, 1 - tx), (1, tx)):
            xi = x0 + dx
            yi = y0 + dy
            ok = ((xi <= w - 1) & (yi <= h - 1)).to(image.dtype)
            idx = (yi.clamp(max=h - 1) * w + xi.clamp(max=w - 1))[:, None, :].expand(n, c, -1)
            out = out + flat.gather(2, idx) * (wx * wy * ok)[:, None, :]
    return out.transpose(1, 2)


def align_rigid(p: Tensor, q: Tensor, weights: Tensor) -> Tensor:
    """Weighted rigid fit p -> q, (..., n, 3) x2 + (..., n) -> (..., 4, 4).

    procrustes.py:7-51.  Centroids use weights normalised by (sum + 1e-8) (:23-25); the
    covariance uses the raw weights (:32); R = U diag(1, 1, sign(det U det Vt)) Vt
    (:35-39); t = q_bar - R p_bar (:42); result = [R t; 0 1] (:45-51).
    """
    wn = weights / (weights.sum(dim=-1, keepdim=True) + 1e-8)
    pc = (wn[..., None] * p).sum(dim=-2)
    qc = (wn[..., None] * q).sum(dim=-2)
    pz = p - pc[..., None, :]
    qz = q - qc[..., None, :]
    cov = (qz * weights[..., None]).transpose(-1, -2) @ pz
    u, _, vt = torch.linalg.svd(cov)
    flip = (torch.linalg.det(u) * torch.linalg.det(vt)).sign()
    diag = torch.ones_like(cov[..., 0])
    diag = torch.cat((diag[..., :2], flip[..., None]), dim=-1)
    rot = u @ (diag[..., :, None] * vt)
    trans = qc - matvec(rot, pc)
    top = torch.cat((rot, trans[..., None]), dim=-1)
    bottom = torch.zeros_like(top[..., :1, :])
    bottom[..., 0, 3] = 1
    return torch.cat((top, bottom), dim=-2)


def pose_chain(rel: Tensor) -> Tensor:
    """projection.py:187-210 (get_extrinsics): P_0 = I, P_{k+1} = P_k @ rel_k."""
    eye = torch.eye(4, dtype=rel.dtype, device=rel.device).expand(*rel.shape[:-3], 4, 4)
    poses = [eye.contiguous()]
    for k in range(rel.shape[-3]):
        poses.append(poses[-1] @ rel[..., k, :, :])
    return torch.stack(poses, dim=-3)


def relative_poses(surfaces: Tensor, backward_flows: Tensor, weights: Tensor,
                   indices: Tensor) -> Tensor:
    """Per-pair Procrustes transforms (b, f-1, 4, 4); the body of align_surfaces
    (projection.py:213-249) up to, not including, the chain."""
    b, f, h, w, _ = surfaces.shape
    xy = pixel_grid(h, w, surfaces.dtype, surfaces.device)
    later_pts = surfaces[:, 1:].reshape(b, f - 1, h * w, 3)[:, :, indices]
    flowed = (xy + backward_flows).reshape(b, f - 1, h * w, 2)[:, :, indices]
    earlier_img = surfaces[:, :-1].reshape(b * (f - 1), h, w, 3).permute(0, 3, 1, 2)
    earlier_pts = bilinear_border(earlier_img, flowed.reshape(b * (f - 1), -1, 2))
    earlier_pts = earlier_pts.reshape(b, f - 1, -1, 3)
    wts = weights.reshape(b, f - 1, h * w)[..., indices]
    return align_rigid(later_pts, earlier_pts, wts)


def align_surfaces(surfaces: Tensor, backward_flows: Tensor, weights: Tensor,
                   indices: Tensor) -> Tensor:
    """projection.py:213-252: camera-to-world extrinsics (b, f, 4, 4)."""
    return pose_chain(relative_poses(surfaces, backward_flows, weights, indices))


# --------------------------------------------------------------------------------------
# a12 / a13: projection and pose-induced flow
# --------------------------------------------------------------------------------------


def project_camera_space(points: Tensor, k: Tensor, epsilon: float = 1e-5,
                         infinity: float = 1e8) -> Tensor:
    """projection.py:49-58: divide all components by (z + eps), nan_to_num, apply K, keep xy."""
    points = points / (points[..., -1:] + epsilon)
    points = points.nan_to_num(posinf=infinity, neginf=-infinity)
    return matvec(k, points)[..., :-1]


def reproject(xyz: Tensor, transform: Tensor, k: Tensor) -> Tensor:
    """projection.py:116-134 (reproject_points)."""
    moved = matvec(transform, to_homogeneous(xyz))[..., :3]
    return project_camera_space(moved, k)


def _expand_over_grid(m: Tensor, ndim_points: int) -> Tensor:
    # (b, f, i, j) -> (b, f, 1..., i, j) so that it broadcasts over the point axes.
    extra = ndim_points - 3
    return m.reshape(*m.shape[:2], *([1] * extra), *m.shape[2:])


def forward_flow_positions(surfaces: Tensor, extrinsics: Tensor, k: Tensor) -> Tensor:
    """projection.py:143-162: points of frame i moved by inv(P_{i+1}) P_i, projected with K_{i+1}."""
    t = torch.linalg.inv(extrinsics[:, 1:]) @ extrinsics[:, :-1]
    return reproject(surfaces[:, :-1], _expand_over_grid(t, surfaces.ndim),
                     _expand_over_grid(k[:, 1:], surfaces.ndim))


def backward_flow_positions(surfaces: Tensor, extrinsics: Tensor, k: Tensor) -> Tensor:
    """projection.py:165-184: points of frame i+1 moved by inv(P_i) P_{i+1}, projected with K_i."""
    t = torch.linalg.inv(extrinsics[:, :-1]) @ extrinsics[:, 1:]
    return reproject(surfaces[:, 1:], _expand_over_grid(t, surfaces.ndim),
                     _expand_over_grid(k[:, :-1], surfaces.ndim))


# --------------------------------------------------------------------------------------
# a14: robust mappings
# --------------------------------------------------------------------------------------


def aspect_correct(v: Tensor, h: int, w: int) -> Tensor:
    """mapping.py:9-24 (fix_aspect_ratio): scale (x, y) by (w, h) / sqrt(hw)."""
    s = (h * w) ** 0.5
    return v * torch.tensor((w / s, h / s), dtype=v.dtype, device=v.device)


def robust_map(a: Tensor, b: Tensor, h: int, w: int, mapping: str = "huber",
               delta: float = 0.01) -> Tensor:
    """mapping.py:35-43 + mapping_huber.py:19-34 / mapping_l1.py:16-20 / mapping_l2.py:16-21."""
    d = aspect_correct(a, h, w) - aspect_correct(b, h, w)
    if mapping == "l2":
        return 0.5 * (d * d).sum(dim=-1)
    n = d.norm(dim=-1)
    if mapping == "l1":
        return n
    if mapping == "huber":
        return F.huber_loss(n, torch.zeros_like(n), reduction="none", delta=delta) / delta
    raise ValueError(mapping)


# --------------------------------------------------------------------------------------
# a15: dense bidirectional flow loss
# --------------------------------------------------------------------------------------


@dataclass
class Flows:
    """flow/flow_predictor.py:17-21."""
    forward: Tensor  # (b, p, h, w, 2)
    backward: Tensor  # (b, p, h, w, 2)
    forward_mask: Tensor  # (b, p, h, w)
    backward_mask: Tensor  # (b, p, h, w)


@dataclass
class Tracks:
    """tracking/track_predictor.py:14-20."""
    xy: Tensor  # (b, f_seg, n, 2)
    visibility: Tensor  # (b, f_seg, n) bool
    start_frame: int


def flow_loss(surfaces: Tensor, extrinsics: Tensor, k: Tensor, flows: Flows,
              mapping: str = "huber", delta: float = 0.01) -> Tensor:
    """loss_flow.py:31-70 (unweighted): (sum fwd + sum bwd) / (mask sum or 1)."""
    _, _, h, w, _ = surfaces.shape
    xy = pixel_grid(h, w, surfaces.dtype, surfaces.device)
    fwd = robust_map(forward_flow_positions(surfaces, extrinsics, k) - xy, flows.forward,
                     h, w, mapping, delta)
    bwd = robust_map(backward_flow_positions(surfaces, extrinsics, k) - xy, flows.backward,
                     h, w, mapping, delta)
    num = (fwd * flows.forward_mask).sum() + (bwd * flows.backward_mask).sum()
    den = flows.forward_mask.sum() + flows.backward_mask.sum()
    return num / (den if float(den) != 0.0 else 1)


# --------------------------------------------------------------------------------------
# a16: track reprojection loss
# --------------------------------------------------------------------------------------


def track_positions(surfaces: Tensor, extrinsics: Tensor, k: Tensor, tracks: Tracks):
    """projection.py:255-298 (compute_track_flow) for one segment.

    Returns target xy (b, fs, ft, n, 2) and the validity mask (b, fs, ft, n): both ends
    visible, source inside [0,1)^2, *predicted* target inside [0,1)^2.
    """
    b, f, h, w, _ = surfaces.shape
    img = surfaces.reshape(b * f, h, w, 3).permute(0, 3, 1, 2)
    xyz = bilinear_border(img, tracks.xy.reshape(b * f, -1, 2)).reshape(b, f, -1, 3)
    rel = torch.linalg.inv(extrinsics)[:, None, :, None] @ extrinsics[:, :, None, None]
    target = reproject(xyz[:, :, None], rel, k[:, None, :, None])
    src = tracks.xy[:, :, None]
    inside = lambda v: ((v >= 0) & (v < 1)).all(dim=-1)  # noqa: E731
    vis = tracks.visibility[:, :, None] & tracks.visibility[:, None, :]
    return target, vis & inside(src) & inside(target)


def tracking_loss(surfaces: Tensor, extrinsics: Tensor, k: Tensor,
                  tracks: Sequence[Tracks], mapping: str = "huber",
                  delta: float = 0.01) -> Tensor:
    """loss_tracking.py:28-61 (unweighted)."""
    _, _, h, w, _ = surfaces.shape
    num = 0
    den = 0
    for seg in tracks:
        n_f = seg.xy.shape[1]
        s = seg.start_frame
        target, vis = track_positions(surfaces[:, s:s + n_f], extrinsics[:, s:s + n_f],
                                      k[:, s:s + n_f], seg)
        per = robust_map(target, seg.xy[:, None], h, w, mapping, delta) * vis
        num = num + per.sum()
        den = den + vis.sum()
    return num / (den if float(den) != 0.0 else 1)


# --------------------------------------------------------------------------------------
# a9 / a10: intrinsics
# --------------------------------------------------------------------------------------


def softmin_residuals(depths: Tensor, weights: Tensor, backward_flow: Tensor, indices: Tensor,
                      candidates: Tensor) -> Tensor:
    """Weighted backward-flow residuals of the sweep of intrinsics_softmin.py:84-124 on the first
    frame pair: Procrustes with each candidate's intrinsics at the points `indices`, then
    (induced flow - flow) * weight there.

    depths (b, f, h, w), weights (b, f-1, h, w), backward_flow (b, f-1, h, w, 2),
    indices (p,), candidates (n,).  Returns (b, n, p, 2).
    """
    b, _, h, w = depths.shape
    n = candidates.shape[0]
    dt, dev = depths.dtype, depths.device
    cand_k = intrinsics_from_focal(candidates.to(dt), h, w)  # (n, 3, 3)
    xy = pixel_grid(h, w, dt, dev)
    d2 = depths[:, :2].repeat_interleave(n, dim=0)  # (b n) 2 h w
    k2 = cand_k.repeat(b, 1, 1)[:, None].expand(b * n, 2, 3, 3)
    surf = unproject(xy, d2, k2[:, :, None, None])
    rel = relative_poses(surf, backward_flow[:, :1].repeat_interleave(n, dim=0),
                         weights[:, :1].repeat_interleave(n, dim=0), indices)
    ext = pose_chain(rel)
    pts = surf.reshape(b * n, 2, h * w, 3)[:, :, indices]
    pos = backward_flow_positions(pts, ext, k2).reshape(b, n, -1, 2)
    flow = pos - xy.reshape(h * w, 2)[indices]
    flow_gt = backward_flow[:, :1].reshape(b, 1, h * w, 2)[:, :, indices]
    wsel = weights[:, :1].reshape(b, 1, h * w, 1)[:, :, indices]
    return (flow - flow_gt) * wsel


def softmin_errors(depths: Tensor, weights: Tensor, backward_flow: Tensor, indices: Tensor,
                   candidates: Tensor) -> Tensor:
    """Per-candidate flow errors of the sweep (intrinsics_softmin.py:125): the L1 norm of
    :func:`softmin_residuals` over the points, (b, n)."""
    return softmin_residuals(depths, weights, backward_flow, indices, candidates).abs().sum(dim=(-1, -2))


def softmin_intrinsics(err: Tensor, candidates: Tensor, h: int, w: int):
    """intrinsics_softmin.py:126-131: the softmin over the sweep's errors (b, n) weights the
    candidates' intrinsics.  Returns (K (b, 3, 3), softmin weights (b, n))."""
    cand_k = intrinsics_from_focal(candidates.to(err.dtype), h, w)  # (n, 3, 3)
    sm = F.softmin((err - err.min(dim=1, keepdim=True).values) * 10, dim=1)
    k = (cand_k[None] * sm[:, :, None, None]).sum(dim=1)
    return k, sm


def softmin_focal(depths: Tensor, weights: Tensor, backward_flow: Tensor, indices: Tensor,
                  candidates: Tensor):
    """Candidate sweep of intrinsics_softmin.py:84-131 on the first frame pair:
    :func:`softmin_intrinsics` of :func:`softmin_errors`.

    Returns (K (b, 3, 3), softmin weights (b, n)).
    """
    _, _, h, w = depths.shape
    err = softmin_errors(depths, weights, backward_flow, indices, candidates)
    return softmin_intrinsics(err, candidates, h, w)


# --------------------------------------------------------------------------------------
# a11 / a17: model forward and the overfit training step
# --------------------------------------------------------------------------------------


@dataclass
class OverfitConfig:
    """Values of config/**.yaml that the hot path reads."""
    initial_depth: float = 0.1  # model/backbone/explicit_depth.yaml
    weight_sensitivity: float = 100.0
    use_correspondence_weights: bool = True  # overfit.yaml:44-45
    procrustes_points: Optional[int] = None  # ablation_explicit_depth.yaml:11-12 (default 1000)
    procrustes_randomize: bool = False
    intrinsics: str = "softmin"  # "softmin" | "regressed"
    initial_focal: float = 0.85  # model/intrinsics/regressed.yaml
    softmin_points: int = 8192  # model/intrinsics/softmin.yaml
    softmin_min: float = 0.5
    softmin_max: float = 2.0
    softmin_candidates: int = 60
    regression_after: Optional[int] = 1000
    regression_window: int = 100
    flow_weight: float = 1000.0  # loss/flow.yaml
    flow_enable_after: int = 0
    tracking_weight: float = 100.0  # loss/tracking.yaml
    tracking_enable_after: int = 50
    use_tracking: bool = False
    mapping: str = "huber"
    delta: float = 0.01  # loss/mapping/huber.yaml
    lr: float = 3e-5  # overfit.yaml:30


@dataclass
class ModelOutput:
    """model.py:24-30."""
    depths: Tensor
    surfaces: Tensor
    intrinsics: Tensor
    extrinsics: Tensor
    backward_correspondence_weights: Tensor


class OverfitOracle:
    """Model + losses + Adam for the explicit-depth overfit run.

    Restates model.py:54-90 (forward), loss.py:31-47 (gating/weighting),
    model_wrapper_overfit.py:51-73 (training_step) and :104-105 (Adam(lr)).
    ``global_step`` is the number of optimiser steps already taken.
    """

    def __init__(self, cfg: OverfitConfig, num_frames: int, h: int, w: int,
                 dtype=torch.float32):
        self.cfg, self.f, self.h, self.w, self.dtype = cfg, num_frames, h, w, dtype
        self.depth = torch.full((num_frames, h, w), cfg.initial_depth, dtype=dtype,
                                requires_grad=True)
        self.weights = torch.zeros((num_frames - 1, h, w), dtype=dtype, requires_grad=True)
        focal0 = cfg.initial_focal if cfg.intrinsics == "regressed" else 0.0
        self.focal = torch.tensor(focal0, dtype=dtype, requires_grad=True)
        self.candidates = torch.linspace(cfg.softmin_min, cfg.softmin_max,
                                         cfg.softmin_candidates, dtype=dtype)
        self.window: list[Tensor] = []
        self.global_step = 0
        self.training = True
        self.optimizer = torch.optim.Adam(self.parameters(), lr=cfg.lr)

    def parameters(self):
        return [self.depth, self.weights, self.focal]

    # -- intrinsics (intrinsics_softmin.py:63-141, intrinsics_regressed.py:32-41) --
    def _intrinsics(self, depths, weights, flows: Flows, step: int,
                    softmin_indices: Optional[Tensor]):
        c = self.cfg
        b = depths.shape[0]
        regress = c.intrinsics == "regressed" or (
            c.regression_after is not None and step >= c.regression_after)
        if regress:
            if c.intrinsics == "softmin" and step == c.regression_after:
                self.focal.data = torch.stack(self.window).mean().to(self.dtype)
            k = intrinsics_from_focal(self.focal, self.h, self.w)
            return k.expand(b, self.f, 3, 3)
        if softmin_indices is None:
            softmin_indices = torch.randperm(self.h * self.w)[:c.softmin_points]
        k, sm = softmin_focal(depths, weights, flows.backward, softmin_indices,
                              self.candidates)
        if c.regression_after is not None:
            start = c.regression_after - c.regression_window
            if step >= start and self.training:
                self.window.append((self.candidates.to(sm.dtype) * sm).sum().detach())
        return k[:, None].expand(b, self.f, 3, 3)

    def forward(self, flows: Flows, step: Optional[int] = None,
                softmin_indices: Optional[Tensor] = None,
                procrustes_idx: Optional[Tensor] = None) -> ModelOutput:
        """`procrustes_idx` replaces the point set that `procrustes_points` /
        `procrustes_randomize` would select (a5): to compare with an implementation on the exact
        indices it used."""
        c = self.cfg
        step = self.global_step if step is None else step
        depths, weights = explicit_backbone(self.depth, self.weights, c.weight_sensitivity)
        if not c.use_correspondence_weights:
            weights = torch.ones_like(weights)
        k = self._intrinsics(depths, weights, flows, step, softmin_indices)
        xy = pixel_grid(self.h, self.w, self.dtype)
        surfaces = unproject(xy, depths, k[:, :, None, None])
        idx = procrustes_idx if procrustes_idx is not None else \
            procrustes_indices(self.h, self.w, c.procrustes_points, c.procrustes_randomize)
        extrinsics = align_surfaces(surfaces, flows.backward, weights, idx)
        return ModelOutput(depths, surfaces, k, extrinsics, weights)

    def losses(self, out: ModelOutput, flows: Flows, tracks, step: int) -> dict:
        c = self.cfg
        res = {}
        if step < c.flow_enable_after:
            res["flow"] = torch.zeros((), dtype=torch.float32)
        else:
            res["flow"] = c.flow_weight * flow_loss(out.surfaces, out.extrinsics,
                                                    out.intrinsics, flows, c.mapping, c.delta)
        if c.use_tracking:
            if step < c.tracking_enable_after:
                res["tracking"] = torch.zeros((), dtype=torch.float32)
            else:
                res["tracking"] = c.tracking_weight * tracking_loss(
                    out.surfaces, out.extrinsics, out.intrinsics, tracks, c.mapping, c.delta)
        return res

    def training_step(self, flows: Flows, tracks=None,
                      softmin_indices: Optional[Tensor] = None,
                      procrustes_idx: Optional[Tensor] = None) -> dict:
        """One optimiser step; returns the logged quantities (detached)."""
        step = self.global_step
        self.optimizer.zero_grad(set_to_none=True)
        out = self.forward(flows, step, softmin_indices, procrustes_idx)
        parts = self.losses(out, flows, tracks, step)
        total = sum(parts.values())
        total.backward()
        grads = {"depth": self.depth.grad, "weights": self.weights.grad,
                 "focal": self.focal.grad}
        grads = {k: (None if v is None else v.detach().clone()) for k, v in grads.items()}
        self.optimizer.step()
        self.global_step += 1
        return {"loss": float(total.detach()),
                "parts": {k: float(v.detach()) for k, v in parts.items()},
                "extrinsics": out.extrinsics.detach(), "intrinsics": out.intrinsics.detach(),
                "grads": grads}


# --------------------------------------------------------------------------------------
# Synthetic inputs (SURVEY 8(d)); shared by tests and bench so both sides see the same data
# --------------------------------------------------------------------------------------


def synthetic_flows(f: int, h: int, w: int, seed: int = 0, sigma: float = 0.01,
                    dtype=torch.float32, b: int = 1) -> Flows:
    """"Throughput set": iid N(0, sigma^2) flows in normalised units, U(0,1) masks."""
    g = torch.Generator().manual_seed(seed)
    p = f - 1
    mk = lambda *s: torch.randn(*s, generator=g, dtype=torch.float32).to(dtype) * sigma  # noqa
    un = lambda *s: torch.rand(*s, generator=g, dtype=torch.float32).to(dtype)  # noqa
    return Flows(mk(b, p, h, w, 2), mk(b, p, h, w, 2), un(b, p, h, w), un(b, p, h, w))


def synthetic_tracks(f: int, n_points: int = 1225, interval: int = 5, radius: int = 20,
                     seed: int = 0, dtype=torch.float32, p_visible: float = 0.7,
                     b: int = 1) -> list[Tracks]:
    """Segment layout of tracking/__init__.py:80-110 (one segment per `interval` frames,
    covering [mid - radius, mid + radius]); uniform xy, Bernoulli visibility."""
    g = torch.Generator().manual_seed(seed + 1)
    segs = []
    for mid in range(0, f, interval):
        lo, hi = max(0, mid - radius), min(f, mid + radius + 1)
        xy = torch.rand(b, hi - lo, n_points, 2, generator=g).to(dtype)
        vis = torch.rand(b, hi - lo, n_points, generator=g) < p_visible
        segs.append(Tracks(xy, vis, lo))
    return segs


def consistent_scene(f: int, h: int, w: int, seed: int = 0, focal: float = 0.85,
                     dtype=torch.float64, rotation: float = 0.02, translation: float = 0.03):
    """"Parity set": one static surface (the inside of a sphere) seen by cameras that move by
    an SE(3) step per frame (axis-angle ~ N(0, rotation^2), translation ~ N(0, translation^2)
    per component); depths are exact ray/sphere intersections and flows the exact induced
    correspondences, so Procrustes is well conditioned and recovers the motion up to
    bilinear-interpolation error.  Returns (depth (f,h,w), Flows, focal, extrinsics (1,f,4,4))."""
    g = torch.Generator().manual_seed(seed)
    rel = torch.eye(4, dtype=torch.float64).repeat(f - 1, 1, 1)
    ang = rotation * torch.randn(f - 1, 3, generator=g, dtype=torch.float64)
    for i in range(f - 1):
        ax, ay, az = ang[i]
        skew = torch.tensor([[0, -az, ay], [az, 0, -ax], [-ay, ax, 0]], dtype=torch.float64)
        rel[i, :3, :3] = torch.linalg.matrix_exp(skew)
    rel[:, :3, 3] = translation * torch.randn(f - 1, 3, generator=g, dtype=torch.float64)
    ext = pose_chain(rel[None])  # camera-to-world
    k = intrinsics_from_focal(torch.tensor(focal, dtype=torch.float64), h, w).expand(1, f, 3, 3)
    xy = pixel_grid(h, w, torch.float64)
    rays = unproject(xy, torch.ones(1, f, h, w, dtype=torch.float64), k[:, :, None, None])
    # ray/sphere: | o + z d - c |^2 = r^2 with o, d the camera centre / ray in world space
    centre = torch.tensor([0.2, -0.1, 0.5], dtype=torch.float64)
    radius = 3.0
    d = matvec(ext[:, :, None, None, :3, :3], rays)
    o = ext[:, :, None, None, :3, 3] - centre
    a_ = (d * d).sum(-1)
    b_ = 2 * (d * o).sum(-1)
    c_ = (o * o).sum(-1) - radius ** 2
    depth = ((-b_ + torch.sqrt(b_ * b_ - 4 * a_ * c_)) / (2 * a_))[0]  # far root: inside wall
    surf = unproject(xy, depth[None], k[:, :, None, None])
    fwd = forward_flow_positions(surf, ext, k) - xy
    bwd = backward_flow_positions(surf, ext, k) - xy
    u = lambda *s: 0.5 + 0.5 * torch.rand(*s, generator=g, dtype=torch.float64)  # noqa
    flows = Flows(fwd.to(dtype), bwd.to(dtype), u(1, f - 1, h, w).to(dtype),
                  u(1, f - 1, h, w).to(dtype))
    return depth.to(dtype), flows, focal, ext


def scene_tracks(depth: Tensor, ext: Tensor, focal: float, segments: Sequence[tuple[int, int]],
                 n_points: int, seed: int = 0, p_occluded: float = 0.1,
                 dtype=torch.float64) -> list[Tracks]:
    """Point tracks consistent with a :func:`consistent_scene` (depth (f,h,w), camera-to-world
    extrinsics (1,f,4,4)).  For each (start_frame, rows) segment, `n_points` pixel centres of the
    first frame are unprojected with the scene depth and projected into every frame of the segment.
    A point is visible where it lies in front of the camera and inside [0,1)^2, except for a random
    fraction `p_occluded` of the samples.  The tracks agree with the scene up to the depth
    interpolation, so their reprojection residuals are small (the Huber quadratic branch)."""
    g = torch.Generator().manual_seed(seed + 2)
    _, h, w = depth.shape
    k = intrinsics_from_focal(torch.tensor(focal, dtype=torch.float64), h, w)
    xy_all = pixel_grid(h, w, torch.float64).reshape(h * w, 2)
    segs = []
    for start, rows in segments:
        pix = torch.randint(0, h * w, (n_points,), generator=g)
        cam = unproject(xy_all[pix], depth[start].reshape(h * w)[pix].to(torch.float64), k)
        world = matvec(ext[0, start], to_homogeneous(cam))
        moved = matvec(torch.linalg.inv(ext[0, start:start + rows])[:, None], world[None])[..., :3]
        xy = project_camera_space(moved, k)
        front = moved[..., 2] > 0
        vis = front & ((xy >= 0) & (xy < 1)).all(dim=-1)
        vis &= torch.rand(rows, n_points, generator=g, dtype=torch.float64) >= p_occluded
        xy = torch.where(front[..., None], xy, torch.full_like(xy, 2.0))
        segs.append(Tracks(xy[None].to(dtype), vis[None], start))
    return segs


def flow_regime(kind: str, f: int, h: int, w: int, seed: int = 0, b: int = 1):
    """Float64 depth (b,f,h,w), Flows, focal and camera-to-world extrinsics (b,f,4,4) or None, for
    the flow regimes the hot path meets beyond :func:`synthetic_flows`' few-pixel noise:

    - ``iid``: synthetic_flows (sigma 0.01), depth 1 + U(0,1);
    - ``shift``: iid + a coherent (0.2, -0.2) backward motion (forward: the opposite), larger than
      the scatter window's halo at widths above 80 px and heights above 60;
    - ``leave``: iid + (0.3, 0): the right 30 % of every later frame maps past the right border;
    - ``outliers``: 5 % of the flows replaced by N(0, 0.5^2), far outside any window;
    - ``zoom``: iid + a divergent backward flow 0.6 (xy - 0.5) about the centre, so the taps of one
      tile spread over 1.6x its extent and leave the frame near the borders;
    - ``scene``: :func:`consistent_scene` with 0.08 rad / 0.3 steps per frame (about a fifth of
      the correspondences leave the frame), one seed per batch item."""
    if kind == "scene":
        parts = [consistent_scene(f, h, w, seed=seed + i, rotation=0.08, translation=0.3) for i in range(b)]
        flows = Flows(*(torch.cat([getattr(p[1], n) for p in parts])
                        for n in ("forward", "backward", "forward_mask", "backward_mask")))
        return torch.stack([p[0] for p in parts]), flows, parts[0][2], torch.cat([p[3] for p in parts])
    fl = synthetic_flows(f, h, w, seed=seed, dtype=torch.float64, b=b)
    g = torch.Generator().manual_seed(seed + 7)
    depth = 1.0 + torch.rand(b, f, h, w, generator=g, dtype=torch.float64)
    fwd, bwd = fl.forward, fl.backward
    if kind in ("shift", "leave"):
        s = torch.tensor([0.2, -0.2] if kind == "shift" else [0.3, 0.0], dtype=torch.float64)
        fwd, bwd = fwd - s, bwd + s
    elif kind == "outliers":
        for t in (fwd, bwd):
            m = torch.rand(t.shape[:-1], generator=g) < 0.05
            t[m] = 0.5 * torch.randn(int(m.sum()), 2, generator=g, dtype=torch.float64)
    elif kind == "zoom":
        c = pixel_grid(h, w, torch.float64) - 0.5
        fwd, bwd = fwd - (0.6 / 1.6) * c, bwd + 0.6 * c
    elif kind != "iid":
        raise ValueError(kind)
    return depth, Flows(fwd.contiguous(), bwd.contiguous(), fl.forward_mask, fl.backward_mask), 0.85, None


DEPTH_REGIMES = ("centre_far", "centre_far_weighted", "horizon", "centre_near", "scale_small", "scale_large",
                 "corner_weights")


def depth_regime(kind: str, f: int, h: int, w: int, seed: int = 0, b: int = 1):
    """Float64 depth (b,f,h,w), Flows, focal and weight logits (b,f-1,h,w) for depth maps whose
    centre pixel is not typical of the frame, and for depth scales and weight layouts far from the
    defaults.  Everything starts from ``flow_regime("iid")`` with logits 0.01 N(0, 1); a logit of -1
    is a weight of sigmoid(-100), about 0, and of +1 a weight of about 1 (sensitivity 100).

    - ``centre_far``: pixel (h//2, w//2) of every frame at depth 1000, logits -1 on the 9 x 9 block
      around it, so the outlier sits where the image centre is but takes no part in the fit;
    - ``centre_far_weighted``: the same with ordinary weights on the block, so the outlier is fitted;
    - ``horizon``: rows 0 .. h//2 + 2 (the centre pixel among them) at depth 200, the rows below at
      1 + 2 U(0,1), logits -1 on the band and on the ceil(0.04 h) rows below it (whose flows reach
      into it): the vanishing point of a forward-moving video;
    - ``centre_near``: the centre pixel at 0.01, logits -1 on its 9 x 9 block;
    - ``scale_small`` / ``scale_large``: the whole depth x 1e-2 / x 1e2 (a free gauge of FlowMap);
    - ``corner_weights``: logits +1 on the top-left block of h//6 x w//5 pixels, -1 elsewhere, so
      the weighted cloud sits far off the optical axis."""
    depth, fl, focal, _ = flow_regime("iid", f, h, w, seed=seed, b=b)
    g = torch.Generator().manual_seed(seed + 11)
    logits = 0.01 * torch.randn(b, f - 1, h, w, generator=g, dtype=torch.float64)
    cy, cx = h // 2, w // 2
    block = (slice(max(cy - 4, 0), cy + 5), slice(max(cx - 4, 0), cx + 5))
    if kind in ("centre_far", "centre_far_weighted"):
        depth[:, :, cy, cx] = 1000.0
        if kind == "centre_far":
            logits[:, :, block[0], block[1]] = -1.0
    elif kind == "horizon":
        far = h // 2 + 3
        depth[:, :, :far] = 200.0
        depth[:, :, far:] = 1.0 + 2.0 * torch.rand(b, f, h - far, w, generator=g, dtype=torch.float64)
        # weight ~0 also on the rows below the band whose backward flows (0.01 h px) reach into it: the
        # 200-deep taps of their bilinear samples would make the fit ill-posed even in float64
        logits[:, :, : far + math.ceil(0.04 * h)] = -1.0
    elif kind == "centre_near":
        depth[:, :, cy, cx] = 0.01
        logits[:, :, block[0], block[1]] = -1.0
    elif kind in ("scale_small", "scale_large"):
        depth = depth * (1e-2 if kind == "scale_small" else 1e2)
    elif kind == "corner_weights":
        logits[:] = -1.0
        logits[:, :, : max(h // 6, 1), : max(w // 5, 1)] = 1.0
    else:
        raise ValueError(kind)
    return depth.contiguous(), fl, focal, logits.contiguous()
