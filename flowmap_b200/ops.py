"""torch.autograd.Functions over the C ABI (include/flowmap_b200.h).

PyTorch is used for device memory, streams and autograd bookkeeping only; every number
is produced by the sm_90a kernels in csrc/.  Inputs must be CUDA float32 tensors in the
reference's layouts; anything else raises (there is no CPU or eager fallback).
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor

from ._lib import check, lib

MAPPINGS = {"huber": 0, "l1": 1, "l2": 2}
K_MODES = {"full": 0, "shared_focal": 1, "const": 2}


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _canon(t: Tensor, name: str, dtype=torch.float32) -> Tensor:
    if not isinstance(t, Tensor) or not t.is_cuda:
        raise ValueError(f"flowmap_b200: `{name}` must be a CUDA tensor (no CPU path exists)")
    if t.dtype != dtype:
        raise ValueError(f"flowmap_b200: `{name}` must be {dtype}, got {t.dtype}")
    return t.contiguous()


def workspace(B: int, F: int, H: int, W: int, device) -> Tensor:
    n = lib().fm_workspace_bytes(B, F, H, W)
    return torch.empty(n, dtype=torch.uint8, device=device)


def intrinsics_to_k4(intrinsics: Tensor) -> Tensor:
    """(..., 3, 3) normalised intrinsics -> (..., 4) = (fx, fy, cx, cy); differentiable."""
    return torch.stack((intrinsics[..., 0, 0], intrinsics[..., 1, 1], intrinsics[..., 0, 2],
                        intrinsics[..., 1, 2]), dim=-1)


class _Procrustes(torch.autograd.Function):
    """depths, weights, k4, backward flow [, indices] -> relative poses rt (B, F-1, 3, 4).

    flowmap/model/projection.py:213-249 + flowmap/model/procrustes.py:7-51."""

    @staticmethod
    def forward(ctx, depths, weights, k4, backward_flows, indices):
        depths = _canon(depths, "depths")
        k4 = _canon(k4, "k4")
        backward_flows = _canon(backward_flows, "backward_flows")
        weights = None if weights is None else _canon(weights, "weights")
        indices = None if indices is None else _canon(indices, "indices", torch.int64)
        B, F, H, W = depths.shape
        if backward_flows.shape != (B, F - 1, H, W, 2) or k4.shape != (B, F, 4):
            raise ValueError("flowmap_b200: procrustes shape mismatch")
        ws = workspace(B, F, H, W, depths.device)
        rt = torch.empty((B, F - 1, 3, 4), dtype=torch.float32, device=depths.device)
        with torch.cuda.device(depths.device):
            check(lib().fm_procrustes_fwd(_ptr(depths), _ptr(k4), _ptr(backward_flows),
                                          _ptr(weights), _ptr(indices),
                                          0 if indices is None else indices.numel(), _ptr(rt),
                                          _ptr(ws), B, F, H, W, _stream()), "fm_procrustes_fwd")
        ctx.save_for_backward(depths, weights, k4, backward_flows, indices, ws)
        return rt

    @staticmethod
    def backward(ctx, g_rt):
        depths, weights, k4, backward_flows, indices, ws = ctx.saved_tensors
        B, F, H, W = depths.shape
        g_rt = _canon(g_rt, "g_rt")
        g_depth = torch.zeros_like(depths)
        g_weights = None
        if weights is not None:
            g_weights = torch.empty_like(weights) if indices is None else torch.zeros_like(weights)
        g_k4 = torch.empty_like(k4)
        with torch.cuda.device(depths.device):
            check(lib().fm_procrustes_bwd(_ptr(depths), _ptr(k4), _ptr(backward_flows),
                                          _ptr(weights), _ptr(indices),
                                          0 if indices is None else indices.numel(), _ptr(g_rt),
                                          0, None, _ptr(g_depth), _ptr(g_weights), _ptr(g_k4),
                                          _ptr(ws), B, F, H, W, _stream()), "fm_procrustes_bwd")
        return g_depth, g_weights, g_k4, None, None


def procrustes_poses(depths: Tensor, weights: Optional[Tensor], k4: Tensor,
                     backward_flows: Tensor, indices: Optional[Tensor] = None) -> Tensor:
    return _Procrustes.apply(depths, weights, k4, backward_flows, indices)


def mask_sum(forward_mask: Tensor, backward_mask: Tensor) -> Tensor:
    """Device float64 scalar sum(forward_mask) + sum(backward_mask) (loss_flow.py:56,68)."""
    fm, bm = _canon(forward_mask, "forward_mask"), _canon(backward_mask, "backward_mask")
    if fm.numel() != bm.numel():
        raise ValueError("flowmap_b200: mask shapes differ")
    out = torch.empty((), dtype=torch.float64, device=fm.device)
    with torch.cuda.device(fm.device):
        check(lib().fm_mask_sum(_ptr(fm), _ptr(bm), _ptr(out), fm.numel(), _stream()),
              "fm_mask_sum")
    return out


class _FlowLoss(torch.autograd.Function):
    """Weighted dense flow loss; forward and analytic backward in one kernel pass.

    flowmap/loss/loss_flow.py:31-70, loss.py:46, projection.py:116-184, loss/mapping/*."""

    @staticmethod
    def forward(ctx, depths, rt, k4, fflow, bflow, fmask, bmask, msum, mapping, delta, weight,
                k_mode):
        depths, rt, k4 = _canon(depths, "depths"), _canon(rt, "rt"), _canon(k4, "k4")
        fflow, bflow = _canon(fflow, "flows.forward"), _canon(bflow, "flows.backward")
        fmask, bmask = _canon(fmask, "flows.forward_mask"), _canon(bmask, "flows.backward_mask")
        msum = _canon(msum, "mask_sum", torch.float64)
        B, F, H, W = depths.shape
        if (rt.shape != (B, F - 1, 3, 4) or k4.shape != (B, F, 4) or
                fflow.shape != (B, F - 1, H, W, 2) or bflow.shape != fflow.shape or
                fmask.shape != (B, F - 1, H, W) or bmask.shape != fmask.shape):
            raise ValueError("flowmap_b200: flow loss shape mismatch")
        dev = depths.device
        ws = workspace(B, F, H, W, dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        g_depth = torch.empty_like(depths)
        g_rt = torch.empty_like(rt)
        g_k4 = torch.empty_like(k4)
        with torch.cuda.device(dev):
            check(lib().fm_flow_loss_fwd_bwd(_ptr(depths), _ptr(k4), _ptr(rt), _ptr(fflow),
                                             _ptr(bflow), _ptr(fmask), _ptr(bmask), _ptr(msum),
                                             MAPPINGS[mapping], float(delta), float(weight),
                                             K_MODES[k_mode], _ptr(loss), _ptr(g_depth), _ptr(g_rt),
                                             _ptr(g_k4),
                                             _ptr(ws), B, F, H, W, _stream()),
                  "fm_flow_loss_fwd_bwd")
        ctx.save_for_backward(g_depth, g_rt, g_k4)
        return loss

    @staticmethod
    def backward(ctx, go):
        g_depth, g_rt, g_k4 = ctx.saved_tensors
        return (g_depth * go, g_rt * go, g_k4 * go) + (None,) * 9


def flow_loss(depths, rt, k4, fflow, bflow, fmask, bmask, msum, mapping="huber", delta=0.01,
              weight=1.0, k_mode="full") -> Tensor:
    """k_mode: "full" (any per-frame intrinsics), "shared_focal" (k4 derives from ONE focal
    length with a fixed principal point: cheaper kernel, gradient routed through fx only) or
    "const" (intrinsics receive no gradient)."""
    return _FlowLoss.apply(depths, rt, k4, fflow, bflow, fmask, bmask, msum, mapping, delta, weight,
                           k_mode)


class _PoseChain(torch.autograd.Function):
    """rt (B, F-1, 3, 4) -> camera-to-world extrinsics (B, F, 4, 4); projection.py:187-210."""

    @staticmethod
    def forward(ctx, rt):
        rt = _canon(rt, "rt")
        B, P = rt.shape[:2]
        ext = torch.empty((B, P + 1, 4, 4), dtype=torch.float32, device=rt.device)
        with torch.cuda.device(rt.device):
            check(lib().fm_pose_chain(_ptr(rt), _ptr(ext), B, P + 1, _stream()), "fm_pose_chain")
        ctx.save_for_backward(rt, ext)
        return ext

    @staticmethod
    def backward(ctx, g_ext):
        rt, ext = ctx.saved_tensors
        g_ext = _canon(g_ext, "g_extrinsics")
        g_rt = torch.empty_like(rt)
        B, P = rt.shape[:2]
        with torch.cuda.device(rt.device):
            check(lib().fm_pose_chain_bwd(_ptr(rt), _ptr(ext), _ptr(g_ext), _ptr(g_rt), B, P + 1,
                                          _stream()), "fm_pose_chain_bwd")
        return g_rt


def pose_chain(rt: Tensor) -> Tensor:
    return _PoseChain.apply(rt)


class _Unproject(torch.autograd.Function):
    """depths (B, F, H, W), k4 (B, F, 4) -> surfaces (B, F, H, W, 3); projection.py:76-90 on
    the pixel grid of :93-113."""

    @staticmethod
    def forward(ctx, depths, k4):
        depths, k4 = _canon(depths, "depths"), _canon(k4, "k4")
        B, F, H, W = depths.shape
        surf = torch.empty((B, F, H, W, 3), dtype=torch.float32, device=depths.device)
        with torch.cuda.device(depths.device):
            check(lib().fm_unproject(_ptr(depths), _ptr(k4), _ptr(surf), B * F, H, W, _stream()),
                  "fm_unproject")
        ctx.save_for_backward(depths, k4)
        return surf

    @staticmethod
    def backward(ctx, g_surf):
        depths, k4 = ctx.saved_tensors
        B, F, H, W = depths.shape
        g_surf = _canon(g_surf, "g_surfaces")
        g_depth, g_k4 = torch.empty_like(depths), torch.empty_like(k4)
        ws = workspace(B, F, H, W, depths.device)
        with torch.cuda.device(depths.device):
            check(lib().fm_unproject_bwd(_ptr(depths), _ptr(k4), _ptr(g_surf), _ptr(g_depth),
                                         _ptr(g_k4), _ptr(ws), B, F, H, W, _stream()),
                  "fm_unproject_bwd")
        return g_depth, g_k4


def unproject_depth(depths: Tensor, k4: Tensor) -> Tensor:
    return _Unproject.apply(depths, k4)


def reproject(xyz: Tensor, rt: Tensor, k4: Tensor, with_in_front: bool = False):
    """Forward-only: xyz (items, n, 3), rt (items, 3, 4), k4 (items, 4) -> xy (items, n, 2)
    [, in_front (items, n) bool]."""
    xyz, rt, k4 = _canon(xyz, "xyz"), _canon(rt, "rt"), _canon(k4, "k4")
    items, n = xyz.shape[:2]
    out = torch.empty((items, n, 2), dtype=torch.float32, device=xyz.device)
    front = torch.empty((items, n), dtype=torch.uint8, device=xyz.device) if with_in_front else None
    with torch.cuda.device(xyz.device):
        check(lib().fm_reproject(_ptr(xyz), _ptr(rt), _ptr(k4), _ptr(out), _ptr(front), items, n,
                                 _stream()), "fm_reproject")
    return (out, front.bool()) if with_in_front else out


class _UnprojectPoints(torch.autograd.Function):
    """projection.py:76-90 on explicit coordinates."""

    @staticmethod
    def forward(ctx, xy, z, k4):
        xy, z, k4 = _canon(xy, "coordinates"), _canon(z, "z"), _canon(k4, "k4")
        items, n = z.shape
        shared = 1 if xy.shape[0] == 1 and items > 1 else 0
        out = torch.empty((items, n, 3), dtype=torch.float32, device=z.device)
        with torch.cuda.device(z.device):
            check(lib().fm_unproject_points(_ptr(xy), _ptr(z), _ptr(k4), _ptr(out), items, n, shared,
                                            _stream()), "fm_unproject_points")
        ctx.save_for_backward(xy, z, k4)
        ctx.shared = shared
        return out

    @staticmethod
    def backward(ctx, g_out):
        xy, z, k4 = ctx.saved_tensors
        items, n = z.shape
        g_out = _canon(g_out, "g_out")
        g_z, g_k4 = torch.empty_like(z), torch.empty_like(k4)
        ws = torch.empty(lib().fm_points_workspace_bytes(items), dtype=torch.uint8, device=z.device)
        with torch.cuda.device(z.device):
            check(lib().fm_unproject_points_bwd(_ptr(xy), _ptr(z), _ptr(k4), _ptr(g_out), _ptr(g_z),
                                                _ptr(g_k4), _ptr(ws), items, n, ctx.shared, _stream()),
                  "fm_unproject_points_bwd")
        return None, g_z, g_k4


def unproject_points(xy: Tensor, z: Tensor, k4: Tensor) -> Tensor:
    """xy (items or 1, n, 2), z (items, n), k4 (items, 4) -> (items, n, 3)."""
    return _UnprojectPoints.apply(xy, z, k4)


class _AlignRigid(torch.autograd.Function):
    """flowmap/model/procrustes.py:7-51 on explicit points; returns rt (items, 3, 4)."""

    @staticmethod
    def forward(ctx, p, q, w):
        p, q, w = _canon(p, "p"), _canon(q, "q"), _canon(w, "weights")
        items, n = w.shape
        ws = torch.empty(lib().fm_points_workspace_bytes(items), dtype=torch.uint8, device=p.device)
        rt = torch.empty((items, 3, 4), dtype=torch.float32, device=p.device)
        with torch.cuda.device(p.device):
            check(lib().fm_align_rigid_fwd(_ptr(p), _ptr(q), _ptr(w), _ptr(rt), _ptr(ws), items, n,
                                           _stream()), "fm_align_rigid_fwd")
        ctx.save_for_backward(p, q, w, ws)
        return rt

    @staticmethod
    def backward(ctx, g_rt):
        p, q, w, ws = ctx.saved_tensors
        items, n = w.shape
        g_rt = _canon(g_rt, "g_rt")
        gp, gq, gw = torch.empty_like(p), torch.empty_like(q), torch.empty_like(w)
        with torch.cuda.device(p.device):
            check(lib().fm_align_rigid_bwd(_ptr(p), _ptr(q), _ptr(w), _ptr(g_rt), _ptr(gp), _ptr(gq),
                                           _ptr(gw), _ptr(ws), items, n, _stream()), "fm_align_rigid_bwd")
        return gp, gq, gw


def align_rigid_rt(p: Tensor, q: Tensor, w: Tensor) -> Tensor:
    return _AlignRigid.apply(p, q, w)


def adam_step(param: Tensor, grad: Tensor, exp_avg: Tensor, exp_avg_sq: Tensor, step: int,
              lr: float, betas=(0.9, 0.999), eps: float = 1e-8) -> None:
    """In-place torch.optim.Adam update (model_wrapper_overfit.py:104-105)."""
    for t in (param, grad, exp_avg, exp_avg_sq):
        if not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError("flowmap_b200: adam_step needs contiguous CUDA float32 tensors")
    with torch.cuda.device(param.device):
        check(lib().fm_adam_step(_ptr(param), _ptr(grad), _ptr(exp_avg), _ptr(exp_avg_sq),
                                 param.numel(), lr, betas[0], betas[1], eps, step, _stream()),
              "fm_adam_step")


class StepClock:
    """Device-resident step state (fm_step_clock_tick): Adam's bias-correction scalars on the
    optimiser's own step counts and a per-step seed.  With it every optimisation step is the same
    sequence of launches with the same arguments -- the precondition for replaying it as a CUDA graph."""

    def __init__(self, device, lr: float, betas=(0.9, 0.999), base_seed: int | None = None):
        self.buf = torch.zeros(32, dtype=torch.uint8, device=device)  # FM_STEP_CLOCK_BYTES
        self.lr, self.betas = lr, betas
        self.base_seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if base_seed is None else base_seed
        self.steps = self.focal_steps = 0  # host mirror of the device counters

    @property
    def ptr(self) -> int:
        return self.buf.data_ptr()

    def set(self, steps: int, focal_steps: int) -> None:
        """Counts of completed updates (the next tick makes them steps + 1)."""
        if (steps, focal_steps) != (self.steps, self.focal_steps):
            self.buf.view(torch.int32)[:2].copy_(torch.tensor([steps, focal_steps], dtype=torch.int32))
            self.steps, self.focal_steps = steps, focal_steps

    def tick(self, tick_focal: bool) -> None:
        with torch.cuda.device(self.buf.device):
            check(lib().fm_step_clock_tick(self.ptr, self.lr, self.betas[0], self.betas[1], self.base_seed,
                                           int(tick_focal), _stream()), "fm_step_clock_tick")
        self.steps += 1
        self.focal_steps += int(tick_focal)


def adam_step_clock(param: Tensor, grad: Tensor, exp_avg: Tensor, exp_avg_sq: Tensor, clock: StepClock,
                    focal_clock: bool = False, eps: float = 1e-8) -> None:
    """adam_step with the bias corrections of the current tick of `clock`."""
    for t in (param, grad, exp_avg, exp_avg_sq):
        if not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError("flowmap_b200: adam_step needs contiguous CUDA float32 tensors")
    with torch.cuda.device(param.device):
        check(lib().fm_adam_step_clock(_ptr(param), _ptr(grad), _ptr(exp_avg), _ptr(exp_avg_sq), param.numel(),
                                       clock.ptr, int(focal_clock), clock.betas[0], clock.betas[1], eps, _stream()),
              "fm_adam_step_clock")


def random_subset_clock(clock: StepClock, num_items: int, out: Tensor) -> Tensor:
    """random_subset seeded by the current tick of `clock`, into the caller's int64 buffer."""
    with torch.cuda.device(out.device):
        check(lib().fm_random_subset_clock(clock.ptr, num_items, out.numel(), _ptr(out), _stream()),
              "fm_random_subset_clock")
    return out


class PackedTracks:
    """All segments of a list[Tracks] in the flat layout fm_track_loss_* expects.

    Several videos (the packed fused step): `tracks` is a list of B such lists and `video_frames` the list
    of their frame counts F_b, or one count F for videos of one length; segment s of video b is packed
    with start frame fo_b + s.start_frame, fo_b = F_0 + ... + F_{b-1}, so the segments of one video
    address its rows of the packed frame arrays and never cross videos."""

    def __init__(self, tracks, device, video_frames=None):
        videos = [tracks] if video_frames is None else tracks
        if isinstance(video_frames, int):
            video_frames = [video_frames] * len(videos)
        counts = None if video_frames is None else [int(n) for n in video_frames]
        if counts is not None and len(counts) != len(videos):
            raise ValueError("flowmap_b200: one frame count per video")
        firsts = None if counts is None else [sum(counts[:b]) for b in range(len(counts))]
        segs, xy, vis, off = [], [], [], 0
        for b, video in enumerate(videos):
            for t in video:
                _, f, n, _ = t.xy.shape
                if t.xy.shape[0] != 1:
                    raise ValueError("flowmap_b200: tracking supports batch size 1 "
                                     "(flowmap/tracking/__init__.py:92-93)")
                start = int(t.start_frame)
                if counts is not None:
                    if start < 0 or start + f > counts[b]:
                        raise ValueError(f"flowmap_b200: a track segment of video {b} leaves its {counts[b]} frames")
                    start += firsts[b]
                segs.append((off, f, n, start))
                xy.append(t.xy[0].reshape(-1, 2))
                vis.append(t.visibility[0].reshape(-1))
                off += f * n
        if not segs:
            raise ValueError("flowmap_b200: no track segments")
        self.total = off
        self.num_segments = len(segs)
        self.max_rows = max(s[1] for s in segs)
        self.max_points = max(s[2] for s in segs)
        self.last_frame = max(s[3] + s[1] for s in segs)
        self.seg = torch.tensor(segs, dtype=torch.int32).to(device).contiguous()
        self.xy = torch.cat(xy).to(device=device, dtype=torch.float32).contiguous()
        self.vis = torch.cat(vis).to(device=device, dtype=torch.uint8).contiguous()


class _TrackLoss(torch.autograd.Function):
    """Weighted track reprojection loss over all segments.

    flowmap/loss/loss_tracking.py:28-61 + flowmap/model/projection.py:255-298."""

    @staticmethod
    def forward(ctx, depths, extrinsics, k4, packed, mapping, delta, weight, shared_k=False):
        depths, extrinsics, k4 = _canon(depths, "depths"), _canon(extrinsics, "extrinsics"), _canon(k4, "k4")
        B, F, H, W = depths.shape
        if B != 1 or extrinsics.shape != (1, F, 4, 4) or k4.shape != (1, F, 4):
            raise ValueError("flowmap_b200: tracking loss needs batch size 1 and matching shapes")
        if packed.last_frame > F:
            raise ValueError("flowmap_b200: a track segment runs past the last frame")
        dev = depths.device
        n = lib().fm_track_workspace_bytes(F, packed.total)
        ws = torch.empty(n, dtype=torch.uint8, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            check(lib().fm_track_loss_fwd_sharded(_ptr(depths), _ptr(k4), _ptr(extrinsics), _ptr(packed.seg),
                                                  packed.num_segments, packed.max_rows, packed.max_points,
                                                  _ptr(packed.xy), _ptr(packed.vis), packed.total,
                                                  MAPPINGS[mapping], float(delta), float(weight), _ptr(loss),
                                                  _ptr(ws), F, H, W, 0, 0, F, int(bool(shared_k)), _stream()),
                  "fm_track_loss_fwd")
        ctx.save_for_backward(depths, extrinsics, k4, ws)
        ctx.packed, ctx.cfg = packed, (mapping, delta, weight)
        return loss

    @staticmethod
    def backward(ctx, go):
        depths, extrinsics, k4, ws = ctx.saved_tensors
        packed, (mapping, delta, weight) = ctx.packed, ctx.cfg
        _, F, H, W = depths.shape
        go = _canon(go, "grad_output").reshape(())
        g_depth = torch.zeros_like(depths)
        g_ext = torch.empty_like(extrinsics)
        g_k4 = torch.empty_like(k4)
        with torch.cuda.device(depths.device):
            check(lib().fm_track_loss_bwd(_ptr(depths), _ptr(k4), _ptr(extrinsics), _ptr(packed.seg),
                                          packed.num_segments, packed.max_rows, packed.max_points,
                                          _ptr(packed.xy), _ptr(packed.vis), packed.total,
                                          MAPPINGS[mapping], float(delta), float(weight), _ptr(go),
                                          _ptr(g_depth), _ptr(g_ext), _ptr(g_k4), _ptr(ws), F, H, W,
                                          _stream()), "fm_track_loss_bwd")
        return g_depth, g_ext, g_k4, None, None, None, None, None


def track_loss(depths, extrinsics, k4, packed: PackedTracks, mapping="huber", delta=0.01,
               weight=1.0, shared_k: bool = False) -> Tensor:
    """shared_k: the caller only uses the sum over frames of d loss / d k4 -- true when k4 is an expand
    of one row (one focal length), and when the intrinsics take no gradient at all (ground-truth K,
    k_mode "const", which may differ per frame).  The loss, depth and pose gradients still use every
    frame's own k4; only the intrinsics gradient is left unreduced per target frame, so g_k4 is then
    meaningful only as its sum over frames."""
    return _TrackLoss.apply(depths, extrinsics, k4, packed, mapping, delta, weight, shared_k)


def candidate_k4(candidates: Tensor, h: int, w: int, batch: int) -> Tensor:
    """k4 rows (batch * n, 2, 4) of the candidate focal lengths (intrinsics/common.py:6-20)."""
    scaled = candidates.float() * (h * w) ** 0.5
    half = torch.full_like(scaled, 0.5)
    k = torch.stack((scaled / w, scaled / h, half, half), dim=-1)  # (n, 4)
    return k[None, :, None, :].expand(batch, -1, 2, -1).reshape(-1, 2, 4).contiguous()


class _SoftminErrors(torch.autograd.Function):
    """Per-candidate flow error of the focal-length sweep, (B, n).

    flowmap/model/intrinsics/intrinsics_softmin.py:84-125."""

    @staticmethod
    def forward(ctx, depths, weights, backward_flows, indices, cand_k4, n):
        depths, backward_flows = _canon(depths, "depths"), _canon(backward_flows, "backward_flows")
        weights = None if weights is None else _canon(weights, "weights")
        indices = _canon(indices, "indices", torch.int64)
        cand_k4 = _canon(cand_k4, "cand_k4")
        B, F, H, W = depths.shape
        dev = depths.device
        ws = torch.empty(lib().fm_softmin_workspace_bytes(B, n), dtype=torch.uint8, device=dev)
        err = torch.empty((B, n), dtype=torch.float32, device=dev)
        rt = torch.empty((B * n, 3, 4), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            check(lib().fm_softmin_sweep_fwd(_ptr(depths), _ptr(weights), 0.0, _ptr(backward_flows),
                                             _ptr(indices), indices.numel(), _ptr(cand_k4), n,
                                             _ptr(err), _ptr(rt), _ptr(ws), B, F, H, W, _stream()),
                  "fm_softmin_sweep_fwd")
        ctx.save_for_backward(depths, weights, backward_flows, indices, cand_k4, rt, ws)
        ctx.n = n
        return err

    @staticmethod
    def backward(ctx, g_err):
        depths, weights, backward_flows, indices, cand_k4, rt, ws = ctx.saved_tensors
        B, F, H, W = depths.shape
        g_err = _canon(g_err, "g_err")
        g_depth = torch.zeros_like(depths)
        g_weights = None if weights is None else torch.zeros_like(weights)
        with torch.cuda.device(depths.device):
            check(lib().fm_softmin_sweep_bwd(_ptr(depths), _ptr(weights), 0.0, _ptr(backward_flows),
                                             _ptr(indices), indices.numel(), _ptr(cand_k4), ctx.n,
                                             _ptr(rt), _ptr(g_err), _ptr(g_depth), _ptr(g_weights),
                                             _ptr(ws), B, F, H, W, _stream()), "fm_softmin_sweep_bwd")
        return g_depth, g_weights, None, None, None, None


def softmin_errors(depths, weights, backward_flows, indices, candidates) -> Tensor:
    b, _, h, w = depths.shape
    n = candidates.numel()
    return _SoftminErrors.apply(depths, weights, backward_flows, indices,
                                candidate_k4(candidates, h, w, b), n)


def random_subset(num_items: int, n: int, device, seed: int | None = None) -> Tensor:
    """n distinct uniformly random indices of range(num_items) (int64, random order): what
    `torch.randperm(num_items)[:n]` samples, without sorting num_items keys.  The seed is drawn
    from torch's CPU generator (so torch.manual_seed controls it) unless given."""
    if seed is None:
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    out = torch.empty(n, dtype=torch.int64, device=device)
    with torch.cuda.device(device):
        check(lib().fm_random_subset(seed, num_items, n, _ptr(out), _stream()), "fm_random_subset")
    return out
