"""CPU oracle for the stages either side of the hot path (SURVEY.md 8(f) rank 4): the
flow-side preprocessing that produces ``Flows`` and the COLMAP / point-cloud export that
consumes ``ModelExports``.

TEST INFRASTRUCTURE ONLY (same rule as ``flowmap_oracle.py``): nothing under
``flowmap_b200/`` imports this file.

Parity status: PINNED against outputs of the unmodified reference
(``tests/golden/make_golden_io.py`` -> ``tests/golden/io_*.npz``, checked by
``tests/test_oracle_golden.py``).  Everything is spelled out with index arithmetic instead of
``F.grid_sample`` / ``F.interpolate`` so that the sampling rules the CUDA kernels implement
are explicit.  Citations are relative to the reference checkout.
"""

from __future__ import annotations

import struct
from typing import Callable, Sequence

import numpy as np
import torch
from torch import Tensor


# --------------------------------------------------------------------------------------
# flow/flow_predictor.py:40-101: rescaling, consistency masks, bidirectional flow
# --------------------------------------------------------------------------------------

def bilinear_zeros(image: Tensor, xy: Tensor) -> Tensor:
    """``F.grid_sample(image, xy*2-1, bilinear, padding_mode="zeros", align_corners=False)``
    (flow_predictor.py:72-78).  image (n, c, h, w), xy (n, hh, ww, 2) in normalised [0,1]
    coordinates -> (n, c, hh, ww).  Pixel position px = x*w - .5, the four neighbours
    floor / floor+1; a neighbour outside the image contributes zero."""
    n, c, h, w = image.shape
    px = xy[..., 0] * w - 0.5
    py = xy[..., 1] * h - 0.5
    x0 = px.floor()
    y0 = py.floor()
    tx = px - x0
    ty = py - y0
    x0 = x0.long()
    y0 = y0.long()
    flat = image.reshape(n, c, h * w)
    out = torch.zeros(n, c, *xy.shape[1:3], dtype=image.dtype)
    for dy, wy in ((0, 1 - ty), (1, ty)):
        for dx, wx in ((0, 1 - tx), (1, tx)):
            xi = x0 + dx
            yi = y0 + dy
            ok = ((xi >= 0) & (xi <= w - 1) & (yi >= 0) & (yi <= h - 1)).to(image.dtype)
            idx = (yi.clamp(0, h - 1) * w + xi.clamp(0, w - 1)).reshape(n, 1, -1).expand(n, c, -1)
            tap = flat.gather(2, idx).reshape(n, c, *xy.shape[1:3])
            out = out + tap * (wx * wy * ok)[:, None]
    return out


def pixel_centres(h: int, w: int, dtype) -> Tensor:
    """projection.py:93-113 sample_image_grid: (h, w, 2) of ((col+.5)/w, (row+.5)/h)."""
    x = (torch.arange(w, dtype=dtype) + 0.5) / w
    y = (torch.arange(h, dtype=dtype) + 0.5) / h
    return torch.stack((x[None, :].expand(h, w), y[:, None].expand(h, w)), dim=-1)


def consistency_mask(videos: Tensor, flow: Tensor) -> Tensor:
    """flow_predictor.py:60-82 compute_consistency_mask.  videos (b, f, 3, h, w), flow
    (b, f-1, h, w, 2) -> (b, f-1, h, w): the colour of frame i at a pixel against the
    bilinear (zero padded) colour of frame i+1 at pixel + flow; mask = (1 - max_c |d|)^8."""
    b, f, c, h, w = videos.shape
    source = videos[:, :-1].reshape(b * (f - 1), c, h, w)
    target = videos[:, 1:].reshape(b * (f - 1), c, h, w)
    xy = pixel_centres(h, w, videos.dtype) + flow.reshape(b * (f - 1), h, w, 2)
    deltas = (source - bilinear_zeros(target, xy)).abs().max(dim=1).values
    return ((1 - deltas) ** 8).reshape(b, f - 1, h, w)


def resize_bilinear(x: Tensor, shape: Sequence[int]) -> Tensor:
    """``F.interpolate(x, shape, mode="bilinear", align_corners=False)`` (no antialiasing), x
    (n, c, h, w).  Source index = (dst + .5) * (in / out) - .5 clamped below at 0; neighbours
    i0 = floor, i1 = min(i0 + 1, in - 1); weights (1 - t, t)."""
    n, c, h, w = x.shape
    ho, wo = shape

    def axis(n_in, n_out):
        src = ((torch.arange(n_out, dtype=x.dtype) + 0.5) * (n_in / n_out) - 0.5).clamp(min=0)
        i0 = src.floor().long().clamp(max=n_in - 1)
        i1 = (i0 + 1).clamp(max=n_in - 1)
        return i0, i1, src - i0

    y0, y1, ty = axis(h, ho)
    x0, x1, tx = axis(w, wo)
    top = x[:, :, y0][:, :, :, x0] * (1 - tx) + x[:, :, y0][:, :, :, x1] * tx
    bot = x[:, :, y1][:, :, :, x0] * (1 - tx) + x[:, :, y1][:, :, :, x1] * tx
    return top * (1 - ty)[:, None] + bot * ty[:, None]


def rescale_flow(flow: Tensor, shape: Sequence[int]) -> Tensor:
    """flow_predictor.py:40-48: (b, f, h, w, 2) -> (b, f, h', w', 2); values are in normalised
    units and are NOT rescaled."""
    b, f, h, w, _ = flow.shape
    out = resize_bilinear(flow.reshape(b * f, h, w, 2).permute(0, 3, 1, 2), shape)
    return out.permute(0, 2, 3, 1).reshape(b, f, *shape, 2)


def rescale_mask(mask: Tensor, shape: Sequence[int]) -> Tensor:
    """flow_predictor.py:50-58."""
    b, f, h, w = mask.shape
    return resize_bilinear(mask.reshape(b * f, 1, h, w), shape).reshape(b, f, *shape)


def bidirectional_flows(predict: Callable[[Tensor], Tensor], videos: Tensor, flow_shape):
    """flow_predictor.py:84-101 compute_bidirectional_flow: forward flow on the video,
    backward flow = forward flow of the time-reversed video, flipped back; each with its
    consistency mask computed at the predictor's resolution and then rescaled."""
    forward = predict(videos)
    forward_mask = rescale_mask(consistency_mask(videos, forward), flow_shape)
    forward = rescale_flow(forward, flow_shape)
    reversed_videos = videos.flip(dims=(1,))
    backward = predict(reversed_videos)
    backward_mask = rescale_mask(consistency_mask(reversed_videos, backward), flow_shape)
    backward = rescale_flow(backward, flow_shape)
    return forward, backward.flip(dims=(1,)), forward_mask, backward_mask.flip(dims=(1,))


# --------------------------------------------------------------------------------------
# export/colmap.py:56-111, 171-213 and misc/cropping.py:55-70: export
# --------------------------------------------------------------------------------------

def center_crop_intrinsics(k: Tensor, old_shape, new_shape) -> Tensor:
    """misc/cropping.py:55-70: fx *= w_old / w_new, fy *= h_old / h_new."""
    k = k.clone()
    k[..., 0, 0] *= old_shape[1] / new_shape[1]
    k[..., 1, 1] *= old_shape[0] / new_shape[0]
    return k


def world_points(depths: Tensor, intrinsics: Tensor, extrinsics: Tensor) -> Tensor:
    """export/colmap.py:84-101: per frame, unproject every pixel centre with its depth and
    move it to world space with the camera-to-world matrix.  depths (f, h, w), intrinsics
    (f, 3, 3), extrinsics (f, 4, 4) -> (f*h*w, 3), frames concatenated, row-major pixels."""
    f, h, w = depths.shape
    xy = pixel_centres(h, w, depths.dtype)
    hom = torch.cat((xy, torch.ones(h, w, 1, dtype=depths.dtype)), dim=-1)
    rays = torch.einsum("fij,hwj->fhwi", torch.linalg.inv(intrinsics), hom)
    cam = rays * depths[..., None]
    cam_h = torch.cat((cam, torch.ones(f, h, w, 1, dtype=depths.dtype)), dim=-1)
    return torch.einsum("fij,fhwj->fhwi", extrinsics, cam_h)[..., :3].reshape(-1, 3)


def colmap_model_bytes(extrinsics: Tensor, intrinsics: Tensor, names: Sequence[str],
                       image_shape) -> tuple[bytes, bytes]:
    """export/colmap.py:171-213 write_colmap_model + third_party/colmap/read_write_model.py
    :188-202 (cameras.bin) and :334-352 (images.bin): one PINHOLE camera (model id 1) per
    frame with (fx*w, fy*h, cx*w, cy*h), one image per frame with the world-to-camera rotation
    as (qw, qx, qy, qz) (scipy convention, as the reference) and translation; little endian."""
    from scipy.spatial.transform import Rotation

    h, w = image_shape
    cams = struct.pack("<Q", len(intrinsics))
    for i, k in enumerate(intrinsics):
        k = k.detach().clone()
        k[0] *= w
        k[1] *= h
        cams += struct.pack("<iiQQ", i + 1, 1, w, h)
        for p in (k[0, 0], k[1, 1], k[0, 2], k[1, 2]):
            cams += struct.pack("<d", float(p))
    imgs = struct.pack("<Q", len(extrinsics))
    for i, (c2w, name) in enumerate(zip(extrinsics, names)):
        w2c = c2w.inverse().detach().cpu().numpy()
        qx, qy, qz, qw = Rotation.from_matrix(w2c[:3, :3]).as_quat()
        imgs += struct.pack("<i", i + 1)
        imgs += struct.pack("<dddd", *np.array((qw, qx, qy, qz)).tolist())
        imgs += struct.pack("<ddd", *w2c[:3, 3].tolist())
        imgs += struct.pack("<i", i + 1)
        imgs += name.encode("utf-8") + b"\x00"
        imgs += struct.pack("<Q", 0)
    return cams, imgs
