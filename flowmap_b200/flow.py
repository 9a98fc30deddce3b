"""Flow-side preprocessing just before the hot path: what turns a flow predictor's raw output
into the ``Flows`` the losses consume (flowmap/flow/flow_predictor.py:40-101).

The predictor networks themselves (RAFT, GMFlow) stay with the reference; any callable
``videos (b f 3 h w) -> flow (b f-1 h w 2)`` can be plugged in.  The consistency masks and the
rescaling run on the sm_90a kernels of csrc/fm_io.cu (no CPU path).
"""
from __future__ import annotations

from typing import Callable

import torch
from torch import Tensor

from ._lib import check, lib
from .ops import _canon, _ptr, _stream
from .types import Batch, Flows


def _resize(images: Tensor, shape, channels: int) -> Tensor:
    """images (items, h, w, channels) channels-last -> (items, h', w', channels)."""
    items, h, w = images.shape[:3]
    ho, wo = int(shape[0]), int(shape[1])
    out = torch.empty((items, ho, wo, channels), dtype=torch.float32, device=images.device)
    with torch.cuda.device(images.device):
        # the y grid dimension carries the items
        for lo in range(0, items, 65535):
            hi = min(items, lo + 65535)
            check(lib().fm_resize_bilinear(_ptr(images[lo:hi]), _ptr(out[lo:hi]), hi - lo, h, w, ho, wo,
                                           channels, _stream()), "fm_resize_bilinear")
    return out


def rescale_flow(flow: Tensor, shape) -> Tensor:
    """flow_predictor.py:40-48: (b, f, h, w, 2) -> (b, f, h', w', 2); normalised flow values are
    interpolated, not rescaled."""
    flow = _canon(flow, "flow")
    b, f, h, w, _ = flow.shape
    return _resize(flow.view(b * f, h, w, 2), shape, 2).view(b, f, int(shape[0]), int(shape[1]), 2)


def rescale_mask(mask: Tensor, shape) -> Tensor:
    """flow_predictor.py:50-58: (b, f, h, w) -> (b, f, h', w')."""
    mask = _canon(mask, "mask")
    b, f, h, w = mask.shape
    return _resize(mask.view(b * f, h, w, 1), shape, 1).view(b, f, int(shape[0]), int(shape[1]))


def compute_consistency_mask(videos: Tensor, flow: Tensor, reverse: bool = False) -> Tensor:
    """flow_predictor.py:60-82.  ``reverse=True`` gives the mask of a backward flow stored in the
    reference's order (pair i = frame i+1 -> frame i) without flipping the video."""
    videos = _canon(videos, "videos")
    flow = _canon(flow, "flow")
    b, f, c, h, w = videos.shape
    if c != 3 or flow.shape != (b, f - 1, h, w, 2):
        raise ValueError("flowmap_b200: consistency mask shape mismatch")
    mask = torch.empty((b, f - 1, h, w), dtype=torch.float32, device=videos.device)
    with torch.cuda.device(videos.device):
        if b * (f - 1) <= 65535:  # the y grid dimension carries the (batch, pair) items
            check(lib().fm_consistency_mask(_ptr(videos), _ptr(flow), _ptr(mask), b, f, h, w, int(reverse),
                                            _stream()), "fm_consistency_mask")
        else:  # very long / heavily batched videos: one batch element (and <= 65535 pairs) per launch
            for bi in range(b):
                for lo in range(0, f - 1, 65535):
                    hi = min(f - 1, lo + 65535)
                    check(lib().fm_consistency_mask(_ptr(videos[bi, lo:hi + 1]), _ptr(flow[bi, lo:hi]),
                                                    _ptr(mask[bi, lo:hi]), 1, hi - lo + 1, h, w, int(reverse),
                                                    _stream()), "fm_consistency_mask")
    return mask


def compute_bidirectional_flow(predict: Callable[[Tensor], Tensor], batch: Batch, flow_shape) -> Flows:
    """flow_predictor.py:84-101: forward flow of the video; backward flow = forward flow of the
    time-reversed video, flipped back; consistency masks at the predictor's resolution; everything
    rescaled to ``flow_shape``."""
    videos = batch.videos
    forward = predict(videos)
    forward_mask = rescale_mask(compute_consistency_mask(videos, forward), flow_shape)
    forward = rescale_flow(forward, flow_shape)
    backward = predict(videos.flip(dims=(1,))).flip(dims=(1,))  # pair i: frame i+1 -> frame i
    backward_mask = rescale_mask(compute_consistency_mask(videos, backward, reverse=True), flow_shape)
    backward = rescale_flow(backward, flow_shape)
    return Flows(forward, backward, forward_mask, backward_mask)


def resize_videos(videos: Tensor, shape) -> Tensor:
    """misc/cropping.py:19-27 resize_batch on (b, f, 3, h, w) planar frames."""
    videos = _canon(videos, "videos")
    b, f, c, h, w = videos.shape
    if c != 3:
        raise ValueError("flowmap_b200: videos must have 3 channels")
    # each colour plane is a one-channel image
    out = _resize(videos.view(b * f * c, h, w, 1), shape, 1)
    return out.view(b, f, c, int(shape[0]), int(shape[1]))
