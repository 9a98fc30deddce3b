"""ctypes binding of csrc/libflowmap_b200.so (the C ABI declared in include/flowmap_b200.h).

There is deliberately no fallback: if the shared library is missing or a call fails, the
caller gets an exception.  The library is built in-tree by ``flowmap_b200.build.build()``
(``nvcc -gencode arch=compute_90a,code=sm_90a``), see ``__graft_entry__.build``.
"""
from __future__ import annotations

import ctypes
from ctypes import c_double, c_float, c_int, c_size_t, c_void_p
from pathlib import Path

CSRC = Path(__file__).resolve().parent / "csrc"
SO_PATH = CSRC / "libflowmap_b200.so"

_lib = None

# name -> (restype, argtypes); must list every symbol of include/flowmap_b200.h
_P = c_void_p
SIGNATURES = {
    "fm_version": (c_int, []),
    "fm_last_error": (ctypes.c_char_p, []),
    "fm_launch_count": (ctypes.c_ulonglong, []),
    "fm_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "fm_workspace_reset": (c_int, [_P, c_int, c_int, c_int, c_int, _P]),
    "fm_unproject": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    "fm_unproject_bwd": (c_int, [_P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    "fm_reproject": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, _P]),
    "fm_unproject_points": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, _P]),
    "fm_unproject_points_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, _P]),
    "fm_points_workspace_bytes": (c_size_t, [c_int]),
    "fm_align_rigid_fwd": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, _P]),
    "fm_align_rigid_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, _P]),
    "fm_procrustes_fwd": (c_int, [_P, _P, _P, _P, _P, c_int, _P, _P, c_int, c_int, c_int, c_int, _P]),
    "fm_procrustes_bwd": (c_int, [_P, _P, _P, _P, _P, c_int, _P, c_int, _P, _P, _P, _P, _P,
                                  c_int, c_int, c_int, c_int, _P]),
    "fm_procrustes_moments": (c_int, [_P, _P, _P, _P, c_float, _P, c_int, c_int, c_int, _P]),
    "fm_mask_sum": (c_int, [_P, _P, _P, c_size_t, _P]),
    "fm_flow_loss_fwd_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, c_int, c_float, c_float, c_int,
                                     _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    "fm_pose_chain": (c_int, [_P, _P, c_int, c_int, _P]),
    "fm_pose_chain_bwd": (c_int, [_P, _P, _P, _P, c_int, c_int, _P]),
    "fm_trajectory_ate": (c_int, [_P, _P, c_int, c_int, _P, _P, _P, _P, _P]),
    "fm_track_workspace_bytes": (c_size_t, [c_int, ctypes.c_longlong]),
    "fm_track_loss_fwd": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, _P, _P, ctypes.c_longlong,
                                  c_int, c_float, c_float, _P, _P, c_int, c_int, c_int, _P]),
    "fm_track_loss_bwd": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, _P, _P, ctypes.c_longlong,
                                  c_int, c_float, c_float, _P, _P, _P, _P, _P, c_int, c_int, c_int,
                                  _P]),
    "fm_track_reduce_bytes": (c_size_t, [c_int]),
    "fm_track_loss_fwd_sharded": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, _P, _P, ctypes.c_longlong,
                                          c_int, c_float, c_float, _P, _P, c_int, c_int, c_int, c_int, c_int,
                                          c_int, c_int, _P]),
    "fm_track_loss_fwd_const_k": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, _P, _P, ctypes.c_longlong,
                                          c_int, c_float, c_float, _P, _P, c_int, c_int, c_int, c_int, c_int,
                                          c_int, _P]),
    "fm_track_loss_value": (c_int, [_P, c_float, _P, _P]),
    "fm_track_loss_bwd_sharded": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, _P, _P, ctypes.c_longlong,
                                          c_int, c_float, c_float, _P, _P, _P, _P, _P, c_int, c_int, c_int,
                                          c_int, c_int, c_int, _P]),
    "fm_random_subset": (c_int, [ctypes.c_ulonglong, ctypes.c_longlong, c_int, _P, _P]),
    "fm_softmin_workspace_bytes": (c_size_t, [c_int, c_int]),
    "fm_softmin_sweep_fwd": (c_int, [_P, _P, c_float, _P, _P, c_int, _P, c_int, _P, _P, _P, c_int, c_int,
                                     c_int, c_int, _P]),
    "fm_softmin_sweep_bwd": (c_int, [_P, _P, c_float, _P, _P, c_int, _P, c_int, _P, _P, _P, _P, _P,
                                     c_int, c_int, c_int, c_int, _P]),
    "fm_softmin_focal": (c_int, [_P, _P, c_int, c_int, _P, _P, _P]),
    "fm_softmin_focal_bwd": (c_int, [_P, _P, _P, _P, c_int, c_int, _P, _P]),
    "fm_consistency_mask": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "fm_resize_bilinear": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "fm_world_points": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, _P]),
    "fm_adam_step": (c_int, [_P, _P, _P, _P, c_size_t, c_double, c_double, c_double, c_double,
                             c_int, _P]),
    "fm_step_clock_tick": (c_int, [_P, c_double, c_double, c_double, ctypes.c_ulonglong, c_int, _P]),
    "fm_adam_step_clock": (c_int, [_P, _P, _P, _P, c_size_t, _P, c_int, c_double, c_double, c_double, _P]),
    "fm_random_subset_clock": (c_int, [_P, ctypes.c_longlong, c_int, _P, _P]),
}


class PackedTracksC(ctypes.Structure):
    """fm_packed_tracks"""
    _fields_ = [("segments", _P), ("xy", _P), ("vis", _P), ("num_segments", c_int),
                ("max_rows", c_int), ("max_points", c_int), ("total_samples", ctypes.c_longlong)]


class OverfitStepArgs(ctypes.Structure):
    """fm_overfit_step_args (field order as in include/flowmap_b200.h)"""
    _fields_ = [("F", c_int), ("H", c_int), ("W", c_int),
                ("depth", _P), ("weight_logits", _P), ("weight_sensitivity", c_float),
                ("focal", _P), ("k4", _P), ("indices", _P), ("num_indices", c_int),
                ("fflow", _P), ("bflow", _P), ("fmask", _P), ("bmask", _P), ("mask_sum", _P),
                ("mapping", c_int), ("delta", c_float), ("flow_weight", c_float),
                ("tracks", ctypes.POINTER(PackedTracksC)), ("track_weight", c_float),
                ("m_depth", _P), ("v_depth", _P), ("m_weights", _P), ("v_weights", _P),
                ("m_focal", _P), ("v_focal", _P),
                ("beta1", c_double), ("beta2", c_double), ("eps", c_double),
                ("step", c_int),
                ("g_depth", _P), ("g_weights", _P), ("g_focal", _P), ("g_k4", _P),
                ("rt", _P), ("loss", _P),
                ("extrinsics", _P), ("g_extrinsics", _P), ("g_rt", _P), ("track_g_k4", _P),
                ("track_loss", _P),
                ("ws", _P), ("track_ws", _P), ("defer_adam", c_int),
                ("phase", c_int),
                ("flow_grad_scale", _P), ("track_grad_scale", _P), ("clock", _P), ("moments_k4", _P),
                ("gt_positions", _P), ("gt_fx", c_float), ("gt_fy", c_float), ("metrics_log", _P),
                ("metrics_capacity", c_int), ("video_grad_scales", c_int), ("B", c_int), ("gt_fxfy", _P)]


class VideoLayout(ctypes.Structure):
    """fm_video_layout: videos of different lengths packed along the frame axis (device tables)"""
    _fields_ = [("B", c_int), ("T", c_int), ("frame_offset", _P), ("frame_video", _P), ("pair_video", _P)]


_L = ctypes.POINTER(VideoLayout)
SIGNATURES["fm_overfit_step"] = (c_int, [ctypes.POINTER(OverfitStepArgs), _P])
SIGNATURES.update({
    "fm_overfit_step_videos": (c_int, [ctypes.POINTER(OverfitStepArgs), _L, _P]),
    "fm_workspace_bytes_videos": (c_size_t, [c_int, c_int]),
    "fm_procrustes_moments_videos": (c_int, [_P, _P, _P, _P, c_float, _P, _L, c_int, c_int, _P]),
    "fm_softmin_sweep_fwd_videos": (c_int, [_P, _P, c_float, _P, _P, c_int, _P, c_int, _P, _P, _P, _L, c_int,
                                            c_int, _P]),
    "fm_softmin_sweep_bwd_videos": (c_int, [_P, _P, c_float, _P, _P, c_int, _P, c_int, _P, _P, _P, _P, _P, _L,
                                            c_int, c_int, _P]),
    "fm_adam_step_clock_frames_videos": (c_int, [_P, _P, _P, _P, c_size_t, _L, c_int, c_int, c_int, _P, c_int,
                                                 c_double, c_double, c_double, _P]),
    "fm_pose_chain_videos": (c_int, [_P, _P, _L, _P]),
    "fm_pose_chain_bwd_videos": (c_int, [_P, _P, _P, _P, _L, _P]),
})


class FlowmapLibraryError(RuntimeError):
    pass


def load_library(path) -> ctypes.CDLL:
    """dlopen one build of the library and type every entry point of include/flowmap_b200.h."""
    handle = ctypes.CDLL(str(path))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(handle, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    return handle


def lib() -> ctypes.CDLL:
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not SO_PATH.exists():
            raise FlowmapLibraryError(
                f"{SO_PATH} not found: build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` (nvcc, sm_90a).  flowmap_b200 has no CPU or PyTorch fallback.")
        _lib = load_library(SO_PATH)
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().fm_last_error().decode("utf-8", "replace")
        raise FlowmapLibraryError(f"{what or 'flowmap_b200'} failed ({rc}): {msg}")
