"""flowmap_b200: H100-native (sm_90a) implementation of FlowMap's per-iteration
optimisation hot path behind the reference's Python surface.  See DESIGN.md."""
from .types import Batch, Flows, Tracks, BackboneOutput, ModelOutput, ModelExports  # noqa: F401

__all__ = ["Batch", "Flows", "Tracks", "BackboneOutput", "ModelOutput", "ModelExports", "install"]


def install() -> dict:
    """Swap the hot path of an importable reference checkout (`flowmap` on sys.path) for the
    CUDA implementation, under the reference's own names:

      * ``flowmap.model.model.Model``      -> flowmap_b200.model.Model (same cfg / forward)
      * ``flowmap.loss.LOSSES["flow"|"tracking"]`` -> flowmap_b200.loss.LossFlow / LossTracking
      * ``flowmap.model.intrinsics.INTRINSICS`` / ``flowmap.model.extrinsics.EXTRINSICS`` entries
        (``regressed`` / ``softmin`` / ``ground_truth``; ``procrustes`` / ``regressed``),
      * ``flowmap.model.projection.{sample_image_grid, unproject, project, reproject_points,
        compute_forward_flow, compute_backward_flow, get_extrinsics, align_surfaces}`` and
        ``flowmap.model.procrustes.align_rigid`` (module attributes; also re-bound in the reference
        modules that imported them by name: model.model, intrinsics.intrinsics_softmin, export.colmap,
        visualization.visualizer_summary when importable),
      * ``flowmap.flow.flow_predictor.FlowPredictor.rescale_flow / rescale_mask /
        compute_consistency_mask`` (static methods; the RAFT / GMFlow subclasses inherit them,
        so ``compute_bidirectional_flow`` runs on the kernels with the reference's predictor),
      * ``flowmap.export.colmap.export_to_colmap / write_colmap_model / read_colmap_model``
        (when that module imports; it needs ``plyfile``),
      * ``flowmap.misc.ate.compute_ate`` -> flowmap_b200.ate.compute_ate, also the copy in
        ``flowmap.visualization.visualizer_trajectory`` (when that module imports; it needs
        ``matplotlib``),

    so that ``flowmap/overfit.py`` (Hydra/Lightning harness) runs unchanged.  Call it before
    ``flowmap.overfit`` is imported.  Backbones that are outside the hot path (MiDaS) keep
    the reference's class.  Returns what was replaced (for logging / tests)."""
    import importlib

    from . import loss as my_loss
    from . import model as my_model

    replaced = {}
    ref_model = importlib.import_module("flowmap.model.model")
    replaced["flowmap.model.model.Model"] = ref_model.Model
    ref_model.Model = my_model.Model
    ref_loss = importlib.import_module("flowmap.loss")
    for key, cls in (("flow", my_loss.LossFlow), ("tracking", my_loss.LossTracking)):
        replaced[f"flowmap.loss.LOSSES[{key}]"] = ref_loss.LOSSES.get(key)
        ref_loss.LOSSES[key] = cls
    ref_intr = importlib.import_module("flowmap.model.intrinsics")
    for key, cls in my_model.INTRINSICS.items():
        replaced[f"flowmap.model.intrinsics.INTRINSICS[{key}]"] = ref_intr.INTRINSICS.get(key)
        ref_intr.INTRINSICS[key] = cls
    ref_extr = importlib.import_module("flowmap.model.extrinsics")
    for key, cls in my_model.EXTRINSICS.items():
        replaced[f"flowmap.model.extrinsics.EXTRINSICS[{key}]"] = ref_extr.EXTRINSICS.get(key)
        ref_extr.EXTRINSICS[key] = cls
    from . import procrustes as my_procrustes
    from . import projection as my_projection
    ref_proj = importlib.import_module("flowmap.model.projection")
    proj_names = ("sample_image_grid", "unproject", "project", "reproject_points", "compute_forward_flow",
                  "compute_backward_flow", "get_extrinsics", "align_surfaces")
    users = [ref_proj]
    for mod in ("flowmap.model.model", "flowmap.model.intrinsics.intrinsics_softmin", "flowmap.export.colmap",
                "flowmap.visualization.visualizer_summary", "flowmap.model.extrinsics.extrinsics_regressed"):
        try:
            users.append(importlib.import_module(mod))
        except ImportError:
            pass
    for name in proj_names:
        replaced[f"flowmap.model.projection.{name}"] = getattr(ref_proj, name)
        for mod in users:  # `from ..projection import name` made a copy of the binding there
            if mod is ref_proj or hasattr(mod, name):
                setattr(mod, name, getattr(my_projection, name))
    ref_procrustes = importlib.import_module("flowmap.model.procrustes")
    replaced["flowmap.model.procrustes.align_rigid"] = ref_procrustes.align_rigid
    ref_procrustes.align_rigid = my_procrustes.align_rigid
    from . import export as my_export
    from . import flow as my_flow
    try:
        ref_flow = importlib.import_module("flowmap.flow.flow_predictor")
        for name in ("rescale_flow", "rescale_mask", "compute_consistency_mask"):
            replaced[f"flowmap.flow.flow_predictor.FlowPredictor.{name}"] = getattr(ref_flow.FlowPredictor, name)
            setattr(ref_flow.FlowPredictor, name, staticmethod(getattr(my_flow, name)))
    except ImportError:  # torchvision-less environments: the flow side stays with the caller
        pass
    try:
        ref_colmap = importlib.import_module("flowmap.export.colmap")
        for name in ("export_to_colmap", "write_colmap_model", "read_colmap_model"):
            replaced[f"flowmap.export.colmap.{name}"] = getattr(ref_colmap, name)
            setattr(ref_colmap, name, getattr(my_export, name))
    except ImportError:
        pass
    from . import ate as my_ate
    # misc.ate and the copy visualization.visualizer_trajectory imported by name (that module needs
    # matplotlib)
    for mod in ("flowmap.misc.ate", "flowmap.visualization.visualizer_trajectory"):
        try:
            ref = importlib.import_module(mod)
        except ImportError:
            continue
        replaced[f"{mod}.compute_ate"] = ref.compute_ate
        ref.compute_ate = my_ate.compute_ate
    ref_back = importlib.import_module("flowmap.model.backbone")
    for key, cls in ref_back.BACKBONES.items():  # e.g. midas: produced by the reference
        my_model.BACKBONES.setdefault(key, cls)
    return replaced
