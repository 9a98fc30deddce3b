"""The C-ABI library loads on a CPU-only box and exports every symbol the header declares."""
import ctypes
import re

from conftest import ROOT


def declared_symbols():
    text = (ROOT / "include" / "flowmap_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(fm_[a-z0-9_]+)\s*\(", text)))


def test_library_builds_and_exports_header_symbols():
    from flowmap_b200.build import build
    from flowmap_b200 import _lib
    so = build()
    handle = ctypes.CDLL(str(so))
    names = declared_symbols()
    assert len(names) >= 10
    for name in names:
        assert hasattr(handle, name), f"{name} declared in the header but not exported"
        assert name in _lib.SIGNATURES, f"{name} has no ctypes signature"
    assert set(_lib.SIGNATURES) == set(names)
    assert _lib.lib().fm_version() >= 100
    # pure host-side query works without a GPU
    assert _lib.lib().fm_workspace_bytes(1, 150, 360, 640) > 0
    assert _lib.lib().fm_workspace_bytes(1, 1, 8, 8) == 0


def test_product_has_no_cpu_path():
    import pytest
    import torch
    from flowmap_b200 import ops
    d = torch.zeros(1, 2, 4, 4)
    with pytest.raises(ValueError, match="CUDA"):
        ops.procrustes_poses(d, None, torch.zeros(1, 2, 4), torch.zeros(1, 1, 4, 4, 2))


def test_package_does_not_import_oracle():
    import subprocess, sys
    code = ("import sys, flowmap_b200, flowmap_b200.model, flowmap_b200.loss, flowmap_b200.overfit;"
            "bad=[m for m in sys.modules if m.startswith('oracle')]; assert not bad, bad")
    subprocess.check_call([sys.executable, "-c", code], cwd=str(ROOT))


# Stand-in for the reference's `flowmap` package: the modules, registries and names that
# install() rebinds, with placeholder values (the reference itself is not part of this repository).
_REFERENCE_STANDIN = """
import sys, types

def module(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m

class Placeholder:
    def __init__(self, *args, **kwargs):
        pass

def placeholder(*args, **kwargs):
    raise AssertionError("reference placeholder called")

PROJECTION = ("sample_image_grid", "unproject", "project", "reproject_points", "compute_forward_flow",
              "compute_backward_flow", "get_extrinsics", "align_surfaces")
module("flowmap")
module("flowmap.model")
module("flowmap.model.model", Model=Placeholder, **{n: placeholder for n in PROJECTION[:2]})
losses = {"flow": Placeholder, "tracking": Placeholder}
module("flowmap.loss", LOSSES=losses, get_losses=lambda cfgs: [losses[c.name](c) for c in cfgs])
module("flowmap.model.intrinsics", INTRINSICS={"regressed": Placeholder, "softmin": Placeholder,
                                               "ground_truth": Placeholder})
module("flowmap.model.extrinsics", EXTRINSICS={"procrustes": Placeholder, "regressed": Placeholder})
module("flowmap.model.projection", **{n: placeholder for n in PROJECTION})
module("flowmap.model.procrustes", align_rigid=placeholder)
module("flowmap.model.backbone", BACKBONES={"explicit_depth": Placeholder, "midas": Placeholder})
module("flowmap.flow")
FlowPredictor = type("FlowPredictor", (), {n: staticmethod(placeholder) for n in
                                            ("rescale_flow", "rescale_mask", "compute_consistency_mask")})
module("flowmap.flow.flow_predictor", FlowPredictor=FlowPredictor)
module("flowmap.export")
module("flowmap.export.colmap", **{n: placeholder for n in
                                   ("export_to_colmap", "write_colmap_model", "read_colmap_model")})
"""


def test_install_patches_reference_registries():
    """flowmap_b200.install() rebinds every registry entry and module attribute of the reference's
    `flowmap` package (a stand-in with the same module layout), and the patched registries build
    this package's classes from cfg objects."""
    import sys
    code = _REFERENCE_STANDIN + (
        "import flowmap.model.model as rm, flowmap.loss as rl, flowmap.model.intrinsics as ri\n"
        "import flowmap.model.extrinsics as re, flowmap.model.projection as rp, flowmap.model.procrustes as rpr\n"
        "import flowmap.model.backbone as rb, flowmap.export.colmap as rc\n"
        "import flowmap_b200\n"
        "rep = flowmap_b200.install()\n"
        "from flowmap_b200 import export as ex, flow as fl, model as mm, procrustes as pr, projection as pj\n"
        "from flowmap_b200.model import Model\nfrom flowmap_b200.loss import LossFlow, LossTracking\n"
        "assert rm.Model is Model and rl.LOSSES['flow'] is LossFlow and rl.LOSSES['tracking'] is LossTracking\n"
        "assert ri.INTRINSICS == mm.INTRINSICS and re.EXTRINSICS == mm.EXTRINSICS\n"
        "for n in PROJECTION:\n"
        "    assert getattr(rp, n) is getattr(pj, n), n\n"
        "assert rm.sample_image_grid is pj.sample_image_grid and rm.unproject is pj.unproject\n"
        "assert rpr.align_rigid is pr.align_rigid\n"
        "assert rb.BACKBONES['explicit_depth'] is Placeholder and mm.BACKBONES['midas'] is Placeholder\n"
        "assert mm.BACKBONES['explicit_depth'] is mm.BackboneExplicitDepth\n"
        "for n in ('export_to_colmap', 'write_colmap_model', 'read_colmap_model'):\n"
        "    assert getattr(rc, n) is getattr(ex, n), n\n"
        "from flowmap_b200.model import BackboneExplicitDepthCfg, ExtrinsicsProcrustesCfg, IntrinsicsSoftminCfg, ModelCfg, RegressionCfg\n"
        "cfg = ModelCfg(BackboneExplicitDepthCfg('explicit_depth', 0.1, 100.0), IntrinsicsSoftminCfg('softmin', 8192, 0.5, 2.0, 60, RegressionCfg(1000, 100)), ExtrinsicsProcrustesCfg('procrustes', None, False), True)\n"
        "m = rm.Model(cfg, 4, (8, 12))\n"
        "names = sorted(n for n, _ in m.named_parameters())\n"
        "assert names == ['backbone.depth', 'backbone.weights', 'intrinsics.intrinsics_regressed.focal_length'], names\n"
        "from flowmap_b200.loss import LossFlowCfg, MappingHuberCfg\n"
        "l = rl.get_losses([LossFlowCfg(0, 1000.0, 'flow', MappingHuberCfg('huber', 0.01))])\n"
        "assert type(l[0]) is LossFlow\n"
        "assert FlowPredictor.rescale_flow is fl.rescale_flow and FlowPredictor.compute_consistency_mask is fl.compute_consistency_mask\n"
        "assert 'flowmap.flow.flow_predictor.FlowPredictor.rescale_mask' in rep\n")
    import subprocess
    from conftest import ROOT
    subprocess.check_call([sys.executable, "-c", code], cwd=str(ROOT))
