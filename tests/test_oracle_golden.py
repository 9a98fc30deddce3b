"""Pins oracle/flowmap_oracle.py against outputs of the unmodified reference
(tests/golden/*.npz, produced by tests/golden/make_golden.py).  CPU only."""
import numpy as np
import pytest
import torch

from conftest import load_golden, max_abs, rel_l2
from oracle import flowmap_oracle as O

T = torch.as_tensor


@pytest.mark.parametrize("f64", [False, True])
def test_units(f64):
    g = load_golden("units", f64)
    dt = torch.float64 if f64 else torch.float32
    tol = 1e-12 if f64 else 2e-6
    h, w = g["grid_xy"].shape[:2]
    assert max_abs(O.pixel_grid(h, w, dt), g["grid_xy"]) <= tol
    k3 = O.intrinsics_from_focal(T(g["focals"]), h, w)
    assert max_abs(k3, g["k3"]) <= tol
    xy = O.pixel_grid(h, w, dt)
    surf = O.unproject(xy, T(g["z"]), T(g["k3"])[:, None, None])
    assert max_abs(surf, g["surfaces"]) <= tol * 10
    proj = O.project_camera_space(T(g["proj_pts"]), T(g["proj_k"]))
    assert np.allclose(proj.numpy(), g["proj_xy"], rtol=1e-5 if not f64 else 1e-12, atol=tol)
    rig = O.align_rigid(T(g["rigid_p"]), T(g["rigid_q"]), T(g["rigid_w"]))
    assert max_abs(rig, g["rigid_t"]) <= (1e-10 if f64 else 5e-6)
    assert max_abs(O.pose_chain(T(g["rigid_t"])[None]), g["chain"]) <= (1e-12 if f64 else 2e-6)
    for m in ("huber", "l1", "l2"):
        out = O.robust_map(T(g["map_a"]), T(g["map_b"]), h, w, m, 0.01)
        assert max_abs(out, g[f"map_{m}"]) <= tol
    assert max_abs(O.aspect_correct(T(g["map_a"]), h, w), g["aspect"]) <= tol
    for fn in (O.bilinear_border, O.bilinear_border_explicit):
        assert max_abs(fn(T(g["samp_img"]), T(g["samp_xy"])), g["samp_out"]) <= tol * 5


def _state_from(g, dt, cfg):
    f, h, w = g["in_depth"].shape
    st = O.OverfitOracle(cfg, f, h, w, dtype=dt)
    with torch.no_grad():
        st.depth.copy_(T(g["in_depth"]).to(dt))
        st.weights.copy_(T(g["in_wparam"]).to(dt))
    flows = O.Flows(*(T(g[k]).to(dt) for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    return st, flows


CASES = [
    ("flow_huber", dict()),
    ("flow_l1", dict(mapping="l1")),
    ("flow_l2", dict(mapping="l2")),
    ("flow_pts1000", dict(procrustes_points=1000)),
    ("flow_rough", dict(initial_focal=1.3)),
]


@pytest.mark.parametrize("name,kw", CASES)
@pytest.mark.parametrize("f64", [False, True])
def test_flow_step(name, kw, f64):
    g = load_golden(name, f64)
    dt = torch.float64 if f64 else torch.float32
    cfg = O.OverfitConfig(intrinsics="regressed", **kw)
    st, flows = _state_from(g, dt, cfg)
    r = st.training_step(flows)
    lt, gt, et = (1e-11, 1e-8, 1e-11) if f64 else (2e-5, 2e-3, 2e-5)
    assert abs(r["loss"] - float(g["loss"])) <= lt * abs(float(g["loss"]))
    assert max_abs(r["extrinsics"], g["extrinsics"]) <= et
    assert max_abs(r["intrinsics"], g["intrinsics"]) <= et
    assert rel_l2(r["grads"]["depth"], g["g_depth"]) <= gt
    assert rel_l2(r["grads"]["weights"], g["g_wparam"]) <= gt
    assert abs(float(r["grads"]["focal"]) - float(g["g_focal"])) <= gt * abs(float(g["g_focal"]))


@pytest.mark.parametrize("f64", [False, True])
def test_ground_truth_intrinsics(f64):
    """OverfitOracle with intrinsics="ground_truth" against the reference's Model with
    IntrinsicsGroundTruth on a K per frame (fx x1.5, fy x1.4 over the video, principal point drifting
    from (0.3, 0.7) to (0.7, 0.3)), flow + tracking loss: poses, loss parts, gradients, the induced flow
    positions (K of the later / earlier frame) and the track targets of a segment that starts at frame 2.
    Then the projection unit under the same K: unproject, project (incl. the nan_to_num branch) and
    reproject_points."""
    g = load_golden("gt_intrinsics", f64)
    dt = torch.float64 if f64 else torch.float32
    f, h, w = g["in_depth"].shape
    st = O.OverfitOracle(O.OverfitConfig(intrinsics="ground_truth", use_tracking=True, tracking_enable_after=0),
                         f, h, w, dtype=dt, intrinsics=T(g["intrinsics"]))
    with torch.no_grad():
        st.depth.copy_(T(g["in_depth"]).to(dt))
        st.weights.copy_(T(g["in_wparam"]).to(dt))
    flows = O.Flows(*(T(g[k]).to(dt) for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    tracks = [O.Tracks(T(g[f"trk{i}_xy"]).to(dt), T(g[f"trk{i}_vis"]), int(g[f"trk{i}_start"])) for i in range(2)]
    tol = 1e-11 if f64 else 2e-5
    out = st.forward(flows, 0)
    assert max_abs(out.extrinsics.detach(), g["extrinsics"]) <= tol
    # the first two pairs, as stored
    fwd = O.forward_flow_positions(out.surfaces, out.extrinsics, out.intrinsics).detach()
    bwd = O.backward_flow_positions(out.surfaces, out.extrinsics, out.intrinsics).detach()
    assert max_abs(fwd[:, :2], g["fwd_xy"]) <= tol
    assert max_abs(bwd[:, :2], g["bwd_xy"]) <= tol
    tgt, valid = O.track_positions(out.surfaces[:, 2:6], out.extrinsics[:, 2:6], out.intrinsics[:, 2:6], tracks[1])
    assert bool((valid.numpy() == g["trk1_valid"]).all())
    v = T(g["trk1_valid"])
    assert max_abs(tgt.detach()[v], T(g["trk1_target"])[v]) <= (1e-10 if f64 else 1e-4)
    r = st.training_step(flows, tracks)
    lt, gt = (1e-10, 1e-7) if f64 else (5e-5, 5e-3)
    assert abs(r["loss"] - float(g["loss"])) <= lt * abs(float(g["loss"]))
    assert abs(r["parts"]["flow"] - float(g["loss_flow"])) <= lt * abs(float(g["loss_flow"]))
    assert abs(r["parts"]["tracking"] - float(g["loss_tracking"])) <= lt * abs(float(g["loss_tracking"]))
    assert rel_l2(r["grads"]["depth"], g["g_depth"]) <= gt
    assert rel_l2(r["grads"]["weights"], g["g_wparam"]) <= gt
    assert r["grads"]["focal"] is None

    k = T(g["intrinsics"]).to(dt)
    surf = O.unproject(O.pixel_grid(h, w, dt), T(g["unit_z"]), k[:, :, None, None])
    assert max_abs(surf, g["unit_surfaces"]) <= tol * 10
    cam = T(g["unit_cam"])
    xy = O.project_camera_space(cam, k[:, :, None])  # identity extrinsics: world = camera space
    assert np.allclose(xy.numpy(), g["unit_proj_xy"], rtol=1e-5 if not f64 else 1e-12, atol=tol)
    assert bool(((cam[..., 2] >= 0).numpy() == g["unit_proj_front"]).all())
    rxy = O.reproject(cam, T(g["unit_rel"])[:, :, None], k[:, :, None])
    # float32: a moved point 1e-3 in front of the camera plane amplifies rounding of the transform by 1e3
    assert np.allclose(rxy.numpy(), g["unit_reproj_xy"], rtol=1e-4 if not f64 else 1e-12, atol=tol)


@pytest.mark.parametrize("f64", [False, True])
def test_flow_positions(f64):
    g = load_golden("flow_huber", f64)
    dt = torch.float64 if f64 else torch.float32
    st, flows = _state_from(g, dt, O.OverfitConfig(intrinsics="regressed"))
    out = st.forward(flows, 0)
    tol = 1e-11 if f64 else 2e-5
    fwd = O.forward_flow_positions(out.surfaces, out.extrinsics, out.intrinsics)
    bwd = O.backward_flow_positions(out.surfaces, out.extrinsics, out.intrinsics)
    assert max_abs(fwd[:, :2], g["fwd_xy"]) <= tol
    assert max_abs(bwd[:, :2], g["bwd_xy"]) <= tol
    assert max_abs(out.backward_correspondence_weights, g["weights"]) <= tol


@pytest.mark.parametrize("f64", [False, True])
def test_softmin(f64):
    g = load_golden("softmin", f64)
    dt = torch.float64 if f64 else torch.float32
    cfg = O.OverfitConfig(intrinsics="softmin", softmin_points=300, regression_after=None)
    st, flows = _state_from(g, dt, cfg)
    r = st.training_step(flows, softmin_indices=T(g["indices"]))
    lt, gt, et = (1e-10, 1e-7, 1e-10) if f64 else (5e-5, 5e-3, 5e-5)
    assert abs(r["loss"] - float(g["loss"])) <= lt * abs(float(g["loss"]))
    assert max_abs(r["intrinsics"], g["intrinsics"]) <= et
    assert max_abs(r["extrinsics"], g["extrinsics"]) <= et
    assert rel_l2(r["grads"]["depth"], g["g_depth"]) <= gt
    assert rel_l2(r["grads"]["weights"], g["g_wparam"]) <= gt


@pytest.mark.parametrize("f64", [False, True])
def test_tracking(f64):
    g = load_golden("tracking", f64)
    dt = torch.float64 if f64 else torch.float32
    cfg = O.OverfitConfig(intrinsics="regressed", use_tracking=True, tracking_enable_after=0)
    st, flows = _state_from(g, dt, cfg)
    tracks = [O.Tracks(T(g[f"trk{i}_xy"]).to(dt), T(g[f"trk{i}_vis"]), int(g[f"trk{i}_start"]))
              for i in range(2)]
    out = st.forward(flows, 0)
    tgt, valid = O.track_positions(out.surfaces[:, :6], out.extrinsics[:, :6],
                                   out.intrinsics[:, :6], tracks[0])
    assert bool((valid.numpy() == g["trk0_valid"]).all())
    v = T(g["trk0_valid"])
    assert max_abs(tgt[v], T(g["trk0_target"])[v]) <= (1e-10 if f64 else 1e-4)
    r = st.training_step(flows, tracks)
    lt, gt = (1e-10, 1e-7) if f64 else (5e-5, 5e-3)
    assert abs(r["parts"]["flow"] - float(g["loss_flow"])) <= lt * abs(float(g["loss_flow"]))
    assert abs(r["parts"]["tracking"] - float(g["loss_tracking"])) <= lt * abs(float(g["loss_tracking"]))
    assert rel_l2(r["grads"]["depth"], g["g_depth"]) <= gt
    assert rel_l2(r["grads"]["weights"], g["g_wparam"]) <= gt
    assert abs(float(r["grads"]["focal"]) - float(g["g_focal"])) <= gt * abs(float(g["g_focal"]))


@pytest.mark.parametrize("name", ["traj_generic", "traj_init"])
@pytest.mark.parametrize("f64", [False, True])
def test_trajectory(name, f64):
    g = load_golden(name, f64)
    dt = torch.float64 if f64 else torch.float32
    st, flows = _state_from(g, dt, O.OverfitConfig(intrinsics="regressed"))
    steps = len(g["loss"])
    for s in range(steps):
        r = st.training_step(flows)
        tol = 1e-9 if f64 else 1e-3
        assert abs(r["loss"] - g["loss"][s]) <= tol * abs(g["loss"][s]), s
        assert max_abs(r["extrinsics"], g["extrinsics"][s]) <= (1e-9 if f64 else 1e-3), s
    assert rel_l2(st.depth, g["depth_final"]) <= (1e-10 if f64 else 1e-5)
    assert rel_l2(st.weights, g["wparam_final"]) <= (1e-8 if f64 else 1e-2)
