"""GPU parity tests: the CUDA path (through the C ABI) against the golden vectors of the
reference and against the oracle.  Tolerances: north_star asks for 1e-4 relative on
poses / intrinsics / depth / loss; gradients are compared against the float64 run of the
reference and must be no worse than max(1e-4, 3x the reference's own float32 error)."""
import numpy as np
import pytest
import torch

from conftest import load_golden, max_abs, rel_l2

pytestmark = pytest.mark.gpu

T = torch.as_tensor


def _setup(g, mapping="huber", focal=0.85, npts=None, cfg_kw=None):
    from flowmap_b200.overfit import OverfitCfg, Overfitter
    from flowmap_b200.types import Batch, Flows
    f, h, w = g["in_depth"].shape
    cfg = OverfitCfg(mapping=mapping, initial_focal=focal, procrustes_points=npts,
                     **(cfg_kw or {}))
    batch = Batch(torch.zeros(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    flows = Flows(*(T(g[k]).float() for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    o = Overfitter(cfg, batch, flows)
    with torch.no_grad():
        o.model.backbone.depth.copy_(T(g["in_depth"]).float())
        o.model.backbone.weights.copy_(T(g["in_wparam"]).float())
    return o


CASES = [("flow_huber", "huber", 0.85, None), ("flow_l1", "l1", 0.85, None),
         ("flow_l2", "l2", 0.85, None), ("flow_rough", "huber", 1.3, None),
         ("flow_pts1000", "huber", 0.85, 1000)]


@pytest.mark.parametrize("name,mapping,focal,npts", CASES)
def test_step_matches_reference_golden(name, mapping, focal, npts):
    g64, g32 = load_golden(name, True), load_golden(name, False)
    o = _setup(g64, mapping, focal, npts)
    out = o.model(o.batch, o.flows, 0)
    loss = o.losses[0].forward(o.batch, o.flows, None, out, 0)
    loss.backward()
    torch.cuda.synchronize()
    assert abs(float(loss) - float(g64["loss"])) <= 1e-4 * abs(float(g64["loss"]))
    assert max_abs(out.extrinsics.cpu(), g64["extrinsics"]) <= 1e-5
    assert max_abs(out.intrinsics.cpu(), g64["intrinsics"]) <= 1e-6
    gd, gw = o.model.backbone.depth.grad.cpu(), o.model.backbone.weights.grad.cpu()
    gf = float(o.model.intrinsics.focal_length.grad)
    assert rel_l2(gd, g64["g_depth"]) <= max(1e-4, 3 * rel_l2(g32["g_depth"], g64["g_depth"]))
    assert rel_l2(gw, g64["g_wparam"]) <= max(1e-4, 3 * rel_l2(g32["g_wparam"], g64["g_wparam"]))
    assert abs(gf - float(g64["g_focal"])) <= 1e-4 * abs(float(g64["g_focal"]))


@pytest.mark.parametrize("name", ["traj_generic", "traj_init"])
def test_adam_trajectory_matches_reference(name):
    g64 = load_golden(name, True)
    o = _setup(g64)
    steps = len(g64["loss"])
    for s in range(steps):
        total, out = o.training_step()
        assert abs(float(total) - g64["loss"][s]) <= 1e-4 * abs(g64["loss"][s]), s
        assert max_abs(out.extrinsics.cpu(), g64["extrinsics"][s]) <= 1e-4, s
    assert rel_l2(o.model.backbone.depth.detach().cpu(), g64["depth_final"]) <= 1e-5
    # 6 Adam steps of lr 3e-5 from |w| ~ 1e-2: compare the update, not just the value
    w0, w1 = T(g64["in_wparam"]), T(g64["wparam_final"])
    upd = o.model.backbone.weights.detach().cpu().double() - w0
    assert rel_l2(upd, w1 - w0) <= 2e-2


def test_matches_oracle_c1_shape():
    """configs[0] shape (8 x 128 x 128, random flow): loss, poses and every gradient vs the
    float64 oracle on the same seeded inputs."""
    from oracle import flowmap_oracle as O
    f, h, w = 8, 128, 128
    flows64 = O.synthetic_flows(f, h, w, seed=0, dtype=torch.float64)
    gen = torch.Generator().manual_seed(5)
    depth = (1.0 + torch.rand(f, h, w, generator=gen, dtype=torch.float64))
    wparam = 0.01 * torch.randn(f - 1, h, w, generator=gen, dtype=torch.float64)
    st = O.OverfitOracle(O.OverfitConfig(intrinsics="regressed"), f, h, w, dtype=torch.float64)
    with torch.no_grad():
        st.depth.copy_(depth)
        st.weights.copy_(wparam)
    ref = st.training_step(flows64)
    g = {"in_depth": depth.numpy(), "in_wparam": wparam.numpy(), "in_fwd": flows64.forward.numpy(),
         "in_bwd": flows64.backward.numpy(), "in_fmask": flows64.forward_mask.numpy(),
         "in_bmask": flows64.backward_mask.numpy()}
    o = _setup(g)
    out = o.model(o.batch, o.flows, 0)
    loss = o.losses[0].forward(o.batch, o.flows, None, out, 0)
    loss.backward()
    assert abs(float(loss) - ref["loss"]) <= 1e-4 * abs(ref["loss"])
    assert max_abs(out.extrinsics.cpu(), ref["extrinsics"]) <= 1e-5
    assert rel_l2(o.model.backbone.depth.grad.cpu(), ref["grads"]["depth"]) <= 1e-4
    assert rel_l2(o.model.backbone.weights.grad.cpu(), ref["grads"]["weights"]) <= 1e-4
    assert abs(float(o.model.intrinsics.focal_length.grad) - float(ref["grads"]["focal"])) <= \
        1e-4 * abs(float(ref["grads"]["focal"]))


def test_pair_locality_at_full_size():
    """Size-independent property at the BASELINE shape (150 x 360 x 640): the flow loss is
    pair-local (SURVEY A.6), so the un-normalised loss and the gradients of a 3-frame
    sub-video equal the corresponding slice of the full problem."""
    from oracle import flowmap_oracle as O
    f, h, w = 150, 360, 640
    flows = O.synthetic_flows(f, h, w, seed=0)
    gen = torch.Generator().manual_seed(9)
    depth = 0.1 + 0.05 * torch.rand(f, h, w, generator=gen)
    wparam = 0.01 * torch.randn(f - 1, h, w, generator=gen)
    g = {"in_depth": depth.numpy(), "in_wparam": wparam.numpy(), "in_fwd": flows.forward.numpy(),
         "in_bwd": flows.backward.numpy(), "in_fmask": flows.forward_mask.numpy(),
         "in_bmask": flows.backward_mask.numpy()}
    o = _setup(g)
    out = o.model(o.batch, o.flows, 0)
    loss = o.losses[0].forward(o.batch, o.flows, None, out, 0)
    loss.backward()
    den_full = float(flows.forward_mask.double().sum() + flows.backward_mask.double().sum())
    assert torch.isfinite(loss)
    # poses are proper rotations
    r = out.relative[0, :, :, :3].double().cpu()
    assert max_abs(r @ r.transpose(-1, -2), torch.eye(3, dtype=torch.float64).expand_as(r)) < 1e-5
    assert max_abs(torch.linalg.det(r), torch.ones(f - 1, dtype=torch.float64)) < 1e-5
    s0 = 70
    sub = {k: v[s0:s0 + 3] if k in ("in_depth",) else (v[s0:s0 + 2] if k == "in_wparam" else v[:, s0:s0 + 2])
           for k, v in g.items()}
    o2 = _setup(sub)
    out2 = o2.model(o2.batch, o2.flows, 0)
    loss2 = o2.losses[0].forward(o2.batch, o2.flows, None, out2, 0)
    loss2.backward()
    den_sub = float(T(sub["in_fmask"]).double().sum() + T(sub["in_bmask"]).double().sum())
    assert max_abs(out2.relative.cpu(), out.relative[:, s0:s0 + 2].cpu()) <= 1e-6
    # middle frame of the sub-video sees both of its pairs: same gradient up to the normaliser
    g_full = o.model.backbone.depth.grad[s0 + 1].cpu().double() * den_full
    g_sub = o2.model.backbone.depth.grad[1].cpu().double() * den_sub
    assert rel_l2(g_sub, g_full) <= 1e-4
    gw_full = o.model.backbone.weights.grad[s0:s0 + 2].cpu().double() * den_full
    gw_sub = o2.model.backbone.weights.grad.cpu().double() * den_sub
    assert rel_l2(gw_sub, gw_full) <= 1e-4


def test_consistent_scene_recovers_motion():
    """Encode -> decode round trip: flows induced by a known rigid motion and depth give back
    that motion from Procrustes and a (near-)zero flow loss."""
    from oracle import flowmap_oracle as O
    f, h, w = 6, 96, 128
    depth, flows, focal, ext_gt = O.consistent_scene(f, h, w, seed=3, dtype=torch.float64)
    g = {"in_depth": depth.numpy(), "in_wparam": np.zeros((f - 1, h, w)),
         "in_fwd": flows.forward.numpy(), "in_bwd": flows.backward.numpy(),
         "in_fmask": flows.forward_mask.numpy(), "in_bmask": flows.backward_mask.numpy()}
    o = _setup(g, focal=focal)
    out = o.model(o.batch, o.flows, 0)
    loss = o.losses[0].forward(o.batch, o.flows, None, out, 0)
    assert float(loss) < 0.05  # only bilinear-interpolation error is left (oracle: 0.0049)
    assert max_abs(out.extrinsics.cpu(), ext_gt) <= 5e-3
    st = O.OverfitOracle(O.OverfitConfig(intrinsics="regressed", initial_focal=focal), f, h, w,
                         dtype=torch.float64)
    with torch.no_grad():
        st.depth.copy_(depth)
    ref = st.forward(flows, 0)
    assert max_abs(out.extrinsics.cpu(), ref.extrinsics) <= 1e-5


def test_fused_adam_matches_torch():
    from flowmap_b200 import ops
    gen = torch.Generator().manual_seed(0)
    p = torch.randn(1000003, generator=gen)
    ref = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=3e-5)
    pc = p.cuda()
    m, v = torch.zeros_like(pc), torch.zeros_like(pc)
    for step in range(1, 6):
        gr = torch.randn(p.shape, generator=gen) * 10 ** (-step)
        ref.grad = gr.clone()
        opt.step()
        ops.adam_step(pc, gr.cuda(), m, v, step, 3e-5)
    assert max_abs(pc.cpu(), ref.detach()) <= 1e-6


def test_unproject_and_pose_chain_against_golden():
    from flowmap_b200 import ops
    g = load_golden("units")
    k3 = T(g["k3"]).cuda()
    surf = ops.unproject_depth(T(g["z"]).cuda()[None], ops.intrinsics_to_k4(k3)[None])
    assert max_abs(surf[0].cpu(), g["surfaces"]) <= 2e-6
    rt = T(g["rigid_t"])[None, :, :3, :].contiguous().cuda()
    assert max_abs(ops.pose_chain(rt).cpu(), g["chain"]) <= 2e-6
    xy = ops.reproject(T(g["proj_pts"]).cuda(),
                       torch.eye(4)[:3].expand(4, 3, 4).contiguous().cuda(),
                       ops.intrinsics_to_k4(T(g["proj_k"]))[None].expand(4, 4).contiguous().cuda())
    assert np.allclose(xy.cpu().numpy(), g["proj_xy"], rtol=1e-5, atol=2e-6)


def test_tracking_loss_matches_reference_golden():
    """loss_tracking.py / compute_track_flow incl. out-of-frame tracks, overlapping segments,
    the dynamic target-in-frame mask and source == target pairs."""
    from flowmap_b200.types import Tracks
    g64, g32 = load_golden("tracking", True), load_golden("tracking", False)
    o = _setup(g64, cfg_kw=dict(use_tracking=True, tracking_enable_after=0))
    tracks = [Tracks(T(g64[f"trk{i}_xy"]).float(), T(g64[f"trk{i}_vis"]), int(g64[f"trk{i}_start"]))
              for i in range(2)]
    o.tracks = [t.to("cuda") for t in tracks]
    out = o.model(o.batch, o.flows, 0)
    lf = o.losses[0].forward(o.batch, o.flows, o.tracks, out, 0)
    lt = o.losses[1].forward(o.batch, o.flows, o.tracks, out, 0)
    (lf + lt).backward()
    assert abs(float(lf) - float(g64["loss_flow"])) <= 1e-4 * abs(float(g64["loss_flow"]))
    assert abs(float(lt) - float(g64["loss_tracking"])) <= 1e-4 * abs(float(g64["loss_tracking"]))
    gd, gw = o.model.backbone.depth.grad.cpu(), o.model.backbone.weights.grad.cpu()
    gf = float(o.model.intrinsics.focal_length.grad)
    assert rel_l2(gd, g64["g_depth"]) <= max(1e-4, 3 * rel_l2(g32["g_depth"], g64["g_depth"]))
    assert rel_l2(gw, g64["g_wparam"]) <= max(1e-4, 3 * rel_l2(g32["g_wparam"], g64["g_wparam"]))
    assert abs(gf - float(g64["g_focal"])) <= 1e-4 * abs(float(g64["g_focal"]))


def test_tracking_only_gradients_vs_oracle():
    """Tracking loss alone (flow loss off) so that its pose/depth/focal gradients are not
    masked by the larger flow-loss gradients."""
    from oracle import flowmap_oracle as O
    from flowmap_b200.types import Tracks
    g64 = load_golden("tracking", True)
    f, h, w = g64["in_depth"].shape
    st = O.OverfitOracle(O.OverfitConfig(intrinsics="regressed", use_tracking=True,
                                         tracking_enable_after=0, flow_enable_after=10**9),
                         f, h, w, dtype=torch.float64)
    with torch.no_grad():
        st.depth.copy_(T(g64["in_depth"]))
        st.weights.copy_(T(g64["in_wparam"]))
    flows64 = O.Flows(*(T(g64[k]) for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    tr64 = [O.Tracks(T(g64[f"trk{i}_xy"]), T(g64[f"trk{i}_vis"]), int(g64[f"trk{i}_start"])) for i in range(2)]
    ref = st.training_step(flows64, tr64)
    o = _setup(g64, cfg_kw=dict(use_tracking=True, tracking_enable_after=0, flow_enable_after=10**9))
    o.tracks = [Tracks(t.xy.float().cuda(), t.visibility.cuda(), t.start_frame) for t in tr64]
    out = o.model(o.batch, o.flows, 0)
    lt = o.losses[1].forward(o.batch, o.flows, o.tracks, out, 0)
    lt.backward()
    assert abs(float(lt) - ref["parts"]["tracking"]) <= 1e-4 * abs(ref["parts"]["tracking"])
    assert rel_l2(o.model.backbone.depth.grad.cpu(), ref["grads"]["depth"]) <= 2e-4
    assert rel_l2(o.model.backbone.weights.grad.cpu(), ref["grads"]["weights"]) <= 2e-4
    assert abs(float(o.model.intrinsics.focal_length.grad) - float(ref["grads"]["focal"])) <= \
        2e-4 * abs(float(ref["grads"]["focal"]))


@pytest.mark.parametrize("name,mapping,focal,npts", CASES)
def test_fused_step_matches_reference_golden(name, mapping, focal, npts):
    """fm_overfit_step (one C-ABI call per optimisation step) against the same golden vectors."""
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows
    g64, g32 = load_golden(name, True), load_golden(name, False)
    f, h, w = g64["in_depth"].shape
    cfg = OverfitCfg(mapping=mapping, initial_focal=focal, procrustes_points=npts)
    batch = Batch(torch.zeros(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    flows = Flows(*(T(g64[k]).float() for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    o = FusedOverfitter(cfg, batch, flows)
    with torch.no_grad():
        o.model.backbone.depth.copy_(T(g64["in_depth"]).float())
        o.model.backbone.weights.copy_(T(g64["in_wparam"]).float())
    loss, rt = o.training_step(update=False)
    gr = o.gradients()
    assert abs(float(loss) - float(g64["loss"])) <= 1e-4 * abs(float(g64["loss"]))
    assert max_abs(o.extrinsics().cpu(), g64["extrinsics"]) <= 1e-5
    assert rel_l2(gr["depth"].cpu(), g64["g_depth"]) <= max(1e-4, 3 * rel_l2(g32["g_depth"], g64["g_depth"]))
    assert rel_l2(gr["weights"].cpu(), g64["g_wparam"]) <= max(1e-4, 3 * rel_l2(g32["g_wparam"], g64["g_wparam"]))
    assert abs(float(gr["focal"]) - float(g64["g_focal"])) <= 1e-4 * abs(float(g64["g_focal"]))


@pytest.mark.parametrize("name", ["traj_generic", "traj_init"])
def test_fused_adam_trajectory_matches_reference(name):
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows
    g64 = load_golden(name, True)
    f, h, w = g64["in_depth"].shape
    batch = Batch(torch.zeros(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    flows = Flows(*(T(g64[k]).float() for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    o = FusedOverfitter(OverfitCfg(), batch, flows)
    with torch.no_grad():
        o.model.backbone.depth.copy_(T(g64["in_depth"]).float())
        o.model.backbone.weights.copy_(T(g64["in_wparam"]).float())
    for s in range(len(g64["loss"])):
        total, _ = o.training_step()
        assert abs(float(total) - g64["loss"][s]) <= 1e-4 * abs(g64["loss"][s]), s
        assert max_abs(o.extrinsics().cpu(), g64["extrinsics"][s]) <= 1e-4, s
    assert rel_l2(o.model.backbone.depth.detach().cpu(), g64["depth_final"]) <= 1e-5
    w0, w1 = T(g64["in_wparam"]), T(g64["wparam_final"])
    assert rel_l2(o.model.backbone.weights.detach().cpu().double() - w0, w1 - w0) <= 2e-2


def test_fused_step_with_tracking_matches_golden():
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows, Tracks
    g64, g32 = load_golden("tracking", True), load_golden("tracking", False)
    f, h, w = g64["in_depth"].shape
    batch = Batch(torch.zeros(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    flows = Flows(*(T(g64[k]).float() for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    tracks = [Tracks(T(g64[f"trk{i}_xy"]).float(), T(g64[f"trk{i}_vis"]), int(g64[f"trk{i}_start"]))
              for i in range(2)]
    o = FusedOverfitter(OverfitCfg(use_tracking=True, tracking_enable_after=0), batch, flows, tracks)
    with torch.no_grad():
        o.model.backbone.depth.copy_(T(g64["in_depth"]).float())
        o.model.backbone.weights.copy_(T(g64["in_wparam"]).float())
    loss, _ = o.training_step(update=False)
    gr = o.gradients()
    assert abs(float(loss) - float(g64["loss"])) <= 1e-4 * abs(float(g64["loss"]))
    assert rel_l2(gr["depth"].cpu(), g64["g_depth"]) <= max(1e-4, 3 * rel_l2(g32["g_depth"], g64["g_depth"]))
    assert rel_l2(gr["weights"].cpu(), g64["g_wparam"]) <= max(1e-4, 3 * rel_l2(g32["g_wparam"], g64["g_wparam"]))
    assert abs(float(gr["focal"]) - float(g64["g_focal"])) <= 1e-4 * abs(float(g64["g_focal"]))


def test_softmin_intrinsics_matches_reference_golden():
    """IntrinsicsSoftmin (60-candidate sweep, injected point indices) + flow loss: loss, K,
    poses and the gradients that flow through the sweep into depth[:2] / weights[:1]."""
    g64, g32 = load_golden("softmin", True), load_golden("softmin", False)
    o = _setup(g64, cfg_kw=dict(intrinsics="softmin", softmin_points=300, regression_after=None))
    o.model.intrinsics.injected_indices = T(g64["indices"]).cuda()
    out = o.model(o.batch, o.flows, 0)
    loss = o.losses[0].forward(o.batch, o.flows, None, out, 0)
    loss.backward()
    assert abs(float(loss) - float(g64["loss"])) <= 1e-4 * abs(float(g64["loss"]))
    assert max_abs(out.intrinsics.cpu(), g64["intrinsics"]) <= 1e-5
    assert max_abs(out.extrinsics.cpu(), g64["extrinsics"]) <= 1e-5
    gd, gw = o.model.backbone.depth.grad.cpu(), o.model.backbone.weights.grad.cpu()
    assert rel_l2(gd, g64["g_depth"]) <= max(1e-4, 3 * rel_l2(g32["g_depth"], g64["g_depth"]))
    assert rel_l2(gw, g64["g_wparam"]) <= max(1e-4, 3 * rel_l2(g32["g_wparam"], g64["g_wparam"]))
    # the part that exists only because of the sweep: gradient on pair 0's weights / frames 0-1
    assert rel_l2(gw[:1], g64["g_wparam"][:1]) <= max(1e-4, 3 * rel_l2(g32["g_wparam"][:1], g64["g_wparam"][:1]))
    assert rel_l2(gd[:2], g64["g_depth"][:2]) <= max(1e-4, 3 * rel_l2(g32["g_depth"][:2], g64["g_depth"][:2]))


def test_fused_softmin_step_matches_reference_golden():
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows
    g64, g32 = load_golden("softmin", True), load_golden("softmin", False)
    f, h, w = g64["in_depth"].shape
    batch = Batch(torch.zeros(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    flows = Flows(*(T(g64[k]).float() for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    o = FusedOverfitter(OverfitCfg(intrinsics="softmin", softmin_points=300, regression_after=None),
                        batch, flows)
    o.injected_indices = T(g64["indices"]).cuda()
    with torch.no_grad():
        o.model.backbone.depth.copy_(T(g64["in_depth"]).float())
        o.model.backbone.weights.copy_(T(g64["in_wparam"]).float())
    loss, _ = o.training_step(update=False)
    gr = o.gradients()
    assert abs(float(loss) - float(g64["loss"])) <= 1e-4 * abs(float(g64["loss"]))
    k4 = o.intrinsics_k4().cpu()
    assert abs(float(k4[0, 0]) - g64["intrinsics"][0, 0, 0, 0]) <= 1e-5
    assert abs(float(k4[0, 1]) - g64["intrinsics"][0, 0, 1, 1]) <= 1e-5
    assert max_abs(o.extrinsics().cpu(), g64["extrinsics"]) <= 1e-5
    assert rel_l2(gr["depth"].cpu(), g64["g_depth"]) <= max(1e-4, 3 * rel_l2(g32["g_depth"], g64["g_depth"]))
    assert rel_l2(gr["weights"].cpu(), g64["g_wparam"]) <= max(1e-4, 3 * rel_l2(g32["g_wparam"], g64["g_wparam"]))


def test_softmin_to_regressed_handover():
    """intrinsics_softmin.py:75-82,133-139: after `after_step` steps the focal length becomes a
    parameter seeded with the mean of the last `window` sweep estimates (autograd path vs the
    fused path vs the oracle, short schedule)."""
    from oracle import flowmap_oracle as O
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg, Overfitter
    from flowmap_b200.types import Batch, Flows
    g64 = load_golden("softmin", True)
    f, h, w = g64["in_depth"].shape
    kw = dict(intrinsics="softmin", softmin_points=300, regression_after=4, regression_window=2)
    st = O.OverfitOracle(O.OverfitConfig(**kw), f, h, w, dtype=torch.float64)
    with torch.no_grad():
        st.depth.copy_(T(g64["in_depth"]))
        st.weights.copy_(T(g64["in_wparam"]))
    flows64 = O.Flows(*(T(g64[k]) for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    idx = T(g64["indices"])
    ref = [st.training_step(flows64, softmin_indices=idx) for _ in range(7)]
    batch = Batch(torch.zeros(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    flows = Flows(*(T(g64[k]).float() for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask")))
    for cls in (Overfitter, FusedOverfitter):
        o = cls(OverfitCfg(**kw), batch, flows)
        if cls is Overfitter:
            o.model.intrinsics.injected_indices = idx.cuda()
        else:
            o.injected_indices = idx.cuda()
        with torch.no_grad():
            o.model.backbone.depth.copy_(T(g64["in_depth"]).float())
            o.model.backbone.weights.copy_(T(g64["in_wparam"]).float())
        for s in range(7):
            total, _ = o.training_step()
            assert abs(float(total) - ref[s]["loss"]) <= 2e-4 * abs(ref[s]["loss"]), (cls.__name__, s)
        assert abs(float(o.model.intrinsics.intrinsics_regressed.focal_length) - float(st.focal)) <= 1e-5
        assert rel_l2(o.model.backbone.depth.detach().cpu(), st.depth.detach()) <= 1e-5


def test_projection_api_against_golden_units():
    """flowmap_b200.projection / procrustes (function-level mirror) vs the reference's unit vectors."""
    from flowmap_b200 import projection as P
    from flowmap_b200.procrustes import align_rigid
    g = load_golden("units")
    h, w = g["grid_xy"].shape[:2]
    xy, ij = P.sample_image_grid((h, w), device="cuda")
    assert max_abs(xy.cpu(), g["grid_xy"]) <= 1e-7 and bool((ij.cpu().numpy() == g["grid_ij"]).all())
    k3 = T(g["k3"]).cuda()
    surf = P.unproject(xy, T(g["z"]).cuda(), k3[:, None, None])
    assert max_abs(surf.cpu(), g["surfaces"]) <= 2e-6
    proj = P.reproject_points(T(g["proj_pts"]).cuda(), torch.eye(4, device="cuda").expand(4, 1, 4, 4),
                              T(g["proj_k"]).cuda())
    assert np.allclose(proj.cpu().numpy(), g["proj_xy"], rtol=1e-5, atol=2e-6)
    rig = align_rigid(T(g["rigid_p"]).cuda(), T(g["rigid_q"]).cuda(), T(g["rigid_w"]).cuda())
    assert max_abs(rig.cpu(), g["rigid_t"]) <= 5e-6
    assert max_abs(P.get_extrinsics(T(g["rigid_t"]).cuda()[None]).cpu(), g["chain"]) <= 2e-6


def test_align_rigid_gradients_vs_oracle():
    from oracle import flowmap_oracle as O
    from flowmap_b200.procrustes import align_rigid
    gen = torch.Generator().manual_seed(0)
    p = torch.randn(3, 200, 3, generator=gen, dtype=torch.float64)
    q = torch.randn(3, 200, 3, generator=gen, dtype=torch.float64) * 0.3 + p
    q[2] = -q[2]  # reflection branch
    w = torch.rand(3, 200, generator=gen, dtype=torch.float64)
    coef = torch.randn(3, 4, 4, generator=gen, dtype=torch.float64)
    pr, qr, wr = (t.clone().requires_grad_(True) for t in (p, q, w))
    (O.align_rigid(pr, qr, wr) * coef).sum().backward()
    pc, qc, wc = (t.float().cuda().requires_grad_(True) for t in (p, q, w))
    (align_rigid(pc, qc, wc) * coef.float().cuda()).sum().backward()
    assert rel_l2(pc.grad.cpu(), pr.grad) <= 1e-4
    assert rel_l2(qc.grad.cpu(), qr.grad) <= 1e-4
    assert rel_l2(wc.grad.cpu(), wr.grad) <= 1e-4


def test_induced_flow_positions_vs_golden():
    """compute_forward_flow / compute_backward_flow on the lazy surfaces of a ModelOutput."""
    from flowmap_b200 import projection as P
    g = load_golden("flow_huber")
    o = _setup(g)
    with torch.no_grad():
        out = o.model(o.batch, o.flows, 0)
        fwd = P.compute_forward_flow(out.surfaces, out.extrinsics, out.intrinsics)
        bwd = P.compute_backward_flow(out.surfaces, out.extrinsics, out.intrinsics)
    assert max_abs(fwd[:, :2].cpu(), g["fwd_xy"]) <= 2e-5
    assert max_abs(bwd[:, :2].cpu(), g["bwd_xy"]) <= 2e-5


def test_random_subset_is_a_uniform_sample_without_replacement():
    from flowmap_b200 import ops
    n_items, n = 360 * 640, 8192
    a = ops.random_subset(n_items, n, "cuda", seed=1).cpu()
    b = ops.random_subset(n_items, n, "cuda", seed=2).cpu()
    assert a.min() >= 0 and a.max() < n_items and a.unique().numel() == n
    assert not torch.equal(a, b)
    # a full-length draw is a permutation
    perm = ops.random_subset(1000, 1000, "cuda", seed=3).cpu()
    assert torch.equal(perm.sort().values, torch.arange(1000))
    # roughly uniform over the range (mean of U[0, N) is N/2, std N/sqrt(12 n))
    assert abs(float(a.double().mean()) - n_items / 2) < 5 * n_items / (12 * n) ** 0.5


def _oracle_flow_step(depth, wparam, flows64, focal=0.85, indices=None, softmin=None, **kw):
    """Oracle loss, extrinsics and gradients for batched inputs (b, f, h, w), in the dtype of
    `depth` (float64: the arbiter; float32: the reference's own rounding noise).  `indices`: the
    Procrustes point set (default: every pixel).  `softmin=(indices, candidates)`: the intrinsics
    come from the candidate sweep at those points instead of `focal`, and in place of the
    focal-length gradient the gradient of the sweep's errors (b, n) is returned."""
    from oracle import flowmap_oracle as O
    b, f, h, w = depth.shape
    d = depth.clone().requires_grad_(True)
    wp = wparam.clone().requires_grad_(True)
    foc = torch.tensor(focal, dtype=depth.dtype, requires_grad=True)
    weights = torch.sigmoid(100.0 * wp) if kw.get("use_weights", True) else torch.ones_like(wp)
    if softmin is None:
        k = O.intrinsics_from_focal(foc, h, w).expand(b, f, 3, 3)
    else:
        err = O.softmin_errors(d, weights, flows64.backward, *softmin)
        err.retain_grad()
        k = O.softmin_intrinsics(err, softmin[1], h, w)[0][:, None].expand(b, f, 3, 3)
    surf = O.unproject(O.pixel_grid(h, w, depth.dtype), d, k[:, :, None, None])
    idx = torch.arange(h * w) if indices is None else indices
    ext = O.align_surfaces(surf, flows64.backward, weights, idx)
    loss = 1000.0 * O.flow_loss(surf, ext, k, flows64, kw.get("mapping", "huber"), 0.01)
    loss.backward()
    return loss.detach(), ext.detach(), d.grad, wp.grad, foc.grad if softmin is None else err.grad


@pytest.mark.parametrize("b,f,h,w", [(2, 4, 16, 24), (1, 2, 12, 20), (1, 3, 18, 22), (3, 3, 7, 9)])
def test_batched_and_odd_shapes_vs_oracle(b, f, h, w):
    """b > 1 (the pretraining use), a single frame pair, and widths that are not a multiple of 4
    (scalar instantiation of every kernel), through the autograd ops."""
    from oracle import flowmap_oracle as O
    from flowmap_b200 import ops
    gen = torch.Generator().manual_seed(b * 100 + f * 10 + w)
    depth = 1.0 + torch.rand(b, f, h, w, generator=gen, dtype=torch.float64)
    wparam = 0.01 * torch.randn(b, f - 1, h, w, generator=gen, dtype=torch.float64)
    fl = O.synthetic_flows(f, h, w, seed=w, dtype=torch.float64, b=b)
    loss_r, ext_r, gd_r, gw_r, gf_r = _oracle_flow_step(depth, wparam, fl)
    d = depth.float().cuda().requires_grad_(True)
    wp = wparam.float().cuda().requires_grad_(True)
    foc = torch.tensor(0.85, device="cuda", requires_grad=True)
    s = (h * w) ** 0.5
    k4 = torch.stack((foc * s / w, foc * s / h, torch.tensor(0.5, device="cuda"), torch.tensor(0.5, device="cuda")))
    k4 = k4.expand(b, f, 4)
    flc = [t.float().cuda() for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)]
    rt = ops.procrustes_poses(d, torch.sigmoid(100.0 * wp), k4, flc[1], None)
    for mode in ("full", "shared_focal"):
        d.grad = wp.grad = foc.grad = None
        loss = ops.flow_loss(d, rt, k4, *flc, ops.mask_sum(flc[2], flc[3]), "huber", 0.01, 1000.0, mode)
        loss.backward(retain_graph=True)
        assert abs(float(loss) - float(loss_r)) <= 1e-4 * abs(float(loss_r)), mode
        assert rel_l2(d.grad.cpu(), gd_r) <= 1e-4, mode
        assert rel_l2(wp.grad.cpu(), gw_r) <= 1e-4, mode
        assert abs(float(foc.grad) - float(gf_r)) <= 1e-4 * abs(float(gf_r)), mode
    assert max_abs(ops.pose_chain(rt).cpu(), ext_r) <= 1e-5


def test_constant_intrinsics_mode_and_no_weights():
    """k_mode="const" (ground-truth intrinsics: no K gradient) and use_correspondence_weights=False."""
    from oracle import flowmap_oracle as O
    from flowmap_b200 import ops
    b, f, h, w = 1, 4, 16, 24
    gen = torch.Generator().manual_seed(5)
    depth = 1.0 + torch.rand(b, f, h, w, generator=gen, dtype=torch.float64)
    wparam = torch.zeros(b, f - 1, h, w, dtype=torch.float64)
    fl = O.synthetic_flows(f, h, w, seed=2, dtype=torch.float64)
    loss_r, ext_r, gd_r, _, _ = _oracle_flow_step(depth, wparam, fl, use_weights=False)
    d = depth.float().cuda().requires_grad_(True)
    s = (h * w) ** 0.5
    k4 = torch.tensor([0.85 * s / w, 0.85 * s / h, 0.5, 0.5], device="cuda").expand(b, f, 4).contiguous()
    flc = [t.float().cuda() for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)]
    rt = ops.procrustes_poses(d, None, k4, flc[1], None)
    loss = ops.flow_loss(d, rt, k4, *flc, ops.mask_sum(flc[2], flc[3]), "huber", 0.01, 1000.0, "const")
    loss.backward()
    assert abs(float(loss) - float(loss_r)) <= 1e-4 * abs(float(loss_r))
    assert rel_l2(d.grad.cpu(), gd_r) <= 1e-4


def test_zero_masks_use_denominator_one():
    """loss_flow.py:70 `valid_sum or 1`: all-zero masks give loss 0 and zero gradients, no NaN."""
    from flowmap_b200 import ops
    b, f, h, w = 1, 3, 8, 12
    d = (1.0 + torch.rand(b, f, h, w)).cuda().requires_grad_(True)
    k4 = torch.tensor([0.9, 1.2, 0.5, 0.5], device="cuda").expand(b, f, 4).contiguous()
    z2, z1 = torch.zeros(b, f - 1, h, w, 2, device="cuda"), torch.zeros(b, f - 1, h, w, device="cuda")
    rt = ops.procrustes_poses(d, torch.ones_like(z1), k4, z2, None)
    loss = ops.flow_loss(d, rt, k4, z2, z2, z1, z1, ops.mask_sum(z1, z1), "huber", 0.01, 1000.0)
    loss.backward()
    assert float(loss) == 0.0 and bool(torch.isfinite(d.grad).all()) and float(d.grad.abs().max()) == 0.0


def test_c2_shape_full_step_vs_oracle():
    """BASELINE configs[1] (LLFF shape: 30 x 360 x 480, flow + tracks): one fused step with
    tracking against the float64 oracle (loss parts, poses, gradients)."""
    from oracle import flowmap_oracle as O
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows, Tracks
    f, h, w = 30, 360, 480
    fl = O.synthetic_flows(f, h, w, seed=1, dtype=torch.float32)
    gen = torch.Generator().manual_seed(2)
    depth = 1.0 + 0.5 * torch.rand(f, h, w, generator=gen)
    wparam = 0.01 * torch.randn(f - 1, h, w, generator=gen)
    trk = O.synthetic_tracks(f, n_points=400, seed=3)
    torch.set_num_threads(min(16, torch.get_num_threads()))

    def oracle_step(dtype):
        st = O.OverfitOracle(O.OverfitConfig(intrinsics="regressed", use_tracking=True,
                                             tracking_enable_after=0), f, h, w, dtype=dtype)
        with torch.no_grad():
            st.depth.copy_(depth.to(dtype))
            st.weights.copy_(wparam.to(dtype))
        flows = O.Flows(*(t.to(dtype) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))
        return st.training_step(flows, [O.Tracks(t.xy.to(dtype), t.visibility, t.start_frame) for t in trk])

    def errors(loss, ext, gd, gw, gf, ref):
        return dict(loss=abs(float(loss) - ref["loss"]) / abs(ref["loss"]),
                    pose=max_abs(ext.double(), ref["extrinsics"]),
                    depth=rel_l2(gd.double(), ref["grads"]["depth"]),
                    weights=rel_l2(gw.double(), ref["grads"]["weights"]),
                    focal=abs(float(gf) - float(ref["grads"]["focal"])) / abs(float(ref["grads"]["focal"])))

    # The reference's own float32 run is 1.9e-4 / 2.8e-4 / 2.3e-4 (depth / weights / focal
    # gradients) away from float64 at this shape: the tolerance is max(1e-4, that noise).
    ref, ref32 = oracle_step(torch.float64), oracle_step(torch.float32)
    noise = errors(ref32["loss"], ref32["extrinsics"], ref32["grads"]["depth"], ref32["grads"]["weights"],
                   ref32["grads"]["focal"], ref)
    batch = Batch(torch.zeros(1, 1, 1, 1, 1).expand(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    o = FusedOverfitter(OverfitCfg(use_tracking=True, tracking_enable_after=0), batch,
                        Flows(fl.forward, fl.backward, fl.forward_mask, fl.backward_mask),
                        [Tracks(t.xy, t.visibility, t.start_frame) for t in trk])
    with torch.no_grad():
        o.model.backbone.depth.copy_(depth)
        o.model.backbone.weights.copy_(wparam)
    loss, _ = o.training_step(update=False)
    gr = o.gradients()
    errs = errors(loss, o.extrinsics().cpu(), gr["depth"].cpu(), gr["weights"].cpu(), gr["focal"], ref)
    print("C2 errors vs float64 oracle:", errs, "reference float32 noise:", noise)
    assert errs["loss"] <= 1e-4 and errs["pose"] <= 2e-5, errs
    for key in ("depth", "weights", "focal"):
        assert errs[key] <= max(1e-4, noise[key]), (key, errs, noise)


def test_c4_shape_properties():
    """BASELINE configs[3] shape (720 x 1280 frames; 24 of the 150 frames to bound the test):
    finite loss, proper rotations, and pair locality against a 3-frame slice."""
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows
    f, h, w = 24, 720, 1280
    gen = torch.Generator(device="cuda").manual_seed(0)
    depth = 0.1 + 0.05 * torch.rand(f, h, w, device="cuda", generator=gen)
    wparam = 0.01 * torch.randn(f - 1, h, w, device="cuda", generator=gen)
    mk = lambda *s: 0.01 * torch.randn(*s, device="cuda", generator=gen)  # noqa: E731
    un = lambda *s: torch.rand(*s, device="cuda", generator=gen)  # noqa: E731
    flows = Flows(mk(1, f - 1, h, w, 2), mk(1, f - 1, h, w, 2), un(1, f - 1, h, w), un(1, f - 1, h, w))

    def run(sl_f, sl_p):
        nf = sl_f.stop - sl_f.start
        batch = Batch(torch.zeros(1, 1, 1, 1, 1, device="cuda").expand(1, nf, 3, h, w),
                      torch.arange(nf, device="cuda")[None], ["s"], ["d"])
        fl = Flows(*(t[:, sl_p].contiguous() for t in (flows.forward, flows.backward, flows.forward_mask,
                                                       flows.backward_mask)))
        o = FusedOverfitter(OverfitCfg(), batch, fl)
        with torch.no_grad():
            o.model.backbone.depth.copy_(depth[sl_f])
            o.model.backbone.weights.copy_(wparam[sl_p])
        loss, rt = o.training_step(update=False)
        den = float(fl.forward_mask.double().sum() + fl.backward_mask.double().sum())
        return float(loss), rt.clone(), o.gradients()["depth"].double() * den, o.gradients()["weights"].double() * den

    loss, rt, gd, gw = run(slice(0, f), slice(0, f - 1))
    assert np.isfinite(loss)
    r = rt[0, :, :, :3].double().cpu()
    assert max_abs(r @ r.transpose(-1, -2), torch.eye(3, dtype=torch.float64).expand_as(r)) < 1e-5
    s0 = 10
    _, rt2, gd2, gw2 = run(slice(s0, s0 + 3), slice(s0, s0 + 2))
    assert max_abs(rt2.cpu(), rt[:, s0:s0 + 2].cpu()) <= 1e-6
    assert rel_l2(gd2[1].cpu(), gd[s0 + 1].cpu()) <= 1e-4
    assert rel_l2(gw2.cpu(), gw[s0:s0 + 2].cpu()) <= 1e-4


@pytest.mark.parametrize("intrinsics", ["regressed", "softmin"])
def test_split_step_with_tracking_equals_fused(intrinsics):
    """The pair-sharded driver (split step, gathered poses, source-sharded tracking, sweep on the
    first rank) on a one-rank group must reproduce the unsharded fused optimisation."""
    import socket
    import torch.distributed as dist
    from oracle import flowmap_oracle as O
    from flowmap_b200 import parallel
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg, ShardedFusedOverfitter
    from flowmap_b200.types import Batch, Flows, Tracks
    f, h, w = 12, 48, 64
    fl = O.synthetic_flows(f, h, w, seed=5)
    trk = [Tracks(t.xy, t.visibility, t.start_frame)
           for t in O.synthetic_tracks(f, n_points=96, interval=4, radius=5, seed=6)]
    gen = torch.Generator().manual_seed(7)
    depth = 1.0 + 0.5 * torch.rand(f, h, w, generator=gen)
    wparam = 0.01 * torch.randn(f - 1, h, w, generator=gen)
    cfg = OverfitCfg(intrinsics=intrinsics, use_tracking=True, tracking_enable_after=1, softmin_points=256,
                     regression_after=3, regression_window=2, lr=1e-3)
    idx = torch.randperm(h * w, generator=gen)[:256].cuda()

    def make(cls, *extra, **kw):
        batch = Batch(torch.zeros(1, 1, 1, 1, 1).expand(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
        o = cls(cfg, batch, Flows(fl.forward, fl.backward, fl.forward_mask, fl.backward_mask), *extra, **kw)
        with torch.no_grad():
            o.model.backbone.depth.copy_(depth)
            o.model.backbone.weights.copy_(wparam)
        o.injected_indices = idx
        return o

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        sh = make(ShardedFusedOverfitter, parallel.make_plan(f - 1), tracks=trk)
        ref = make(FusedOverfitter, trk)
        for step in range(5):   # sweep stage (0-2) incl. tracking from step 1, hand-over at 3, regressed
            l_sh, _ = sh.training_step()
            l_ref, _ = ref.training_step()
            assert abs(float(l_sh) - float(l_ref)) <= 2e-5 * abs(float(l_ref)), step
        assert rel_l2(sh.model.backbone.depth.detach().cpu(), ref.model.backbone.depth.detach().cpu()) <= 1e-6
        upd = lambda o: (o.model.backbone.weights.detach().cpu() - wparam)  # noqa: E731
        assert rel_l2(upd(sh), upd(ref)) <= 1e-3
        assert abs(float(sh._focal) - float(ref._focal)) <= 1e-6
    finally:
        dist.destroy_process_group()


def _tracking_case(tracks64, f=6, h=20, w=28, seed=21):
    """Fused step (flow + tracking) on `tracks64` against the float64 oracle."""
    from oracle import flowmap_oracle as O
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows, Tracks
    fl = O.synthetic_flows(f, h, w, seed=seed, dtype=torch.float64)
    gen = torch.Generator().manual_seed(seed + 1)
    depth = 1.0 + 0.5 * torch.rand(f, h, w, generator=gen, dtype=torch.float64)
    wparam = 0.01 * torch.randn(f - 1, h, w, generator=gen, dtype=torch.float64)
    st = O.OverfitOracle(O.OverfitConfig(intrinsics="regressed", use_tracking=True, tracking_enable_after=0),
                         f, h, w, dtype=torch.float64)
    with torch.no_grad():
        st.depth.copy_(depth)
        st.weights.copy_(wparam)
    ref = st.training_step(fl, tracks64)
    batch = Batch(torch.zeros(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    o = FusedOverfitter(OverfitCfg(use_tracking=True, tracking_enable_after=0), batch,
                        Flows(*(t.float() for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask))),
                        [Tracks(t.xy.float(), t.visibility, t.start_frame) for t in tracks64])
    with torch.no_grad():
        o.model.backbone.depth.copy_(depth.float())
        o.model.backbone.weights.copy_(wparam.float())
    loss, _ = o.training_step(update=False)
    return float(loss), o.gradients(), float(o._track_loss), ref


def test_tracking_edge_cases_vs_oracle():
    """Ragged / degenerate track segments: a one-frame segment, a point count that is not a multiple
    of the block size, a segment longer than the usual 41 frames, tracks entirely outside the image
    or entirely invisible (`valid_sum or 1`, loss_tracking.py:61)."""
    from oracle import flowmap_oracle as O
    f = 6
    gen = torch.Generator().manual_seed(3)
    mk = lambda rows, n, start, vis_p=0.7, lo=0.0, hi=1.0: O.Tracks(  # noqa: E731
        lo + (hi - lo) * torch.rand(1, rows, n, 2, generator=gen, dtype=torch.float64),
        torch.rand(1, rows, n, generator=gen) < vis_p, start)
    ragged = [mk(1, 37, 2), mk(6, 301, 0), mk(3, 5, 3), mk(2, 1, 4)]
    loss, gr, _, ref = _tracking_case(ragged)
    assert abs(loss - ref["loss"]) <= 1e-4 * abs(ref["loss"])
    assert rel_l2(gr["depth"].cpu(), ref["grads"]["depth"]) <= 2e-4
    assert rel_l2(gr["weights"].cpu(), ref["grads"]["weights"]) <= 2e-4
    # nothing valid: every source is outside [0,1)^2, or nothing is visible
    for dead in ([mk(4, 50, 1, lo=1.5, hi=2.5)], [mk(4, 50, 1, vis_p=-1.0)]):
        loss, gr, track_loss, ref = _tracking_case(dead)
        assert track_loss == 0.0 and ref["parts"]["tracking"] == 0.0
        assert abs(loss - ref["loss"]) <= 1e-4 * abs(ref["loss"])
        assert bool(torch.isfinite(gr["depth"]).all())
        assert rel_l2(gr["depth"].cpu(), ref["grads"]["depth"]) <= 1e-4


def test_long_track_segment_uses_more_shared_memory():
    """A 70-frame segment (the default radius gives 41): per-block shared memory grows with the
    segment length; parity with the oracle must hold."""
    from oracle import flowmap_oracle as O
    f = 70
    gen = torch.Generator().manual_seed(9)
    seg = O.Tracks(torch.rand(1, f, 64, 2, generator=gen, dtype=torch.float64),
                   torch.rand(1, f, 64, generator=gen) < 0.7, 0)
    loss, gr, _, ref = _tracking_case([seg], f=f, h=12, w=16)
    assert abs(loss - ref["loss"]) <= 1e-4 * abs(ref["loss"])
    assert rel_l2(gr["depth"].cpu(), ref["grads"]["depth"]) <= 3e-4


def test_vanishing_weights_give_identity_poses():
    """All correspondence weights exactly 0 (float32 sigmoid(100 * -2) underflows): centroids use
    sum + 1e-8 (procrustes.py:24), the covariance is the zero matrix and the reference's SVD returns
    U = V = I, i.e. the identity pose; the Jacobi solve must not produce NaN there."""
    from oracle import flowmap_oracle as O
    from flowmap_b200 import ops
    b, f, h, w = 1, 3, 8, 12
    gen = torch.Generator().manual_seed(1)
    depth = 1.0 + torch.rand(b, f, h, w, generator=gen)
    fl = O.synthetic_flows(f, h, w, seed=4)
    weights = torch.sigmoid(torch.full((b, f - 1, h, w), -200.0))
    assert float(weights.max()) == 0.0
    k = O.intrinsics_from_focal(torch.tensor(0.85), h, w).expand(b, f, 3, 3)
    surf = O.unproject(O.pixel_grid(h, w, torch.float32), depth, k[:, :, None, None])
    ref = O.relative_poses(surf, fl.backward, weights, torch.arange(h * w))
    assert max_abs(ref, torch.eye(4).expand_as(ref)) == 0.0
    s = (h * w) ** 0.5
    k4 = torch.tensor([0.85 * s / w, 0.85 * s / h, 0.5, 0.5], device="cuda").expand(b, f, 4).contiguous()
    rt = ops.procrustes_poses(depth.cuda(), weights.cuda(), k4, fl.backward.cuda(), None)
    assert bool(torch.isfinite(rt).all())
    assert max_abs(rt.cpu(), ref[..., :3, :]) <= 1e-6


def test_set_flows_switches_the_batch():
    """FusedOverfitter.set_flows (the next batch of a prefetching loader): same result as an
    optimiser built on those flows; shape mismatches are rejected."""
    from oracle import flowmap_oracle as O
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows
    f, h, w = 5, 16, 24
    mk = lambda seed: Flows(*(t.cuda() for t in (lambda fl: (fl.forward, fl.backward, fl.forward_mask,  # noqa: E731
                                                             fl.backward_mask))(O.synthetic_flows(f, h, w, seed=seed))))
    batch = Batch(torch.zeros(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    a, b = mk(1), mk(2)
    o = FusedOverfitter(OverfitCfg(), batch, a)
    ref = FusedOverfitter(OverfitCfg(), batch, b)
    first = float(o.training_step(update=False)[0])
    o.set_flows(b)
    second, want = float(o.training_step(update=False)[0]), float(ref.training_step(update=False)[0])
    assert abs(second - want) <= 1e-6 * abs(want) and abs(second - first) > 1e-3 * abs(want)
    assert rel_l2(o.gradients()["depth"].cpu(), ref.gradients()["depth"].cpu()) <= 1e-6  # atomics: order varies
    with pytest.raises(ValueError):
        o.set_flows(Flows(b.forward[:, :-1], b.backward[:, :-1], b.forward_mask[:, :-1], b.backward_mask[:, :-1]))


@pytest.mark.parametrize("b,f", [(1, 2), (1, 3), (2, 150), (1, 257), (1, 258), (3, 1200)])
def test_pose_chain_scan_vs_sequential_float64(b, f):
    """The chain P_{k+1} = P_k T_k (projection.py:187-210) runs as a parallel scan: values and the
    adjoint against the sequential float64 product, incl. chunked (> 256 pairs) and batched cases."""
    from oracle import flowmap_oracle as O
    from flowmap_b200 import ops
    gen = torch.Generator().manual_seed(f)
    # small random rigid motions
    w = 0.05 * torch.randn(b, f - 1, 3, generator=gen, dtype=torch.float64)
    K = torch.zeros(b, f - 1, 3, 3, dtype=torch.float64)
    K[..., 0, 1], K[..., 0, 2], K[..., 1, 0] = -w[..., 2], w[..., 1], w[..., 2]
    K[..., 1, 2], K[..., 2, 0], K[..., 2, 1] = -w[..., 0], -w[..., 1], w[..., 0]
    T = torch.eye(4, dtype=torch.float64).repeat(b, f - 1, 1, 1)
    T[..., :3, :3] = torch.linalg.matrix_exp(K)
    T[..., :3, 3] = 0.1 * torch.randn(b, f - 1, 3, generator=gen, dtype=torch.float64)
    T.requires_grad_(True)
    ref = O.pose_chain(T)
    gout = torch.randn(b, f, 4, 4, generator=gen, dtype=torch.float64)
    gout[..., 3, :] = 0
    ref.backward(gout)
    rt = T.detach()[..., :3, :].float().cuda().requires_grad_(True)
    ext = ops.pose_chain(rt)
    ext.backward(gout.float().cuda())
    scale = float(ref.detach().abs().max())
    assert max_abs(ext.detach().cpu(), ref.detach()) <= 2e-6 * max(1.0, scale) * (1 + f / 150)
    assert rel_l2(rt.grad.cpu(), T.grad[..., :3, :]) <= 1e-5


def twist(rot, g):
    """Left-perturbation twist (F, 6) of an ambient pose gradient g (1, F, 4, 4) at rotations rot (F, 3, 3):
    omega = sum_c R_c x G_c, v = G_t."""
    om = torch.linalg.cross(rot.transpose(-1, -2), g[0, :, :3, :3].transpose(-1, -2), dim=-1).sum(dim=-2)
    return torch.cat((om, g[0, :, :3, 3]), dim=-1)


def test_tracking_per_frame_intrinsics_gradient_and_shared_mode():
    """Tracking loss with PER-FRAME intrinsics (different k4 rows): d loss / d k4 per frame against the
    float64 oracle (general kernel variant); and the shared-intrinsics variant must give the same
    depth / pose gradients and the same SUM over frames of the intrinsics gradient."""
    from oracle import flowmap_oracle as O
    from flowmap_b200 import ops
    f, h, w = 6, 20, 28
    gen = torch.Generator().manual_seed(13)
    depth = (1.0 + 0.5 * torch.rand(1, f, h, w, generator=gen, dtype=torch.float64)).requires_grad_(True)
    # poses: small motions; intrinsics: a different focal per frame
    wv = 0.03 * torch.randn(f, 3, generator=gen, dtype=torch.float64)
    K = torch.zeros(f, 3, 3, dtype=torch.float64)
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 0], K[:, 1, 2], K[:, 2, 0], K[:, 2, 1] = -wv[:, 2], wv[:, 1], wv[:, 2], -wv[:, 0], -wv[:, 1], wv[:, 0]
    ext = torch.eye(4, dtype=torch.float64).repeat(1, f, 1, 1)
    ext[0, :, :3, :3] = torch.linalg.matrix_exp(K)
    ext[0, :, :3, 3] = 0.05 * torch.randn(f, 3, generator=gen, dtype=torch.float64)
    ext.requires_grad_(True)
    focal = (0.8 + 0.1 * torch.rand(f, generator=gen, dtype=torch.float64)).requires_grad_(True)
    s = (h * w) ** 0.5
    half = torch.full_like(focal, 0.5)
    k4 = torch.stack((focal * s / w, focal * s / h, half, half), dim=-1)[None]
    kmat_rows = []
    for i in range(f):
        kmat_rows.append(torch.stack((torch.stack((k4[0, i, 0], torch.zeros((), dtype=torch.float64), k4[0, i, 2])),
                                      torch.stack((torch.zeros((), dtype=torch.float64), k4[0, i, 1], k4[0, i, 3])),
                                      torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64))))
    kmat = torch.stack(kmat_rows)[None]
    tracks = [O.Tracks(torch.rand(1, f, 90, 2, generator=gen, dtype=torch.float64),
                       torch.rand(1, f, 90, generator=gen) < 0.8, 0),
              O.Tracks(torch.rand(1, 3, 33, 2, generator=gen, dtype=torch.float64),
                       torch.rand(1, 3, 33, generator=gen) < 0.8, 2)]
    surf = O.unproject(O.pixel_grid(h, w, torch.float64), depth, kmat[:, :, None, None])
    ref = 100.0 * O.tracking_loss(surf, ext, kmat, tracks)
    ref.backward()
    from flowmap_b200.types import Tracks
    packed = ops.PackedTracks([Tracks(t.xy.float().cuda(), t.visibility.cuda(), t.start_frame) for t in tracks], "cuda")
    out = {}
    for shared in (False, True):
        d = depth.detach().float().cuda().requires_grad_(True)
        e = ext.detach().float().cuda().requires_grad_(True)
        k = k4.detach().float().cuda().requires_grad_(True)
        loss = ops.track_loss(d, e, k, packed, "huber", 0.01, 100.0, shared)
        loss.backward()
        out[shared] = (float(loss), d.grad.cpu(), e.grad.cpu(), k.grad.cpu())
    g_focal_frames = focal.grad  # per-frame d loss / d focal_i
    rot = ext.detach()[0, :, :3, :3]
    for shared in (False, True):
        loss, gd, ge, gk = out[shared]
        assert abs(loss - float(ref)) <= 1e-4 * abs(float(ref))
        assert rel_l2(gd, depth.grad) <= 2e-4
        assert rel_l2(twist(rot, ge.double()), twist(rot, ext.grad)) <= 2e-4   # only the tangent part is defined
    per_frame = out[False][3][0, :, 0].double() * s / w + out[False][3][0, :, 1].double() * s / h
    assert rel_l2(per_frame, g_focal_frames) <= 2e-4
    total = lambda gk: float((gk[0, :, 0].double() * s / w + gk[0, :, 1].double() * s / h).sum())  # noqa: E731
    assert abs(total(out[True][3]) - float(g_focal_frames.sum())) <= 2e-4 * float(g_focal_frames.abs().sum())


@pytest.mark.parametrize("w,npts", [(22, None), (26, 100), (24, 100)])
def test_fused_trajectory_odd_width_and_subsampled_procrustes(w, npts):
    """Fused step with Adam on the code paths the BASELINE shape never takes: a width that is not a
    multiple of 4 (scalar kernel instantiations, separate weight Adam) and / or subsampled Procrustes
    points (sparse weight gradient), with the tracking loss, over 4 Adam steps against the float64
    oracle trajectory."""
    from oracle import flowmap_oracle as O
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows, Tracks
    f, h = 5, 18
    fl = O.synthetic_flows(f, h, w, seed=w, dtype=torch.float64)
    gen = torch.Generator().manual_seed(w + 1)
    depth = 1.0 + 0.5 * torch.rand(f, h, w, generator=gen, dtype=torch.float64)
    wparam = 0.01 * torch.randn(f - 1, h, w, generator=gen, dtype=torch.float64)
    trk = O.synthetic_tracks(f, n_points=70, interval=2, radius=2, seed=5, dtype=torch.float64)
    kw = dict(use_tracking=True, tracking_enable_after=1, procrustes_points=npts)
    st = O.OverfitOracle(O.OverfitConfig(intrinsics="regressed", lr=1e-3, **kw), f, h, w, dtype=torch.float64)
    with torch.no_grad():
        st.depth.copy_(depth)
        st.weights.copy_(wparam)
    batch = Batch(torch.zeros(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    o = FusedOverfitter(OverfitCfg(lr=1e-3, **kw), batch,
                        Flows(*(t.float() for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask))),
                        [Tracks(t.xy.float(), t.visibility, t.start_frame) for t in trk])
    with torch.no_grad():
        o.model.backbone.depth.copy_(depth.float())
        o.model.backbone.weights.copy_(wparam.float())
    pts = None if o._indices is None else o._indices.cpu()  # the point set the kernels use
    for step in range(4):
        ref = st.training_step(fl, trk, procrustes_idx=pts)
        loss, _ = o.training_step()
        assert abs(float(loss) - ref["loss"]) <= 2e-4 * abs(ref["loss"]), step
    assert rel_l2(o.model.backbone.depth.detach().cpu(), st.depth.detach()) <= 1e-5
    assert rel_l2(o.model.backbone.weights.detach().cpu().double() - wparam, st.weights.detach() - wparam) <= 2e-2
    assert abs(float(o._focal) - float(st.focal)) <= 1e-5
