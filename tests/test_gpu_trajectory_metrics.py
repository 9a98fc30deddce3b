"""fm_trajectory_ate / flowmap_b200.ate against the reference's compute_ate (tests/golden/ate.npz), and
the per-step metrics log of the fused overfit step (fm_overfit_step_args.metrics_log)."""
import math

import pytest
import torch

from ate_checks import check_case, golden_cases
from conftest import rel_l2

CASES = golden_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_trajectory_ate_kernel_matches_reference(name):
    from flowmap_b200.ate import trajectory_ate
    c = CASES[name]
    gt, pred = torch.as_tensor(c["gt"]).cuda(), torch.as_tensor(c["pred"]).cuda()
    ate, al_gt, al_pred, status = trajectory_ate(gt, pred)
    torch.cuda.synchronize()
    assert int(status) == int(bool(c["raised"]))
    if c["raised"]:  # all-zero prediction: status 1, NaN, no fault
        assert math.isnan(float(ate))
        return
    check_case(name, c, float(ate), al_gt.cpu().numpy(), al_pred.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("device", ["cuda", "cpu"])
def test_compute_ate_matches_reference(name, device):
    from flowmap_b200.ate import compute_ate
    c = CASES[name]
    gt, pred = torch.as_tensor(c["gt"]).to(device), torch.as_tensor(c["pred"]).to(device)
    if c["raised"]:
        with pytest.raises(ValueError, match="unique points"):
            compute_ate(gt, pred)
        return
    ate, al_gt, al_pred = compute_ate(gt, pred)
    assert ate.shape == () and ate.dtype == torch.float32
    assert ate.device == gt.device and al_gt.device == gt.device and al_pred.device == pred.device
    check_case(name, c, float(ate), al_gt.cpu().numpy(), al_pred.cpu().numpy())
    # the reference's own float32 ATE (of its float32 aligned sets) agrees to its rounding
    assert abs(float(ate) - float(c["ate"])) <= 1e-6 * float(c["ate"]) + 1e-7


@pytest.mark.gpu
def test_compute_ate_raises_scipys_value_errors():
    from flowmap_b200.ate import compute_ate
    x = torch.rand(5, 3, device="cuda")
    with pytest.raises(ValueError, match="two-dimensional"):
        compute_ate(x[0], x[0])
    with pytest.raises(ValueError, match="same shape"):
        compute_ate(x, x[:4])
    with pytest.raises(ValueError, match=">0 rows"):
        compute_ate(x[:0], x[:0])
    with pytest.raises(ValueError, match="unique points"):
        compute_ate(x, x[:1].expand(5, 3) * 0)


@pytest.mark.gpu
def test_batched_trajectories_equal_single_calls_bitwise():
    from flowmap_b200.ate import trajectory_ate
    g = torch.Generator().manual_seed(2)
    T, F = 2000, 150
    gt = torch.cumsum(0.1 * torch.randn(T, F, 3, generator=g), dim=1).cuda()
    pred = (gt @ torch.linalg.qr(torch.randn(3, 3, generator=g))[0].cuda() * 2.0 +
            0.01 * torch.randn(T, F, 3, generator=g).cuda())
    pred[7] = 0.0  # a degenerate trajectory in the batch leaves the others alone
    ate, al_gt, al_pred, status = trajectory_ate(gt, pred)
    for t in range(T):
        a1, g1, p1, s1 = trajectory_ate(gt[t], pred[t])
        assert int(s1) == int(status[t]) == int(t == 7)
        assert torch.equal(a1, ate[t]) or (t == 7 and math.isnan(float(a1)) and math.isnan(float(ate[t])))
        if t != 7:
            assert torch.equal(g1, al_gt[t]) and torch.equal(p1, al_pred[t])


def test_sharded_overfitter_has_no_metrics_log():
    from flowmap_b200.overfit import ShardedFusedOverfitter
    with pytest.raises(ValueError, match="metrics log"):
        ShardedFusedOverfitter.enable_metrics_log(None, 4)


# ---- the per-step log of the fused step ---------------------------------------------------------

F_, H_, W_, STEPS = 8, 96, 192, 10


def _scene():
    from oracle import flowmap_oracle as O
    depth, fl, focal, ext = O.consistent_scene(F_, H_, W_, seed=3)
    tracks = O.scene_tracks(depth, ext, focal, [(0, F_), (2, 4)], n_points=300, seed=4)
    k = O.intrinsics_from_focal(torch.tensor(focal, dtype=torch.float64), H_, W_).expand(1, F_, 3, 3)
    return depth, fl, focal, ext, tracks, k


def _run(capacity=16, with_gt=True, graph=True):
    """Softmin stage with the hand-over after 4 of 10 steps, tracking from step 2.  Returns the
    per-step records of the run and its log (None with capacity 0)."""
    from flowmap_b200 import ate, _lib
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows, Tracks
    depth, fl, focal, ext, tracks, k = _scene()
    batch = Batch(torch.zeros(1, 1, 1, 1, 1).expand(1, F_, 3, H_, W_), torch.arange(F_)[None], ["s"], ["d"],
                  extrinsics=ext.float() if with_gt else None, intrinsics=k.float() if with_gt else None)
    cfg = OverfitCfg(intrinsics="softmin", softmin_points=500, regression_after=4, regression_window=2,
                     use_tracking=True, tracking_enable_after=2)
    o = FusedOverfitter(cfg, batch, Flows(*(t.float() for t in (fl.forward, fl.backward, fl.forward_mask,
                                                                 fl.backward_mask))),
                        [Tracks(t.xy.float(), t.visibility, t.start_frame) for t in tracks])
    o._clock.base_seed = 1234  # the same softmin samples in every run
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        o.model.backbone.depth.copy_((depth * (1 + 0.05 * torch.randn(depth.shape, generator=g, dtype=depth.dtype)))
                                     .float())
    o.use_cuda_graph = graph
    if capacity:
        o.enable_metrics_log(capacity)
    gt = ext[0, :, :3, 3].float().cuda()
    rec = dict(total=[], ate=[], k4=[], launches=[])
    L = _lib.lib()
    for _ in range(STEPS):
        n0 = L.fm_launch_count()
        total, _ = o.training_step()
        rec["launches"].append(L.fm_launch_count() - n0)
        rec["total"].append(total.cpu())
        rec["ate"].append(ate.trajectory_ate(gt, o.extrinsics()[0, :, :3, 3])[0].cpu())
        rec["k4"].append(o.intrinsics_k4().double().cpu())
    rec["depth"] = o.model.backbone.depth.detach().clone()
    rec["weights"] = o.model.backbone.weights.detach().clone()
    rec["graphs"] = len(o._graphs)
    return rec, (o.metrics_log() if capacity else None), k


@pytest.mark.gpu
@pytest.mark.parametrize("capacity", [16, 4])
def test_metrics_log_rows_match_the_steps(capacity):
    rec, log, k = _run(capacity)
    assert rec["graphs"] >= 1  # the regressed stage ran as a replayed graph
    keep = range(STEPS - min(capacity, STEPS), STEPS)  # a ring keeps the last `capacity` rows, in order
    assert all(v.shape == (len(keep),) for v in log.values())
    fx_gt, fy_gt = k[0, :, 0, 0].mean(), k[0, :, 1, 1].mean()
    for row, s in enumerate(keep):
        flow, track = log["train/loss/flow"][row], log["train/loss/tracking"][row]
        assert torch.equal(log["metrics/ate"][row], rec["ate"][s]), (s, log["metrics/ate"][row], rec["ate"][s])
        assert torch.equal(flow + track, rec["total"][s]), s
        assert (float(track) == 0.0) == (s < 2), (s, float(track))
        k4 = rec["k4"][s]
        assert abs(float(log["train/intrinsics/fx_error"][row]) - float((fx_gt - k4[:, 0].mean()).abs())) <= 1e-7
        assert abs(float(log["train/intrinsics/fy_error"][row]) - float((fy_gt - k4[:, 1].mean()).abs())) <= 1e-7


@pytest.mark.gpu
def test_metrics_log_without_ground_truth_is_nan():
    rec, log, _ = _run(16, with_gt=False)
    for name in ("train/intrinsics/fx_error", "train/intrinsics/fy_error", "metrics/ate"):
        assert torch.isnan(log[name]).all(), name
    assert torch.equal(log["train/loss/flow"] + log["train/loss/tracking"], torch.stack(rec["total"]))


@pytest.mark.gpu
def test_metrics_log_leaves_the_optimisation_unchanged():
    """Log on vs off: the same losses and parameters up to the run-to-run noise of the float atomics,
    and per step one more launch with the tracking loss, two without (the pose chain).  Launches are
    counted on the eager steps (graph replays launch nothing from the host).

    The parameters after 10 Adam steps carry that noise amplified: Adam divides each gradient by its own
    running magnitude, so the last bits of a near-zero gradient move its parameter by up to the learning
    rate.  Runs with the log off differ from each other by 1e-8 to 5e-7 in the weights (four runs on one
    H100), and a run with the log on was seen 1.1e-6 away.  So the parameters are held to 1e-6 or 3x the
    largest difference among three runs without the log, whichever is larger."""
    on, _, _ = _run(16)
    offs = [_run(0)[0] for _ in range(3)]
    off = offs[0]
    for s in range(STEPS):
        a, b = float(on["total"][s]), float(off["total"][s])
        assert abs(a - b) <= 1e-6 * abs(b), (s, a, b)
    for name in ("depth", "weights"):
        e = rel_l2(on[name], off[name])
        noise = max(rel_l2(offs[i][name], offs[j][name]) for i in range(3) for j in range(i + 1, 3))
        print(f"{name}: log on vs off {e:.1e}, off vs off {noise:.1e}")
        assert e <= max(1e-6, 3 * noise), (name, e, noise)
    extra = [a - b for a, b in zip(on["launches"][:6], off["launches"][:6])]  # steps 0-5 run eagerly
    assert extra == [2, 2, 1, 1, 1, 1], extra


@pytest.mark.gpu
def test_step0_ate_at_the_exact_scene_matches_float64_oracle():
    """Started at the scene's exact depth and focal length, the logged ATE of step 0 is that of the
    float64 oracle's own Procrustes poses."""
    from ate_oracle import trajectory_ate
    from oracle import flowmap_oracle as O
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows
    depth, fl, focal, ext, _, k = _scene()
    st = O.OverfitOracle(O.OverfitConfig(intrinsics="regressed", initial_focal=focal), F_, H_, W_,
                         dtype=torch.float64)
    with torch.no_grad():
        st.depth.copy_(depth)
    poses = st.forward(fl, step=0).extrinsics.detach()
    ref = trajectory_ate(ext[0, :, :3, 3], poses[0, :, :3, 3])[0]
    batch = Batch(torch.zeros(1, 1, 1, 1, 1).expand(1, F_, 3, H_, W_), torch.arange(F_)[None], ["s"], ["d"],
                  extrinsics=ext.float(), intrinsics=k.float())
    o = FusedOverfitter(OverfitCfg(initial_focal=focal), batch,
                        Flows(*(t.float() for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask))))
    with torch.no_grad():
        o.model.backbone.depth.copy_(depth.float())
    o.enable_metrics_log(4)
    o.training_step()
    log = o.metrics_log()
    assert abs(float(log["metrics/ate"][0]) - float(ref)) <= 1e-5, (float(log["metrics/ate"][0]), float(ref))
    assert float(log["train/intrinsics/fx_error"][0]) <= 1e-6  # the exact focal length
