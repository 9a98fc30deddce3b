"""`-m gpu`: B networks, each overfitting its own video, as one fused step (flowmap_b200.fused.network_videos_step
on a FusedOverfitter bound to a list of network Models, the packed split halves of fm_overfit_step_videos).

Video b must get what a one-video network-bound fused step on it gets (Model.forward and the losses of
test_gpu_network_backbone.py, the reference-shaped surface): its flow loss by its own mask sum, its tracking
loss by its own valid count, its own softmin window, hand-over and focal length, and its gradients scaled by
its own grad_output.  The stand-in backbones are those of test_gpu_network_backbone.py."""
import copy
from dataclasses import replace

import pytest
import torch

from conftest import rel_l2
from test_gpu_network_backbone import _assert_close, _oracle_grads, _setup, _step

H_, W_ = 40, 64


def _ground_truth_k(f, b, scale=1.0):
    """A normalised K per frame, (1, f, 3, 3), different for every frame and video."""
    k = torch.zeros(1, f, 3, 3)
    t = torch.arange(f, dtype=torch.float32)
    k[0, :, 0, 0] = scale * (0.9 + 0.03 * b + 0.01 * t)
    k[0, :, 1, 1] = scale * (1.2 + 0.02 * b - 0.01 * t)
    k[0, :, 0, 2], k[0, :, 1, 2], k[0, :, 2, 2] = 0.5 + 0.01 * b, 0.49 + 0.002 * t, 1.0
    return k.cuda()


def _with_ground_truth(v, b):
    """(model, losses, batch, flows, tracks) of a regressed setup turned into ground-truth K: the same network
    under IntrinsicsGroundTruth, and the batch carrying its K."""
    from flowmap_b200.model import IntrinsicsGroundTruthCfg, Model, ModelCfg
    model, losses, batch, flows, tracks = v
    mc, f = model.cfg, batch.videos.shape[1]
    gt = Model(ModelCfg(mc.backbone, IntrinsicsGroundTruthCfg("ground_truth"), mc.extrinsics,
                        mc.use_correspondence_weights), f, (H_, W_)).cuda()
    gt.backbone.load_state_dict(model.backbone.state_dict())
    return gt, losses, replace(batch, intrinsics=_ground_truth_k(f, b)), flows, tracks


def _videos(frames, intrinsics="regressed", tracking=False, use_weights=True, regression=None, tracking_after=0,
            kind="mlp_original", points=None):
    """One (model, losses, batch, flows, tracks) per video, each with its own network (seeded by b), and a copy
    of every model for its solo run.  intrinsics "ground_truth": a K per frame and video in batch.intrinsics."""
    gt = intrinsics == "ground_truth"
    vids = [_setup(kind, "regressed" if gt else intrinsics, tracking, use_weights, points, f=f, h=H_, w=W_, seed=b,
                   regression=regression, tracking_after=tracking_after) for b, f in enumerate(frames)]
    if gt:
        vids = [_with_ground_truth(v, b) for b, v in enumerate(vids)]
    solo = [copy.deepcopy(v[0]) for v in vids]
    for s, v in zip(solo, vids):
        if hasattr(v[0].intrinsics, "injected_indices"):
            s.intrinsics.injected_indices = v[0].intrinsics.injected_indices
    return vids, solo


def _engine(vids, tracking, tracking_after=0):
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    models = [v[0] for v in vids]
    cfg = OverfitCfg(**models[0]._overfit_fields(), flow_weight=1000.0, flow_enable_after=0,
                     use_tracking=tracking, tracking_enable_after=tracking_after, tracking_weight=100.0,
                     mapping="huber", delta=0.01)
    return FusedOverfitter(cfg, [v[2] for v in vids], [v[3] for v in vids],
                           [v[4] for v in vids] if tracking else None, device="cuda:0", model=models)


def _batched_step(eng, vids, step, c=None, zero=True, intrinsics=None, inputs=None):
    """The networks' outputs concatenated along the frame axis, one fused step, (c * (flow + tracking)).sum()
    backward.  Returns each video's [flow, tracking] losses and parameter gradients; `inputs` (a list) receives
    the packed depths and weights with their gradients."""
    from flowmap_b200.fused import network_videos_step
    models = [v[0] for v in vids]
    if zero:
        for m in models:
            m.zero_grad(set_to_none=True)
    outs = [m.backbone(v[2], v[3]) for m, v in zip(models, vids)]
    depths = torch.cat([o.depths[0] for o in outs])
    weights = torch.cat([o.weights[0] for o in outs]) if eng.cfg.use_correspondence_weights else None
    if inputs is not None:
        depths.retain_grad()
        weights.retain_grad()
        inputs += [depths, weights]
    flow, track = network_videos_step(eng, depths, weights, step, intrinsics=intrinsics)
    c = torch.ones(len(vids), device=flow.device) if c is None else c
    (c * (flow + track)).sum().backward()
    losses = [[float(flow[b]), float(track[b])] for b in range(len(vids))]
    grads = [{n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None} for m in models]
    return losses, grads


def _solo_step(solo, v, step, scale=None):
    _, losses, batch, flows, tracks = v
    parts, grads, _ = _step(solo, losses, batch, flows, tracks, fused=True, scale=scale, step=step)
    if len(parts) == 1:
        parts = parts + [0.0]
    return parts, grads


def _compare(vids, solo, eng, step, tracking, softmin, c=None, intrinsics=None):
    lb, gb = _batched_step(eng, vids, step, c, intrinsics=intrinsics)
    for b, (s, v) in enumerate(zip(solo, vids)):
        ls, gs = _solo_step(s, v, step, None if c is None else float(c[b]))
        if not tracking:
            lb[b][1] = 0.0
        # tracking losses before enable_after: the solo surface reports 0, the step 0 too
        _assert_close(ls, gs, lb[b], gb[b], softmin)


CASES = [(frames, intr, tracking, uw, pts) for frames in ((5, 5), (6, 4, 7), (5, 3, 6, 4))
         for intr in ("regressed", "softmin", "ground_truth") for tracking in (False, True) for uw in (True, False)
         for pts in (None, 1000)]


@pytest.mark.gpu
@pytest.mark.parametrize("frames,intrinsics,tracking,use_weights,points", CASES)
def test_batched_equals_solo(frames, intrinsics, tracking, use_weights, points):
    """Equal and different lengths (the grids' pairs cross video boundaries), B = 2, 3 and 4, regressed and
    softmin focal lengths and ground-truth K (a different K for every frame), with and without weights and tracks,
    all-pixel and 1000-point Procrustes: every video's losses and parameter gradients (network and focal length)
    match its one-video network-bound step."""
    vids, solo = _videos(frames, intrinsics, tracking, use_weights, points=points)
    eng = _engine(vids, tracking)
    _compare(vids, solo, eng, 0, tracking, intrinsics == "softmin")


@pytest.mark.gpu
@pytest.mark.parametrize("points", [None, 1000])
def test_regression_stage_equals_solo(points):
    """Softmin with a regression stage (window 2, hand-over at step 2), tracks from step 1: at every step, before,
    at and after each model's hand-over, every video's losses and gradients, the regressed focal length's
    included, match its solo step, and every model's window holds its solo estimates."""
    vids, solo = _videos((6, 4, 5), "softmin", tracking=True, regression=(2, 2), tracking_after=1, points=points)
    eng = _engine(vids, True, tracking_after=1)
    for step in range(4):
        _compare(vids, solo, eng, step, step >= 1, step < 2)
    for s, v in zip(solo, vids):
        assert rel_l2(torch.stack(v[0].intrinsics.window), torch.stack(s.intrinsics.window)) <= 1e-5
        fs, fb = s.intrinsics.intrinsics_regressed.focal_length, v[0].intrinsics.intrinsics_regressed.focal_length
        assert abs(float(fb) - float(fs)) <= 1e-5 * abs(float(fs))


@pytest.mark.gpu
def test_ground_truth_k_read_every_step():
    """Ground-truth K rewritten in place between steps: network_videos_step(intrinsics=...) reads this step's K,
    as the one-video surface reads batch.intrinsics on every step."""
    vids, solo = _videos((6, 4, 5), "ground_truth", tracking=True)
    eng = _engine(vids, True)
    _compare(vids, solo, eng, 0, True, False)
    for b, v in enumerate(vids):
        v[2].intrinsics.copy_(_ground_truth_k(v[2].videos.shape[1], b, scale=1.3))
    _compare(vids, solo, eng, 1, True, False, intrinsics=[v[2].intrinsics for v in vids])


def _oracle(depths, weights, model, batch, flows, tracks, idx, dtype):
    """_oracle_grads of test_gpu_network_backbone.py, and with ground-truth intrinsics the same total on the
    batch's own K."""
    from flowmap_b200.model import IntrinsicsGroundTruth
    if not isinstance(model.intrinsics, IntrinsicsGroundTruth):
        return _oracle_grads(depths, weights, model, flows, tracks, idx, dtype)
    from oracle import flowmap_oracle as O
    _, f, h, w = depths.shape
    d = depths.detach().to("cpu", dtype).requires_grad_(True)
    wt = weights.detach().to("cpu", dtype).requires_grad_(True)
    fl = O.Flows(*(t.detach().to("cpu", dtype) for t in (flows.forward, flows.backward, flows.forward_mask,
                                                        flows.backward_mask)))
    k = batch.intrinsics.detach().to("cpu", dtype)
    surf = O.unproject(O.pixel_grid(h, w, dtype), d, k[:, :, None, None])
    ext = O.align_surfaces(surf, fl.backward, wt, idx)
    total = 1000.0 * O.flow_loss(surf, ext, k, fl, "huber", 0.01)
    ot = [O.Tracks(t.xy.to("cpu", dtype), t.visibility.cpu(), t.start_frame) for t in tracks]
    total = total + 100.0 * O.tracking_loss(surf, ext, k, ot, "huber", 0.01)
    total.backward()
    return d.grad, wt.grad


@pytest.mark.gpu
@pytest.mark.parametrize("intrinsics,points", [("regressed", None), ("softmin", None), ("regressed", 1000),
                                               ("ground_truth", None)])
def test_input_gradients_vs_float64_oracle(intrinsics, points):
    """A tracked configuration of B = 3 videos of different lengths: every video's d loss / d depths and
    d loss / d weights of the batched step against the float64 oracle on its own depths and weights, within
    max(5e-4, 4 x the float32 oracle's own error), as test_gpu_network_backbone.py checks one video."""
    vids, _ = _videos((6, 4, 5), intrinsics, tracking=True, points=points)
    eng = _engine(vids, True)
    inputs = []
    _batched_step(eng, vids, 0, inputs=inputs)
    depths, weights = inputs
    f0 = 0
    for b, (model, _, batch, flows, tracks) in enumerate(vids):
        f = batch.videos.shape[1]
        d, w = depths[f0:f0 + f][None], weights[f0 - b:f0 - b + f - 1][None]
        idx = model.extrinsics.select_indices(H_, W_, d.device)
        idx = torch.arange(H_ * W_) if idx is None else idx.cpu()
        gd64, gw64 = _oracle(d, w, model, batch, flows, tracks, idx, torch.float64)
        gd32, gw32 = _oracle(d, w, model, batch, flows, tracks, idx, torch.float32)
        for name, got, ref, f32 in (("depths", depths.grad[f0:f0 + f][None], gd64, gd32),
                                    ("weights", weights.grad[f0 - b:f0 - b + f - 1][None], gw64, gw32)):
            err, noise = rel_l2(got.cpu(), ref), rel_l2(f32, ref)
            assert err <= max(5e-4, 4.0 * noise), (b, name, err, noise)
        f0 += f


@pytest.mark.gpu
@pytest.mark.parametrize("intrinsics", ["regressed", "softmin"])
def test_per_video_grad_output(intrinsics):
    """(c * (flow + tracking)).sum().backward() with distinct c_b: video b gets c_b times its solo gradients."""
    vids, solo = _videos((6, 4, 5), intrinsics, tracking=True)
    eng = _engine(vids, True)
    c = torch.tensor([0.5, 2.0, -1.25], device="cuda:0")
    _compare(vids, solo, eng, 0, True, intrinsics == "softmin", c)


@pytest.mark.gpu
def test_adam_run_across_tracking_switch_on_and_hand_over():
    """B = 3, torch Adam per network: steps 0..5 with the tracking loss from step 1 and the softmin ->
    regressed hand-over at step 4 (window 2).  Every network's parameters and focal length track its solo run,
    and every model's window holds its own estimates."""
    frames, steps = (6, 4, 5), 6
    vids, solo = _videos(frames, "softmin", tracking=True, regression=(4, 2), tracking_after=1)
    eng = _engine(vids, True, tracking_after=1)
    opt_b = [torch.optim.Adam(v[0].parameters(), lr=1e-4) for v in vids]
    opt_s = [torch.optim.Adam(s.parameters(), lr=1e-4) for s in solo]
    for step in range(steps):
        _batched_step(eng, vids, step)
        for o in opt_b:
            o.step()
        for s, v, o in zip(solo, vids, opt_s):
            _solo_step(s, v, step)
            o.step()
    for b, (s, v) in enumerate(zip(solo, vids)):
        ws, wb = torch.stack(s.intrinsics.window), torch.stack(v[0].intrinsics.window)
        assert ws.shape == wb.shape == (2,)
        assert rel_l2(wb, ws) <= 1e-4, (b, wb, ws)
        fs, fb = s.intrinsics.intrinsics_regressed.focal_length, v[0].intrinsics.intrinsics_regressed.focal_length
        assert abs(float(fb) - float(fs)) <= 1e-4 * abs(float(fs)), (b, float(fb), float(fs))
        for (n, pb), (_, ps) in zip(v[0].named_parameters(), s.named_parameters()):
            assert rel_l2(pb, ps) <= 1e-4, (b, n, rel_l2(pb, ps))
    # the videos are different: their windows are too
    assert float(torch.stack(vids[0][0].intrinsics.window).sum()) != float(torch.stack(vids[1][0].intrinsics.window).sum())


@pytest.mark.gpu
def test_refusals():
    """Explicit-depth models, a model count other than B, models whose cfg differs from each other or from
    `cfg`, the metrics log and checkpoints."""
    from flowmap_b200.model import IntrinsicsRegressedCfg, Model, ModelCfg
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg, build_model_and_losses
    vids, _ = _videos((5, 4), "regressed")
    models = [v[0] for v in vids]
    base = OverfitCfg(**models[0]._overfit_fields())
    batches, flows = [v[2] for v in vids], [v[3] for v in vids]
    with pytest.raises(ValueError, match="one network Model per video"):
        FusedOverfitter(base, batches, flows, device="cuda:0", model=models[:1])
    explicit = build_model_and_losses(OverfitCfg(), 4, (H_, W_))[0].cuda()
    with pytest.raises(ValueError, match="network backbone"):
        FusedOverfitter(base, batches, flows, device="cuda:0", model=[models[0], explicit])
    other = Model(ModelCfg(models[0].cfg.backbone, IntrinsicsRegressedCfg("regressed", 0.7),
                           models[0].cfg.extrinsics, True), 4, (H_, W_)).cuda()
    with pytest.raises(ValueError, match="differs from model 0"):
        FusedOverfitter(base, batches, flows, device="cuda:0", model=[models[0], other])
    with pytest.raises(ValueError, match="does not describe"):
        FusedOverfitter(OverfitCfg(**{**models[0]._overfit_fields(), "procrustes_points": 1000}), batches, flows,
                        device="cuda:0", model=models)
    eng = FusedOverfitter(base, batches, flows, device="cuda:0", model=models)
    with pytest.raises(ValueError, match="metrics log"):
        eng.enable_metrics_log(4)
    with pytest.raises(ValueError, match="Adam state"):
        eng.state_dict()
