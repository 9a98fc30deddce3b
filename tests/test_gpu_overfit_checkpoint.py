"""`-m gpu`: saving and resuming a FusedOverfitter run (state_dict / load_state_dict), and moving a run
between it and the reference-shaped loop (Model -> losses -> backward() -> torch.optim.Adam) through
flowmap_b200.checkpoint.

The kernels add floats with atomics, so two runs agree to float noise only: a resumed run is compared with
the uninterrupted one within the tolerances of test_gpu_batched_overfit.py (packed against one-video runs)
or test_gpu_dropin_fused.py (the reference-shaped surface), and negative controls show that those
tolerances catch a broken resume."""
import io

import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu
H, W = 40, 64
DEV = torch.device("cuda:0")


def _equal(a, b, path="state"):
    if isinstance(a, torch.Tensor):
        assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.device == b.device, path
        assert torch.equal(a, b), path
    elif isinstance(a, dict):
        assert isinstance(b, dict) and set(a) == set(b), path
        for k in a:
            _equal(a[k], b[k], f"{path}[{k!r}]")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _equal(x, y, f"{path}[{i}]")
    else:
        assert a == b, (path, a, b)


def _saved(state):
    """`state` written with torch.save and read back."""
    buf = io.BytesIO()
    torch.save(state, buf)
    buf.seek(0)
    return torch.load(buf)


def _video(f, seed):
    """One video's (Batch, Flows, tracks, depth, logits), with ground-truth K, on the GPU."""
    import bench
    from flowmap_b200.types import Batch, Flows, Tracks
    inp = bench.synthetic_inputs(f, H, W, seed=seed)
    k = torch.eye(3).repeat(1, f, 1, 1)
    k[..., 0, 0], k[..., 1, 1], k[..., :2, 2] = 0.8 + 0.01 * seed, 0.9, 0.5
    batch = Batch(torch.zeros(1, f, 3, H, W, device=DEV), torch.arange(f, device=DEV)[None], ["s"], ["d"],
                  intrinsics=k.to(DEV))
    flows = Flows(*(inp[n].to(DEV) for n in ("fwd", "bwd", "fmask", "bmask")))
    tracks = [Tracks(xy.to(DEV), vis.to(DEV), s)
              for xy, vis, s in bench.synthetic_track_arrays(f, n_points=40 + 8 * seed, interval=3, radius=2, seed=seed)]
    return batch, flows, tracks, (1.0 + inp["depth"]).to(DEV), inp["wparam"].to(DEV)


def _inputs(form, frames=6):
    """FusedOverfitter inputs of one video, a B = 3 tensor batch or a list of 3 lengths, and the initial
    depth / logits of every video."""
    from flowmap_b200.types import Batch, Flows
    lengths = {"one": [frames], "tensor": [frames] * 3, "list": [frames - 1, frames, frames + 1]}[form]
    vids = [_video(f, i) for i, f in enumerate(lengths)]
    init = [(v[3], v[4]) for v in vids]
    if form == "one":
        return vids[0][0], vids[0][1], vids[0][2], init
    if form == "list":
        return [v[0] for v in vids], [v[1] for v in vids], [v[2] for v in vids], init
    bt = [v[0] for v in vids]
    batch = Batch(torch.cat([b.videos for b in bt]), torch.cat([b.indices for b in bt]), ["s"] * 3, ["d"] * 3,
                  intrinsics=torch.cat([b.intrinsics for b in bt]))
    flows = Flows(*(torch.cat([getattr(v[1], n) for v in vids])
                    for n in ("forward", "backward", "forward_mask", "backward_mask")))
    return batch, flows, [v[2] for v in vids], init


def _build(cfg, inputs, graph=True):
    from flowmap_b200.overfit import FusedOverfitter
    batch, flows, tracks, init = inputs
    o = FusedOverfitter(cfg, batch, flows, tracks if cfg.use_tracking else None, device=DEV)
    with torch.no_grad():
        for m, (d, wl) in zip(o.models, init):
            m.backbone.depth.copy_(d)
            m.backbone.weights.copy_(wl)
    o.use_cuda_graph = graph
    return o


def _cfg(intrinsics, tracking, **kw):
    from flowmap_b200.overfit import OverfitCfg
    extra = dict(regression_after=4, regression_window=2) if intrinsics == "softmin" else {}
    return OverfitCfg(**{**dict(intrinsics=intrinsics, use_tracking=tracking, tracking_enable_after=1,
                                softmin_points=500), **extra, **kw})


# ------------------------------------------------------------------------------------------- round trip
@pytest.mark.parametrize("form", ["one", "tensor", "list"])
@pytest.mark.parametrize("intrinsics", ["softmin", "regressed", "ground_truth"])
@pytest.mark.parametrize("tracking", [False, True])
def test_state_round_trip(form, intrinsics, tracking):
    """state_dict -> torch.save -> load_state_dict on a fresh optimiser -> state_dict gives the same state,
    tensor for tensor; the snapshot synchronises nothing with the host.  5 steps: the softmin run has
    crossed its hand-over (a window of 2 and one focal update)."""
    cfg = _cfg(intrinsics, tracking)
    inputs = _inputs(form)
    o = _build(cfg, inputs)
    for _ in range(5):
        o.training_step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        s1 = o.state_dict()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    b = len(o.models)
    assert (s1["global_step"], s1["optimizer_steps"]) == (5, 5) and len(s1["videos"]) == b
    if intrinsics == "softmin":
        assert s1["focal_steps"] == 1 and s1["window"].shape == ((2,) if b == 1 else (2, b))
    else:
        assert s1["window"] is None and s1["focal_steps"] == (5 if intrinsics == "regressed" else 0)
    for m, v in zip(o.models, s1["videos"]):
        _equal(v["model"], {k: t.detach() for k, t in m.state_dict().items()})
        assert set(v["optimizer"]["state"]) == ({0, 1} if intrinsics == "ground_truth" else {0, 1, 2})
    o2 = _build(cfg, _inputs(form))
    o2.load_state_dict(_saved(s1))
    _equal(o2.state_dict(), s1)


# ------------------------------------------------------------------------------------------- continuation
STEPS, KS = 60, (3, 5, 35, 40, 50)


def _trajectory(o, steps):
    """Run `steps` update steps: per step the totals and the packed rt."""
    totals, rts = [], []
    for _ in range(steps):
        total, _ = o.training_step()
        totals.append(total.reshape(-1).clone())
        rts.append(o.rt.clone())
    return torch.stack(totals), torch.stack(rts)


def _final(o):
    s = o._state
    return {"depth": o._depth.clone(), "logits": o._wlog.clone(), "focal": o._focal.reshape(-1).clone(),
            "m_depth": s[0].clone(), "v_depth": s[1].clone(), "m_logits": s[2].clone(), "v_logits": s[3].clone(),
            "m_focal": s[4].reshape(-1).clone(), "v_focal": s[5].reshape(-1).clone()}


def _errors(ref, got):
    """Each quantity's error over its tolerance (test_gpu_batched_overfit.py's, no looser)."""
    (tr, rr, fr), (tg, rg, fg) = ref, got
    e = {"totals": float(((tg - tr).abs() / tr.abs().clamp_min(1e-30)).max()) / 1e-5,
         "rt": float((rg - rr).abs().max()) / 2e-6,
         "depth": rel_l2(fg["depth"], fr["depth"]) / 1e-5,
         "logits": float((fg["logits"] - fr["logits"]).abs().max()) / 1e-5,
         "focal": float(((fg["focal"] - fr["focal"]).abs() / fr["focal"].abs()).max()) / 1e-6}
    # Adam's moments average the gradients, which two evaluation orders give to float noise: rel. L2 2e-4 in
    # the softmin stage on the reference-shaped surface (test_gpu_dropin_fused.py); 1e-4 here
    for k in ("m_depth", "v_depth", "m_logits", "v_logits"):
        e[k] = rel_l2(fg[k], fr[k]) / 1e-4
    # d loss / d focal is a small difference of large sums, float noise ~1e-4 (test_gpu_dropin_fused.py)
    for k in ("m_focal", "v_focal"):
        e[k] = rel_l2(fg[k], fr[k]) / 5e-4
    return e


@pytest.mark.parametrize("form", ["one", "list"])
def test_resume_continues_the_run(form):
    """A run saved after K steps, rebuilt, loaded and run to step 60 follows the uninterrupted run: K = 3
    before the tracking loss starts, 5 its first step, 35 inside the hand-over window, 40 the hand-over
    itself, 50 after it.  Resuming with zeroed moments or another seed misses the tolerances by >= 10x."""
    cfg = _cfg("softmin", True, regression_after=40, regression_window=10, tracking_enable_after=5)
    inputs = _inputs(form)
    o = _build(cfg, inputs)
    states, totals, rts = {}, [], []
    for k in range(STEPS):
        if k in KS:
            states[k] = _saved(o.state_dict())
        t, r = _trajectory(o, 1)
        totals.append(t)
        rts.append(r)
    totals, rts, final = torch.cat(totals), torch.cat(rts), _final(o)
    assert len(o._graphs) >= 2

    def resume(state, k):
        r = _build(cfg, inputs)
        r.load_state_dict(state)
        t, rt = _trajectory(r, STEPS - k)
        return (totals[k:], rts[k:], final), (t, rt, _final(r))

    for k in KS:
        errs = _errors(*resume(states[k], k))
        print(form, k, {n: f"{e:.3g}" for n, e in errs.items()})
        assert max(errs.values()) <= 1.0, (k, errs)
    k = 35
    zeroed = _saved(states[k])
    for v in zeroed["videos"]:
        for e in v["optimizer"]["state"].values():
            e["exp_avg"].zero_()
            e["exp_avg_sq"].zero_()
    reseeded = {**states[k], "base_seed": states[k]["base_seed"] + 1}
    for name, bad in (("zeroed moments", zeroed), ("another seed", reseeded)):
        errs = _errors(*resume(bad, k))
        print(form, name, {n: f"{e:.3g}" for n, e in errs.items()})
        assert max(errs.values()) >= 10.0, (name, errs)


# ------------------------------------------------------------------------------------------- interchange
def _reference_loop(cfg, model, losses, opt, batch, flows, tracks, steps):
    """Model.forward -> losses -> backward() -> torch.optim.Adam at global steps `steps`: the totals."""
    totals = []
    for step in steps:
        opt.zero_grad()
        out = model(batch, flows, step)
        total = sum(l.forward(batch, flows, tracks, out, step) for l in losses)
        total.backward()
        opt.step()
        totals.append(total.detach().reshape(1))
    return torch.cat(totals)


@pytest.mark.parametrize("k", [2, 4, 7])
def test_fused_run_continues_on_the_reference_loop(k):
    """K fused steps, then to_torch and torch.optim.Adam on the reference-shaped surface, across the softmin
    hand-over at step 6 (K = 2 before the window opens, 4 inside it, 7 after the hand-over): the totals and
    parameters of the uninterrupted fused run.  Both sides draw the softmin sample from injected_indices."""
    from flowmap_b200 import checkpoint
    from flowmap_b200.overfit import build_model_and_losses
    n = 10
    cfg = _cfg("softmin", True, regression_after=6, regression_window=3)
    batch, flows, tracks, init = _inputs("one")
    idx = torch.randperm(H * W, generator=torch.Generator().manual_seed(3))[:500].to(DEV)
    o = _build(cfg, (batch, flows, tracks, init), graph=False)
    o.injected_indices = idx
    ref, state = [], None
    for step in range(n):
        if step == k:
            state = o.state_dict()
        ref.append(o.training_step()[0].reshape(1))
    ref = torch.cat(ref)
    msd, asd, gstep, window = checkpoint.to_torch(state)
    model, losses = build_model_and_losses(cfg, batch.videos.shape[1], (H, W))
    model.to(DEV)
    model.load_state_dict(msd)
    model.intrinsics.window = window
    model.intrinsics.injected_indices = idx
    opt = torch.optim.Adam(model.parameters(), lr=cfg.lr)
    opt.load_state_dict(asd)
    got = _reference_loop(cfg, model, losses, opt, batch, flows, tracks, range(gstep, n))
    assert float(((got - ref[k:]).abs() / ref[k:].abs()).max()) <= 1e-6, (got, ref[k:])
    assert rel_l2(model.backbone.depth.detach(), o.model.backbone.depth.detach()) <= 2e-4
    assert rel_l2(model.backbone.weights.detach(), o.model.backbone.weights.detach()) <= 2e-4
    f_ref = o.model.intrinsics.intrinsics_regressed.focal_length.detach()
    assert abs(float(model.intrinsics.intrinsics_regressed.focal_length.detach() - f_ref)) <= 5e-4 * abs(float(f_ref))


def test_reference_loop_continues_on_the_fused_run():
    """K steps of the reference-shaped loop with torch.optim.Adam, then from_torch and FusedOverfitter: the
    totals and parameters of the uninterrupted reference-shaped loop (regressed intrinsics, tracking on)."""
    from flowmap_b200 import checkpoint
    from flowmap_b200.overfit import build_model_and_losses
    n, k = 10, 4
    cfg = _cfg("regressed", True)
    batch, flows, tracks, init = _inputs("one")

    def fresh():
        model, losses = build_model_and_losses(cfg, batch.videos.shape[1], (H, W))
        model.to(DEV)
        with torch.no_grad():
            model.backbone.depth.copy_(init[0][0])
            model.backbone.weights.copy_(init[0][1])
        return model, losses, torch.optim.Adam(model.parameters(), lr=cfg.lr)

    model, losses, opt = fresh()
    ref = _reference_loop(cfg, model, losses, opt, batch, flows, tracks, range(n))
    model2, losses2, opt2 = fresh()
    _reference_loop(cfg, model2, losses2, opt2, batch, flows, tracks, range(k))
    state = checkpoint.from_torch(cfg, model2, opt2, k)
    assert (state["optimizer_steps"], state["focal_steps"]) == (k, k)
    o = _build(cfg, (batch, flows, tracks, init))
    o.load_state_dict(_saved(state))
    got, _ = _trajectory(o, n - k)
    assert float(((got[:, 0] - ref[k:]).abs() / ref[k:].abs()).max()) <= 1e-6, (got, ref[k:])
    assert rel_l2(o.model.backbone.depth.detach(), model.backbone.depth.detach()) <= 2e-5
    assert rel_l2(o.model.backbone.weights.detach(), model.backbone.weights.detach()) <= 2e-5
    f_ref = model.intrinsics.focal_length.detach()
    assert abs(float(o.model.intrinsics.focal_length.detach() - f_ref)) <= 5e-4 * abs(float(f_ref))


# ------------------------------------------------------------------------------------------- regrouping
def test_merged_runs_continue_as_one_packed_run():
    """Three one-video regressed runs (all-pixel Procrustes, tracking on) for K steps, merged into one list-of-
    videos optimiser: each video continues as it would alone, within the packed-versus-one-video tolerance.
    merge refuses states whose counters differ."""
    from flowmap_b200 import checkpoint
    n, k = 10, 4
    cfg = _cfg("regressed", True)
    batches, flows, tracks, init = _inputs("list")
    solos = [_build(cfg, (batches[i], flows[i], tracks[i], [init[i]])) for i in range(3)]
    for s in solos:
        _trajectory(s, k)
    states = [_saved(s.state_dict()) for s in solos]
    packed = _build(cfg, (batches, flows, tracks, init))
    packed.load_state_dict(checkpoint.merge(states))
    tp, rp = _trajectory(packed, n - k)
    rp_videos = packed._per_video(rp.transpose(0, 1), pairs=True)
    for i, s in enumerate(solos):
        ts, rs = _trajectory(s, n - k)
        assert float(((tp[:, i] - ts[:, 0]).abs() / ts[:, 0].abs()).max()) <= 1e-6, i
        assert float((rp_videos[i].transpose(0, 1) - rs[:, 0]).abs().max()) <= 2e-6, i
        assert rel_l2(packed.models[i].backbone.depth.detach(), s.model.backbone.depth.detach()) <= 1e-5, i
        assert float((packed.models[i].backbone.weights.detach() - s.model.backbone.weights.detach()).abs().max()) <= 1e-5
        fp, fs = (float(m.intrinsics.focal_length.detach()) for m in (packed.models[i], s.model))
        assert abs(fp - fs) <= 1e-6 * abs(fs), i
    _trajectory(solos[0], 1)
    with pytest.raises(ValueError, match="'global_step'"):
        checkpoint.merge([solos[0].state_dict()] + states[1:])


# ------------------------------------------------------------------------------------------- refusals
def test_load_refuses_another_optimiser_and_unowned_state():
    """load_state_dict names the field that differs (format, cfg, number of videos, frames, H x W,
    intrinsics mode); a Model-bound optimiser, explicit or network, keeps no Adam state to save or load."""
    from dataclasses import replace
    from flowmap_b200 import checkpoint
    from flowmap_b200.overfit import FusedOverfitter, build_model_and_losses
    cfg = _cfg("regressed", False)
    inputs = _inputs("one")
    o = _build(cfg, inputs, graph=False)
    o.training_step()
    state = o.state_dict()
    other = {
        "'format'": {**state, "format": 2},
        "'cfg.lr'": {**state, "cfg": {**state["cfg"], "lr": 1e-3}},
        "'videos'": checkpoint.merge([state, state]),
        "'frames'": _build(cfg, _inputs("one", frames=5), graph=False).state_dict(),
        "'intrinsics'": _build(replace(cfg, intrinsics="ground_truth"), inputs, graph=False).state_dict(),
    }
    for match, bad in other.items():
        with pytest.raises(ValueError, match=match):
            o.load_state_dict(bad)
    v = state["videos"][0]
    wide = {**v, "model": {**v["model"], "backbone.depth": torch.zeros(6, H, W + 4, device=DEV)}}
    with pytest.raises(ValueError, match="'H x W'"):
        o.load_state_dict({**state, "videos": [wide]})

    batch, flows, _, _ = inputs
    model, _ = build_model_and_losses(cfg, 6, (H, W))
    bound = FusedOverfitter(cfg, batch, flows, device=DEV, model=model.to(DEV))
    model.backbone = torch.nn.Identity()  # a network backbone
    network = FusedOverfitter(cfg, batch, flows, device=DEV, model=model)
    for opt in (bound, network):
        with pytest.raises(ValueError, match="bound to a caller's Model"):
            opt.state_dict()
        with pytest.raises(ValueError, match="bound to a caller's Model"):
            opt.load_state_dict(state)
