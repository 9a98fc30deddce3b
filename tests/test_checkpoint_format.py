"""The checkpoint format of a FusedOverfitter run (flowmap_b200.checkpoint) on CPU tensors: its interchange
with torch.optim.Adam on the project's Model, split / merge, and the fields a load refuses."""
import io
from dataclasses import replace

import pytest
import torch

from flowmap_b200 import checkpoint
from flowmap_b200.overfit import OverfitCfg, build_model_and_losses

F, H, W = 4, 6, 8


def _equal(a, b, path="state"):
    """Tensors torch.equal (dtype and device included), everything else ==."""
    if isinstance(a, torch.Tensor):
        assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.device == b.device, path
        assert torch.equal(a, b), path
    elif isinstance(a, dict):
        assert isinstance(b, dict) and set(a) == set(b), (path, sorted(map(str, a)), sorted(map(str, b)))
        for k in a:
            _equal(a[k], b[k], f"{path}[{k!r}]")
    elif isinstance(a, (list, tuple)):
        assert type(a) is type(b) and len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _equal(x, y, f"{path}[{i}]")
    else:
        assert a == b, (path, a, b)


def _focal(model):
    intr = model.intrinsics
    return getattr(intr, "focal_length", None) if not hasattr(intr, "intrinsics_regressed") else \
        intr.intrinsics_regressed.focal_length


def _torch_run(cfg, steps=2, focal_steps=None, frames=F, seed=0, hw=(H, W)):
    """A reference-shaped run on CPU: Model of `cfg`, torch.optim.Adam over its parameters, `steps` updates
    with seeded gradients; the focal length (if any) receives gradients in the last `focal_steps` of them."""
    model, _ = build_model_and_losses(cfg, frames, hw)
    opt = torch.optim.Adam(model.parameters(), lr=cfg.lr)
    g = torch.Generator().manual_seed(seed)
    focal = _focal(model)
    focal_steps = steps if focal_steps is None else focal_steps
    for s in range(steps):
        opt.zero_grad()
        model.backbone.depth.grad = torch.randn(model.backbone.depth.shape, generator=g)
        if cfg.use_correspondence_weights:
            model.backbone.weights.grad = torch.randn(model.backbone.weights.shape, generator=g)
        if focal is not None and s >= steps - focal_steps:
            focal.grad = torch.randn((), generator=g)
        opt.step()
    return model, opt


CASES = {
    "weights": (OverfitCfg(), None),
    "no_weights": (OverfitCfg(use_correspondence_weights=False), None),
    "softmin_before_handover": (OverfitCfg(intrinsics="softmin", regression_after=10, regression_window=4), 0),
    "softmin_after_handover": (OverfitCfg(intrinsics="softmin", regression_after=10, regression_window=4), 1),
    "softmin_no_regression": (OverfitCfg(intrinsics="softmin", regression_after=None), None),
    "ground_truth": (OverfitCfg(intrinsics="ground_truth"), None),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_torch_state_survives_from_torch_and_to_torch(case):
    """Adam's state after two steps on the CPU Model goes through from_torch -> torch.save -> to_torch
    unchanged, and a fresh Model + torch.optim.Adam loaded from it continue exactly as the original."""
    cfg, focal_steps = CASES[case]
    model, opt = _torch_run(cfg, focal_steps=focal_steps)
    window = [torch.tensor(0.9), torch.tensor(0.95)] if "softmin_" in case and case != "softmin_no_regression" else None
    state = checkpoint.from_torch(cfg, model, opt, 7, window)
    expect_focal = {"weights": 2, "no_weights": 2, "softmin_after_handover": 1}.get(case, 0)
    assert (state["optimizer_steps"], state["focal_steps"]) == (2, expect_focal)
    buf = io.BytesIO()
    torch.save(state, buf)
    buf.seek(0)
    msd, asd, step, win = checkpoint.to_torch(torch.load(buf))
    _equal(msd, model.state_dict())
    _equal(asd, opt.state_dict())
    assert step == 7 and len(win) == (0 if window is None else 2)
    if window is not None:
        assert all(torch.equal(a, b) for a, b in zip(win, window))

    fresh, _ = build_model_and_losses(cfg, F, (H, W))
    fresh.load_state_dict(msd)
    fresh_opt = torch.optim.Adam(fresh.parameters(), lr=cfg.lr)
    fresh_opt.load_state_dict(asd)
    g = torch.Generator().manual_seed(5)
    grads = [torch.randn(p.shape, generator=g) for p in model.parameters()]
    for m, o in ((model, opt), (fresh, fresh_opt)):
        o.zero_grad()
        for p, gr in zip(m.parameters(), grads):
            p.grad = gr.clone()
        o.step()
    _equal(fresh.state_dict(), model.state_dict())
    _equal(fresh_opt.state_dict(), opt.state_dict())


def test_counters_come_from_the_adam_steps():
    cfg = OverfitCfg(intrinsics="softmin", regression_after=10, regression_window=4)
    model, opt = _torch_run(cfg, steps=3, focal_steps=1)
    s = checkpoint.from_torch(cfg, model, opt, 12, [torch.tensor(1.0)] * 4)
    assert (s["global_step"], s["optimizer_steps"], s["focal_steps"]) == (12, 3, 1)
    assert s["window"].shape == (4,) and isinstance(s["base_seed"], int)
    group = s["videos"][0]["optimizer"]["param_groups"][0]
    assert group["lr"] == cfg.lr and group["betas"] == (0.9, 0.999) and group["eps"] == 1e-8
    assert group["weight_decay"] == 0 and group["amsgrad"] is False and group["params"] == [0, 1, 2]
    assert s["videos"][0]["optimizer"]["state"][0]["step"].dtype == torch.float32


def test_from_torch_refuses_what_a_fused_step_cannot_continue():
    cfg = OverfitCfg()
    model, opt = _torch_run(cfg)
    opt.zero_grad()
    model.backbone.weights.grad = torch.ones_like(model.backbone.weights)
    opt.step()  # only the logits took a third update
    with pytest.raises(ValueError, match="depth has had 2 updates, the weight logits 3"):
        checkpoint.from_torch(cfg, model, opt, 3)
    model, _ = _torch_run(cfg)
    with pytest.raises(ValueError, match="optimizer.lr"):
        checkpoint.from_torch(cfg, model, torch.optim.Adam(model.parameters(), lr=1e-3), 0)
    with pytest.raises(ValueError, match="param group"):
        checkpoint.from_torch(cfg, model, torch.optim.Adam([model.backbone.depth], lr=cfg.lr), 0)
    with pytest.raises(ValueError, match="intrinsics"):
        checkpoint.from_torch(replace(cfg, intrinsics="softmin"), model, torch.optim.Adam(model.parameters()), 0)
    model.backbone = torch.nn.Identity()  # a network backbone: its state is the caller's optimiser's
    with pytest.raises(ValueError, match="explicit depth"):
        checkpoint.from_torch(cfg, model, torch.optim.Adam(model.parameters(), lr=cfg.lr), 0)


def _states(cfg, frames=(4, 5, 6), steps=2):
    out = []
    for i, f in enumerate(frames):
        model, opt = _torch_run(cfg, steps=steps, focal_steps=1, frames=f, seed=i)
        out.append(checkpoint.from_torch(cfg, model, opt, 9, [torch.tensor(0.8 + 0.1 * i), torch.tensor(0.7)]))
    return out


def test_merge_and_split():
    """merge packs the videos in order, with one column of the window each and the first state's seed;
    split gives the one-video states back."""
    cfg = OverfitCfg(intrinsics="softmin", regression_after=10, regression_window=4)
    states = _states(cfg)
    merged = checkpoint.merge(states)
    assert [v["frames"] for v in merged["videos"]] == [4, 5, 6] and merged["window"].shape == (2, 3)
    assert merged["base_seed"] == states[0]["base_seed"]
    checkpoint.check(merged, cfg, [4, 5, 6], (H, W))
    for one, back in zip(states, checkpoint.split(merged)):
        _equal(back, {**one, "base_seed": merged["base_seed"]})
    _equal(checkpoint.merge(states[:1]), states[0])
    _equal(checkpoint.split(states[1])[0], states[1])


def test_merge_refuses_what_one_optimiser_cannot_hold():
    cfg = OverfitCfg(intrinsics="softmin", regression_after=10, regression_window=4)
    states = _states(cfg)
    with pytest.raises(ValueError, match="optimizer_steps"):
        checkpoint.merge(states[:2] + _states(cfg, frames=(6,), steps=3))
    other = _states(replace(cfg, lr=1e-4))
    with pytest.raises(ValueError, match="'cfg'"):
        checkpoint.merge(states[:2] + other[2:])
    model, opt = _torch_run(cfg, focal_steps=1)
    wide, wide_opt = _torch_run(cfg, focal_steps=1, hw=(H, W + 4))
    with pytest.raises(ValueError, match="H x W"):
        checkpoint.merge([checkpoint.from_torch(cfg, model, opt, 9),
                          checkpoint.from_torch(cfg, wide, wide_opt, 9)])
    with pytest.raises(ValueError, match="window"):
        checkpoint.merge([states[0], {**states[1], "window": None}])


def test_check_names_the_field_that_differs():
    """What a FusedOverfitter's load_state_dict refuses: format, cfg, number of videos, frames per video,
    H x W and intrinsics mode; and Adam steps that do not match the counters."""
    cfg = OverfitCfg(intrinsics="softmin", regression_after=10, regression_window=4)
    state = checkpoint.merge(_states(cfg))
    frames = [4, 5, 6]
    checkpoint.check(state, cfg, frames, (H, W))
    cases = [
        ({**state, "format": 2}, cfg, frames, (H, W), "'format'"),
        (state, replace(cfg, flow_weight=10.0), frames, (H, W), "'cfg.flow_weight'"),
        (state, replace(cfg, intrinsics="regressed"), frames, (H, W), "'intrinsics'"),
        (state, cfg, frames[:2], (H, W), "'videos'"),
        (state, cfg, [4, 5, 7], (H, W), "'frames'"),
        (state, cfg, frames, (H, W + 1), "'H x W'"),
        ({**state, "focal_steps": 2}, cfg, frames, (H, W), "'optimizer'"),
        ({**state, "window": state["window"][:, 0]}, cfg, frames, (H, W), "'window'"),
    ]
    for st, c, f, hw, match in cases:
        with pytest.raises(ValueError, match=match):
            checkpoint.check(st, c, f, hw)


def test_sharded_optimiser_refuses_checkpoints():
    from flowmap_b200.overfit import ShardedFusedOverfitter
    o = object.__new__(ShardedFusedOverfitter)
    with pytest.raises(ValueError, match="pair-sharded"):
        o.state_dict()
    with pytest.raises(ValueError, match="pair-sharded"):
        o.load_state_dict({})
