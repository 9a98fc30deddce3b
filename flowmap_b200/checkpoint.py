"""Checkpoints of a FusedOverfitter run, and their interchange with the reference-shaped loop
(Model -> LossFlow / LossTracking -> backward() -> torch.optim.Adam).

A state is a plain dict that torch.save writes:

- "format": FORMAT; "cfg": the OverfitCfg as a dict;
- "global_step", "optimizer_steps", "focal_steps", "base_seed": Python ints (the step clock: Adam's update
  counts, the focal length's counting from the softmin -> regressed hand-over, and the seed of every step's
  softmin point sample);
- "window": the softmin hand-over window, (n,) for one video, (n, B) for several, or None;
- "videos": one dict per video: "frames" F_b, "model" (Model.state_dict(), the reference's names) and
  "optimizer" (torch.optim.Adam.state_dict() over Model.parameters(): depth, weight logits[, focal length]).

Pure Python on whatever device the tensors are on: nothing here launches a kernel of this project."""
from __future__ import annotations

import copy
from dataclasses import asdict

import torch

FORMAT = 1
BETAS, EPS = (0.9, 0.999), 1e-8  # FusedOverfitter's Adam


def _fail(field: str, msg: str):
    raise ValueError(f"flowmap_b200: checkpoint field {field!r}: {msg}")


def adam_steps(cfg, optimizer_steps: int, focal_steps: int) -> list:
    """The update count torch.optim.Adam holds for each parameter of one video's Model, in Model.parameters()
    order (depth, weight logits[, focal length]).  0 marks a parameter that has had no gradient yet, which has
    no state entry: the logits without correspondence weights, the focal length before the hand-over."""
    steps = [optimizer_steps, optimizer_steps if cfg.use_correspondence_weights else 0]
    if cfg.intrinsics == "regressed" or cfg.intrinsics == "softmin" and cfg.regression_after is not None:
        steps.append(focal_steps)
    return steps


def adam_state(slots, lr: float) -> dict:
    """torch.optim.Adam(model.parameters(), lr).state_dict() for `slots`, one (exp_avg, exp_avg_sq, update
    count) per parameter in Model.parameters() order.  The moments are cloned on their device and stream;
    `step` is a CPU float32 scalar, as torch keeps it."""
    group = torch.optim.Adam([torch.empty(0)], lr=lr, betas=BETAS, eps=EPS).state_dict()["param_groups"][0]
    group["params"] = list(range(len(slots)))
    state = {i: {"step": torch.tensor(float(n), dtype=torch.float32), "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
             for i, (m, v, n) in enumerate(slots) if n > 0}
    return {"state": state, "param_groups": [group]}


def load_moments(optimizer_state: dict, slots) -> None:
    """Copy the moments of an Adam state dict into `slots` (exp_avg, exp_avg_sq, ...) in place; a parameter
    without an entry gets zero moments."""
    for i, (m, v, *_) in enumerate(slots):
        e = optimizer_state["state"].get(i)
        if e is None:
            m.zero_()
            v.zero_()
        else:
            m.copy_(e["exp_avg"])
            v.copy_(e["exp_avg_sq"])


def new_state(cfg, global_step: int, optimizer_steps: int, focal_steps: int, base_seed: int, window, videos) -> dict:
    return {"format": FORMAT, "cfg": asdict(cfg), "global_step": int(global_step),
            "optimizer_steps": int(optimizer_steps), "focal_steps": int(focal_steps), "base_seed": int(base_seed),
            "window": window, "videos": videos}


def video_entry(frames: int, model_state: dict, slots, lr: float) -> dict:
    return {"frames": int(frames), "model": model_state, "optimizer": adam_state(slots, lr)}


def _hw(video: dict):
    return tuple(video["model"]["backbone.depth"].shape[-2:])


def check(state: dict, cfg, frames, hw) -> None:
    """ValueError naming the first field in which `state` does not fit an optimiser of `cfg` over videos of
    `frames` frames of H x W = `hw` pixels."""
    if state.get("format") != FORMAT:
        _fail("format", f"version {state.get('format')!r}, this code reads version {FORMAT}")
    videos = state["videos"]
    if len(videos) != len(frames):
        _fail("videos", f"{len(videos)} videos, the optimiser holds {len(frames)}")
    for b, (v, f) in enumerate(zip(videos, frames)):
        if v["frames"] != f:
            _fail("frames", f"video {b} has {v['frames']} frames, the optimiser's has {f}")
        if _hw(v) != tuple(hw):
            _fail("H x W", f"video {b} is {_hw(v)}, the optimiser's videos are {tuple(hw)}")
    saved, want = state["cfg"], asdict(cfg)
    if saved.get("intrinsics") != cfg.intrinsics:
        _fail("intrinsics", f"{saved.get('intrinsics')!r}, the optimiser runs {cfg.intrinsics!r}")
    for key in sorted(set(saved) | set(want)):
        if saved.get(key) != want.get(key):
            _fail(f"cfg.{key}", f"{saved.get(key)!r}, the optimiser's is {want.get(key)!r}")
    w = state["window"]
    if w is not None:
        if cfg.intrinsics != "softmin" or cfg.regression_after is None:
            _fail("window", "a hand-over window needs softmin intrinsics with a regression stage")
        if w.dim() != (1 if len(frames) == 1 else 2) or w.dim() == 2 and w.shape[1] != len(frames):
            _fail("window", f"shape {tuple(w.shape)}: (n,) for one video, (n, B) for several")
    steps = adam_steps(cfg, state["optimizer_steps"], state["focal_steps"])
    expect = {i: n for i, n in enumerate(steps) if n > 0}
    for b, v in enumerate(videos):
        got = {i: int(e["step"]) for i, e in v["optimizer"]["state"].items()}
        if got != expect:
            _fail("optimizer", f"video {b}'s Adam steps {got} do not match the counters' {expect}")


def _columns(window):
    """The window as (n, B) columns, or None."""
    if window is None:
        return None
    return window[:, None] if window.dim() == 1 else window


def to_torch(state: dict, b: int = 0):
    """(model_state_dict, adam_state_dict, global_step, window) of video b, for the reference-shaped loop:
    model.load_state_dict(model_state_dict); opt = torch.optim.Adam(model.parameters(), lr);
    opt.load_state_dict(adam_state_dict); model.intrinsics.window = window (softmin with a regression stage).
    The window is a list of scalar tensors, empty when none is open.  Fresh tensors: continuing the run
    leaves `state` as it was."""
    v = state["videos"][b]
    cols = _columns(state["window"])
    window = [] if cols is None else list(cols[:, b].clone().unbind(0))
    return copy.deepcopy(v["model"]), copy.deepcopy(v["optimizer"]), state["global_step"], window


def from_torch(cfg, model, optimizer, global_step: int, window=None) -> dict:
    """The one-video state of a reference-shaped run: an explicit-depth `model` of `cfg`, `optimizer` =
    torch.optim.Adam(model.parameters(), cfg.lr) and the run's `global_step`; `window` is the model's
    intrinsics.window (a list of scalar tensors, or an (n,) tensor) for softmin with a regression stage.
    optimizer_steps and focal_steps come from the Adam `step` entries.  The base_seed is fresh: the
    reference draws its softmin samples from torch's RNG (randperm), which the step clock cannot continue."""
    from .model import BackboneExplicitDepth
    if not isinstance(model.backbone, BackboneExplicitDepth):
        _fail("model", "FusedOverfitter owns explicit depth only; a network backbone's state stays with its optimiser")
    if model.cfg.intrinsics.name != cfg.intrinsics:
        _fail("intrinsics", f"the model's are {model.cfg.intrinsics.name!r}, cfg.intrinsics is {cfg.intrinsics!r}")
    params = list(model.parameters())
    groups = optimizer.param_groups
    if len(groups) != 1 or len(groups[0]["params"]) != len(params) or \
            any(p is not q for p, q in zip(groups[0]["params"], params)):
        _fail("optimizer", "one param group over model.parameters(), in that order")
    for key, want in (("lr", cfg.lr), ("betas", BETAS), ("eps", EPS), ("weight_decay", 0), ("amsgrad", False),
                      ("maximize", False)):
        got = groups[0].get(key, want)
        if (tuple(got) if key == "betas" else got) != want:
            _fail(f"optimizer.{key}", f"{got!r}; FusedOverfitter runs {want!r}")
    sd = copy.deepcopy(optimizer.state_dict())
    steps = {i: int(e["step"]) for i, e in sd["state"].items()}
    if 0 in steps and 1 in steps and steps[0] != steps[1]:
        _fail("optimizer", f"depth has had {steps[0]} updates, the weight logits {steps[1]}: a fused step "
                           "updates both")
    if window is not None and len(window) == 0:
        window = None
    elif window is not None:
        window = window.detach().clone() if isinstance(window, torch.Tensor) else torch.stack(list(window)).detach()
    frames = model.backbone.depth.shape[0]
    video = {"frames": int(frames), "model": {k: t.detach().clone() for k, t in model.state_dict().items()},
             "optimizer": sd}
    state = new_state(cfg, global_step, steps.get(0, steps.get(1, 0)), steps.get(2, 0),
                      int(torch.randint(0, 2 ** 62, (1,)).item()), window, [video])
    check(state, cfg, [frames], _hw(video))
    return state


def split(state: dict) -> list:
    """One one-video state per video of `state`, with its counters, seed and its column of the window."""
    cols = _columns(state["window"])
    return [{**state, "cfg": dict(state["cfg"]), "window": None if cols is None else cols[:, b].clone(),
             "videos": [v]} for b, v in enumerate(state["videos"])]


def merge(states) -> dict:
    """One state for an optimiser over all videos of `states` in order (a list of Batches, or a tensor batch
    when they have one length).  A packed optimiser has one step clock and one cfg: the states must agree on
    the format, the counters and the cfg, and their videos on H x W.  The base_seed is the first state's: a
    packed batch shares each step's softmin point sample (DESIGN §1.1)."""
    first = states[0]
    for s in states[1:]:
        for key in ("format", "global_step", "optimizer_steps", "focal_steps", "cfg"):
            if s[key] != first[key]:
                _fail(key, f"{s[key]!r} and {first[key]!r}: the videos of one optimiser share it")
    videos = [v for s in states for v in s["videos"]]
    for v in videos:
        if _hw(v) != _hw(videos[0]):
            _fail("H x W", f"{_hw(v)} and {_hw(videos[0])}: the videos of one optimiser share it")
    cols = [_columns(s["window"]) for s in states]
    if any(c is None for c in cols):
        if any(c is not None for c in cols):
            _fail("window", "open in some states and not in others")
        window = None
    else:
        if len({c.shape[0] for c in cols}) != 1:
            _fail("window", "of different lengths")
        window = torch.cat(cols, 1)
        window = window[:, 0] if len(videos) == 1 else window
    return {**first, "cfg": dict(first["cfg"]), "window": window, "videos": videos}
