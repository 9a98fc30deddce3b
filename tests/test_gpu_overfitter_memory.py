"""A standalone one-video FusedOverfitter allocates no device memory beyond the tensors it holds.  The step keeps
its Adam moments in its own state, so nothing else may hold moments of the Model's parameters: at 150 x 360 x 640
those would be 551 MB that no kernel reads."""
import dataclasses
import gc

import pytest
import torch
from torch import nn

from oracle import flowmap_oracle as O


def _held_storages(root) -> dict:
    """{data pointer: bytes} of the distinct CUDA storages that `root` holds: its tensors and those of its
    containers, dataclasses (Batch, Flows, Tracks), Modules (the Models) and the step helpers of flowmap_b200.ops
    (PackedTracks, StepClock).  Other objects it refers to (ctypes structures, streams, the library handle)
    own no device memory of the step."""
    from flowmap_b200 import ops
    seen, storages, todo = set(), {}, [root]
    while todo:
        x = todo.pop()
        if id(x) in seen:
            continue
        seen.add(id(x))
        if isinstance(x, torch.Tensor):
            if x.is_cuda:
                s = x.untyped_storage()
                storages[s.data_ptr()] = s.nbytes()
        elif isinstance(x, (list, tuple)):
            todo.extend(x)
        elif isinstance(x, dict):
            todo.extend(x.values())
        elif (x is root or isinstance(x, nn.Module) or type(x).__module__ == ops.__name__ or
              dataclasses.is_dataclass(x) and not isinstance(x, type)):
            todo.extend(vars(x).values())
    return storages


def _inputs(f, h, w):
    from flowmap_b200.types import Batch, Flows, Tracks
    fl = O.synthetic_flows(f, h, w, seed=0)
    tracks = [Tracks(t.xy, t.visibility, t.start_frame) for t in O.synthetic_tracks(f, n_points=256, seed=0)]
    batch = Batch(torch.zeros(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    return batch, Flows(fl.forward, fl.backward, fl.forward_mask, fl.backward_mask), tracks


@pytest.mark.gpu
def test_standalone_optimiser_allocates_only_what_it_holds():
    """Construct a standalone optimiser from host inputs (softmin + tracking, 30 x 180 x 240): the requested bytes
    it adds on the device, that is memory_allocated() less the allocator's rounding, are at most the bytes of the
    storages it holds."""
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    cfg = OverfitCfg(intrinsics="softmin", use_tracking=True)
    dev = torch.device("cuda:0")
    FusedOverfitter(cfg, *_inputs(4, 16, 24), device=dev)  # the library, the context and one-time allocations
    f, h, w = 30, 180, 240
    inputs = _inputs(f, h, w)
    gc.collect()
    torch.cuda.synchronize(dev)
    torch.cuda.empty_cache()
    stats = lambda: torch.cuda.memory_stats(dev)  # noqa: E731
    before = stats()
    o = FusedOverfitter(cfg, *inputs, device=dev)
    torch.cuda.synchronize(dev)
    after = stats()
    held = sum(_held_storages(o).values())
    requested = after["requested_bytes.all.current"] - before["requested_bytes.all.current"]
    allocated = after["allocated_bytes.all.current"] - before["allocated_bytes.all.current"]
    print(f"held {held} B, requested {requested} B, allocated {allocated} B (rounding {allocated - requested} B)")
    # the depth and logit rows and their moments are part of what it holds
    assert held >= 3 * (2 * f - 1) * h * w * 4
    # memory_allocated() grew by `allocated`: the requested bytes plus the allocator's rounding
    assert requested <= held, f"{requested - held} bytes allocated that the optimiser does not hold"
