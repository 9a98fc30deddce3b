"""Multi-GPU execution of the hot path: frame pairs sharded across ranks.

The flow loss is pair-local (SURVEY A.6): pair i needs depth frames i and i+1, its own
weights/flows/masks and the shared focal length.  Rank g therefore owns a contiguous pair
range [a_g, b_g) and the frames [a_g, b_g]; flows, masks and weights are sharded and
never move.  Per optimisation step there is one exchange (NCCL over NVLink/NVSwitch on the
GPUs, gloo in the CPU tests): an all-reduce of [loss, d(focal)] and, grouped with it, a
send/recv of ONE boundary depth-gradient frame with each neighbour (its size does not grow
with the number of ranks).

A boundary frame (last frame of rank g == first frame of rank g+1) is "later" for a pair
on rank g and "earlier" for a pair on rank g+1; the two ranks swap their partial gradients
of that frame, each adds the other's to its own (a + b == b + a bit for bit), and both then
apply the identical Adam update to their replica, so the replicas stay bit-identical without a
second message.  The reference has no counterpart (its DDP replicas hold the identical
problem, flowmap/overfit.py:99-103).

The tracking loss couples frames up to 40 apart, so it is sharded by SOURCE frame instead
(`source_frame_range`): the relative poses are gathered (`gather_pairs`, 149 x 12 floats), every
rank chains them and evaluates its source frames against all targets; the loss sum, the valid
count and the per-frame pose / intrinsics sums (F x 10 doubles) are all-reduced, after which the
pose gradient is global on every rank and flows back through the chain into the rank's own pairs
(overfit.ShardedFusedOverfitter).  The softmin sweep lives on the rank that owns pair 0: one
broadcast of its focal estimate before the step.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist
from torch import Tensor


def shard_pairs(num_pairs: int, world: int) -> List[Tuple[int, int]]:
    """Contiguous, balanced pair ranges [a, b) per rank (first ranks take the remainder)."""
    if world < 1 or num_pairs < world:
        raise ValueError(f"cannot shard {num_pairs} pairs over {world} ranks")
    base, rem = divmod(num_pairs, world)
    out, a = [], 0
    for r in range(world):
        b = a + base + (1 if r < rem else 0)
        out.append((a, b))
        a = b
    return out


@dataclass
class ShardPlan:
    rank: int
    world: int
    pair_range: Tuple[int, int]  # global [a, b)
    num_pairs_total: int

    @property
    def frame_range(self) -> Tuple[int, int]:  # global [a, b] inclusive -> python slice [a, b+1)
        return self.pair_range[0], self.pair_range[1] + 1

    @property
    def num_local_frames(self) -> int:
        return self.pair_range[1] - self.pair_range[0] + 1

    @property
    def has_left(self) -> bool:
        return self.rank > 0

    @property
    def has_right(self) -> bool:
        return self.rank < self.world - 1


def make_plan(num_pairs_total: int, rank: Optional[int] = None,
              world: Optional[int] = None) -> ShardPlan:
    rank = dist.get_rank() if rank is None else rank
    world = dist.get_world_size() if world is None else world
    return ShardPlan(rank, world, shard_pairs(num_pairs_total, world)[rank], num_pairs_total)


def shard_inputs(plan: ShardPlan, depth: Tensor, wparam: Tensor, flows):
    """Slice a full (unsharded) problem down to this rank's shard.  depth (F,H,W), wparam
    (F-1,H,W), flows with leading (1, F-1, ...)."""
    a, b = plan.pair_range
    sl = slice(a, b)
    return (depth[a:b + 1].clone(), wparam[sl].clone(),
            type(flows)(flows.forward[:, sl].clone(), flows.backward[:, sl].clone(),
                        flows.forward_mask[:, sl].clone(), flows.backward_mask[:, sl].clone()))


def global_mask_sum(local_sum: Tensor, group=None) -> Tensor:
    """The loss normaliser is global (loss_flow.py:70 sums the masks of ALL pairs): all-reduce
    the local mask sums once; the result is loop-invariant."""
    total = local_sum.clone()
    if dist.is_available() and dist.is_initialized():  # a single process without a group: nothing to add
        dist.all_reduce(total, op=dist.ReduceOp.SUM, group=group)
    return total


def source_frame_range(plan: ShardPlan) -> Tuple[int, int]:
    """Tracking loss (not pair-local, SURVEY 8(e)): rank g evaluates the SOURCE frames [lo, hi) of
    every track segment against all target frames.  A boundary frame is held by two ranks; the
    right one owns it as a source, the last rank also owns the last frame."""
    a, b = plan.pair_range
    return a, (b + 1 if plan.rank == plan.world - 1 else b)


def gather_pairs(plan: ShardPlan, local: Tensor, out: Optional[Tensor] = None, group=None) -> Tensor:
    """Per-pair quantities (1, local pairs, ...) of every rank -> (1, all pairs, ...) on every rank.
    The slices are disjoint, so a sum all-reduce of a zero-filled buffer is a gather with one
    collective and no size bookkeeping (149 x 12 floats for the relative poses)."""
    a, b = plan.pair_range
    if out is None:
        out = torch.zeros((local.shape[0], plan.num_pairs_total, *local.shape[2:]), dtype=local.dtype,
                          device=local.device)
    else:
        out.zero_()
    out[:, a:b].copy_(local)
    if plan.world > 1:
        dist.all_reduce(out, op=dist.ReduceOp.SUM, group=group)
    return out


class StepReducer:
    """The per-step exchange: one all-reduce of the scalars (loss, d focal) and one grouped
    send/recv of a boundary depth-gradient frame with each neighbour (0.9 MB at 360x640 per
    boundary, independent of the world size)."""

    def __init__(self, plan: ShardPlan, frame_shape, device, num_scalars: int = 2, group=None):
        self.plan, self.group = plan, group
        self.h, self.w = frame_shape
        self.nscal = num_scalars
        self.scal = torch.zeros(num_scalars, dtype=torch.float32, device=device)
        mk = lambda: torch.zeros(self.h, self.w, dtype=torch.float32, device=device)  # noqa: E731
        self.from_left = mk() if plan.has_left else None
        self.from_right = mk() if plan.has_right else None
        self.to_left = mk() if plan.has_left else None
        self.to_right = mk() if plan.has_right else None

    def _peer(self, offset: int) -> int:
        r = self.plan.rank + offset
        return r if self.group is None else dist.get_global_rank(self.group, r)

    @torch.no_grad()
    def reduce(self, scalars: Tensor, depth_grad: Tensor) -> Tensor:
        """scalars: (num_scalars,) local partials (loss, d focal, ...); depth_grad: this
        rank's (frames, H, W) gradient, modified in place at the shared boundary frames (both
        owners end up with the same sum: a + b is commutative, the replicas stay bit-identical).
        Returns the globally summed scalars."""
        p = self.plan
        self.scal.copy_(scalars)
        if p.world == 1:
            return self.scal.clone()
        ops = []
        if p.has_left:
            self.to_left.copy_(depth_grad[0])
            ops += [dist.P2POp(dist.isend, self.to_left, self._peer(-1), self.group),
                    dist.P2POp(dist.irecv, self.from_left, self._peer(-1), self.group)]
        if p.has_right:
            self.to_right.copy_(depth_grad[-1])
            ops += [dist.P2POp(dist.isend, self.to_right, self._peer(+1), self.group),
                    dist.P2POp(dist.irecv, self.from_right, self._peer(+1), self.group)]
        reqs = dist.batch_isend_irecv(ops) if ops else []
        dist.all_reduce(self.scal, op=dist.ReduceOp.SUM, group=self.group)
        for r in reqs:
            r.wait()
        if p.has_left:
            depth_grad[0].add_(self.from_left)
        if p.has_right:
            depth_grad[-1].add_(self.from_right)
        return self.scal.clone()

    # ---- the same exchange in two halves, so that work that does not depend on it (Adam on the
    # interior frames) runs between them while the boundary frames travel over NVLink
    @torch.no_grad()
    def start(self, depth_grad: Tensor):
        """Begin the exchange of `self.scal` (filled by the caller) and the boundary frames of
        depth_grad; returns the pending requests for finish()."""
        p = self.plan
        if p.world == 1:
            return []
        ops = []
        # the boundary frames are sent from where they lie (contiguous rows of depth_grad; nothing
        # writes them before finish() has waited for the sends)
        if p.has_left:
            ops += [dist.P2POp(dist.isend, depth_grad[0], self._peer(-1), self.group),
                    dist.P2POp(dist.irecv, self.from_left, self._peer(-1), self.group)]
        if p.has_right:
            ops += [dist.P2POp(dist.isend, depth_grad[-1], self._peer(+1), self.group),
                    dist.P2POp(dist.irecv, self.from_right, self._peer(+1), self.group)]
        reqs = dist.batch_isend_irecv(ops) if ops else []
        reqs.append(dist.all_reduce(self.scal, op=dist.ReduceOp.SUM, group=self.group, async_op=True))
        return reqs

    @torch.no_grad()
    def finish(self, reqs, depth_grad: Tensor) -> Tensor:
        """Wait for start()'s requests and add the neighbours' boundary partials (both owners end up
        with the same sum).  Returns self.scal (globally summed, a persistent buffer)."""
        for r in reqs:
            r.wait()
        if self.plan.world > 1:
            if self.plan.has_left:
                depth_grad[0].add_(self.from_left)
            if self.plan.has_right:
                depth_grad[-1].add_(self.from_right)
        return self.scal

    def bytes_per_step(self) -> int:
        """Bytes this rank sends per step (scalars + one frame per neighbour)."""
        return 4 * self.nscal + 4 * self.h * self.w * (int(self.plan.has_left) + int(self.plan.has_right))
