"""world_size-2 (and 3) gloo tests of the pair-sharding host logic (flowmap_b200.parallel):
shard plan, the single per-step all-reduce and the boundary-frame halo.  The per-shard
compute is the oracle (CPU); the CUDA kernels are covered by the -m gpu tests."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT


def test_shard_pairs():
    from flowmap_b200.parallel import shard_pairs
    assert shard_pairs(149, 1) == [(0, 149)]
    s = shard_pairs(149, 8)
    assert s[0][0] == 0 and s[-1][1] == 149
    assert all(a[1] == b[0] for a, b in zip(s, s[1:]))
    assert max(b - a for a, b in s) - min(b - a for a, b in s) <= 1
    with pytest.raises(ValueError):
        shard_pairs(3, 4)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, f, h, w, out_dir):
    sys.path.insert(0, str(ROOT))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from flowmap_b200 import parallel
        from oracle import flowmap_oracle as O
        torch.set_num_threads(2)
        dt = torch.float64
        flows = O.synthetic_flows(f, h, w, seed=3, dtype=dt)
        gen = torch.Generator().manual_seed(4)
        depth = 1.0 + torch.rand(f, h, w, generator=gen, dtype=dt)
        wparam = 0.01 * torch.randn(f - 1, h, w, generator=gen, dtype=dt)
        plan = parallel.make_plan(f - 1)
        d_l, w_l, fl_l = parallel.shard_inputs(plan, depth, wparam, flows)
        st = O.OverfitOracle(O.OverfitConfig(intrinsics="regressed"), plan.num_local_frames, h, w, dtype=dt)
        with torch.no_grad():
            st.depth.copy_(d_l)
            st.weights.copy_(w_l)
        out = st.forward(fl_l, 0)
        # local loss normalised by the GLOBAL mask sum (what the pair-sharded step does with global_mask_sum)
        local_den = fl_l.forward_mask.sum() + fl_l.backward_mask.sum()
        den = parallel.global_mask_sum(local_den.reshape(()).clone())
        loss = 1000.0 * O.flow_loss(out.surfaces, out.extrinsics, out.intrinsics, fl_l) * local_den / den
        loss.backward()
        red = parallel.StepReducer(plan, (h, w), "cpu", 2)
        g_depth = st.depth.grad.float().clone()
        scal = red.reduce(torch.stack((loss.detach().float(), st.focal.grad.float())), g_depth)
        # the same exchange in its two halves (start ... independent work ... finish)
        red2 = parallel.StepReducer(plan, (h, w), "cpu", 2)
        g_depth2 = st.depth.grad.float().clone()
        red2.scal.copy_(torch.stack((loss.detach().float(), st.focal.grad.float())))
        reqs = red2.start(g_depth2)
        interior_untouched = g_depth2[1:-1].clone()
        scal2 = red2.finish(reqs, g_depth2)
        assert torch.equal(scal2, scal) and torch.equal(g_depth2, g_depth)
        assert torch.equal(g_depth2[1:-1], interior_untouched)
        torch.save({"range": plan.pair_range, "g_depth": g_depth, "g_w": st.weights.grad.float(),
                    "scalars": scal, "bytes": red.bytes_per_step()}, f"{out_dir}/r{rank}.pt")
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_step_equals_unsharded(tmp_path, world):
    from oracle import flowmap_oracle as O
    f, h, w = 7, 12, 16
    mp.spawn(_worker, args=(world, _free_port(), f, h, w, str(tmp_path)), nprocs=world, join=True)
    dt = torch.float64
    flows = O.synthetic_flows(f, h, w, seed=3, dtype=dt)
    gen = torch.Generator().manual_seed(4)
    depth = 1.0 + torch.rand(f, h, w, generator=gen, dtype=dt)
    wparam = 0.01 * torch.randn(f - 1, h, w, generator=gen, dtype=dt)
    st = O.OverfitOracle(O.OverfitConfig(intrinsics="regressed"), f, h, w, dtype=dt)
    with torch.no_grad():
        st.depth.copy_(depth)
        st.weights.copy_(wparam)
    ref = st.training_step(flows)
    parts = [torch.load(f"{tmp_path}/r{r}.pt") for r in range(world)]
    for p in parts:
        a, b = p["range"]
        assert abs(float(p["scalars"][0]) - ref["loss"]) <= 1e-5 * abs(ref["loss"])
        assert abs(float(p["scalars"][1]) - float(ref["grads"]["focal"])) <= 1e-4 * abs(float(ref["grads"]["focal"]))
        gd = ref["grads"]["depth"][a:b + 1].float()
        assert float((p["g_depth"] - gd).norm() / gd.norm()) <= 1e-5
        gw = ref["grads"]["weights"][a:b].float()
        assert float((p["g_w"] - gw).norm() / gw.norm()) <= 1e-5
        assert p["bytes"] == 4 * 2 + 4 * h * w * (int(a > 0) + int(b < f - 1))  # scalars + a frame per neighbour
    # replicas of a boundary frame hold bit-identical gradients after the reduce
    for left, right in zip(parts, parts[1:]):
        assert torch.equal(left["g_depth"][-1], right["g_depth"][0])


# ---------------------------------------------------------------- tracking loss, sharded by source frame
def _track_worker(rank, world, port, f, h, w, out_dir):
    """Each rank: poses of its own pairs (oracle), gather_pairs, chain, tracking terms of its
    SOURCE frames against all targets, all-reduce of (sum, count) and of the pose gradient."""
    sys.path.insert(0, str(ROOT))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from flowmap_b200 import parallel
        from oracle import flowmap_oracle as O
        torch.set_num_threads(2)
        dt = torch.float64
        flows = O.synthetic_flows(f, h, w, seed=3, dtype=dt)
        gen = torch.Generator().manual_seed(4)
        depth = 1.0 + torch.rand(f, h, w, generator=gen, dtype=dt)
        wparam = 0.01 * torch.randn(f - 1, h, w, generator=gen, dtype=dt)
        tracks = O.synthetic_tracks(f, n_points=40, interval=3, radius=4, seed=5, dtype=dt)
        plan = parallel.make_plan(f - 1)
        a, b = plan.pair_range
        d_l, w_l, fl_l = parallel.shard_inputs(plan, depth, wparam, flows)
        d_l.requires_grad_(True)
        w_l.requires_grad_(True)
        focal = torch.tensor(0.85, dtype=dt, requires_grad=True)
        k_all = O.intrinsics_from_focal(focal, h, w).expand(1, f, 3, 3)
        depths, weights = O.explicit_backbone(d_l, w_l, 100.0)
        surf_l = O.unproject(O.pixel_grid(h, w, dt), depths, k_all[:, a:b + 1, None, None])
        rel_l = O.relative_poses(surf_l, fl_l.backward, weights, torch.arange(h * w))
        # gather the relative poses (values only), make the gathered tensor a leaf
        rel_all = parallel.gather_pairs(plan, rel_l.detach()).requires_grad_(True)
        ext_all = O.pose_chain(rel_all)
        lo, hi = parallel.source_frame_range(plan)
        owned = torch.zeros(f, dtype=torch.bool)
        owned[lo:hi] = True
        surf_all = torch.zeros(1, f, h, w, 3, dtype=dt)
        surf_all = torch.cat((surf_all[:, :a], surf_l, surf_all[:, b + 1:]), dim=1)
        num, den = 0, 0
        for seg in tracks:
            s, n_f = seg.start_frame, seg.xy.shape[1]
            target, valid = O.track_positions(surf_all[:, s:s + n_f], ext_all[:, s:s + n_f], k_all[:, s:s + n_f], seg)
            valid = valid & owned[s:s + n_f][None, :, None, None]
            target = torch.where(valid[..., None], target, torch.zeros_like(target))
            num = num + (O.robust_map(target, seg.xy[:, None], h, w) * valid).sum()
            den = den + valid.sum()
        sums = torch.stack((num.detach(), den.to(dt)))
        dist.all_reduce(sums)
        loss_local = 100.0 * num / sums[1]          # the count is global and has no gradient
        loss_local.backward(retain_graph=True)   # surfaces are shared with the pose graph below
        g_rel = rel_all.grad.clone()
        dist.all_reduce(g_rel)                      # pose gradient: sum of every rank's sources
        rel_l.backward(g_rel[:, a:b])
        g_focal = focal.grad.clone()
        dist.all_reduce(g_focal)
        torch.save({"range": (a, b), "loss": 100.0 * sums[0] / sums[1], "g_depth": d_l.grad, "g_w": w_l.grad,
                    "g_focal": g_focal}, f"{out_dir}/t{rank}.pt")
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_source_sharded_tracking_equals_unsharded(tmp_path, world):
    from oracle import flowmap_oracle as O
    f, h, w = 10, 12, 16
    mp.spawn(_track_worker, args=(world, _free_port(), f, h, w, str(tmp_path)), nprocs=world, join=True)
    dt = torch.float64
    flows = O.synthetic_flows(f, h, w, seed=3, dtype=dt)
    gen = torch.Generator().manual_seed(4)
    depth = 1.0 + torch.rand(f, h, w, generator=gen, dtype=dt)
    wparam = 0.01 * torch.randn(f - 1, h, w, generator=gen, dtype=dt)
    tracks = O.synthetic_tracks(f, n_points=40, interval=3, radius=4, seed=5, dtype=dt)
    st = O.OverfitOracle(O.OverfitConfig(intrinsics="regressed", use_tracking=True, tracking_enable_after=0,
                                         flow_enable_after=10**9), f, h, w, dtype=dt)
    with torch.no_grad():
        st.depth.copy_(depth)
        st.weights.copy_(wparam)
    ref = st.training_step(flows, tracks)
    parts = [torch.load(f"{tmp_path}/t{r}.pt") for r in range(world)]
    rel = lambda x, y: float((x - y).norm() / y.norm())  # noqa: E731
    g_depth = torch.zeros_like(depth)
    for p in parts:
        a, b = p["range"]
        assert abs(float(p["loss"]) - ref["parts"]["tracking"]) <= 1e-10 * abs(ref["parts"]["tracking"])
        assert abs(float(p["g_focal"]) - float(ref["grads"]["focal"])) <= 1e-8 * abs(float(ref["grads"]["focal"]))
        assert rel(p["g_w"], ref["grads"]["weights"][a:b]) <= 1e-8
        g_depth[a:b + 1] += p["g_depth"]            # what StepReducer does for the boundary frames
    assert rel(g_depth, ref["grads"]["depth"]) <= 1e-8
