"""`-m gpu`: round-2 machinery around the hot path -- the device step clock against by-value Adam,
CUDA-graph replay of the update step against eager execution, the early moment pass of a sweep step and
the tracking sweep sharded by source frame."""
import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu


def test_step_clock_adam_equals_by_value_adam():
    from flowmap_b200 import ops
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    p0 = torch.randn(4099, device=dev, generator=g)
    pa, pb = p0.clone(), p0.clone()
    ma, va, mb, vb = (torch.zeros_like(p0) for _ in range(4))
    clock = ops.StepClock(dev, lr=3e-5)
    clock.set(6, 0)  # six updates already done: the next tick is step 7
    for step in range(7, 12):
        grad = torch.randn(4099, device=dev, generator=g)
        ops.adam_step(pa, grad, ma, va, step, 3e-5)
        clock.tick(tick_focal=False)
        ops.adam_step_clock(pb, grad, mb, vb, clock)
    assert float((pa - pb).abs().max()) <= 1e-9 * float(pa.abs().max()) + 1e-12
    assert torch.equal(ma, mb) and torch.equal(va, vb)


@pytest.mark.parametrize("full", [False, True], ids=["flow_only", "softmin_tracking"])
def test_cuda_graph_replay_equals_eager_steps(full):
    """The update step replayed as one CUDA graph (from its third run on) follows the eager
    trajectory to the noise of the float atomics (the order of the REDs into the depth gradient is
    not fixed from run to run)."""
    import bench
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows, Tracks
    dev = torch.device("cuda:0")
    f, h, w, steps = 12, 72, 96, 8

    def run(graph):
        inp = bench.synthetic_inputs(f, h, w, seed=0)
        batch = Batch(torch.zeros(1, f, 3, h, w, device=dev), torch.arange(f, device=dev)[None], ["s"], ["d"])
        flows = Flows(*(inp[k].to(dev) for k in ("fwd", "bwd", "fmask", "bmask")))
        tracks = [Tracks(xy, vis, s) for xy, vis, s in
                  bench.synthetic_track_arrays(f, n_points=64, interval=3, radius=2)] if full else None
        cfg = OverfitCfg(intrinsics="softmin", use_tracking=True, tracking_enable_after=0, softmin_points=500) \
            if full else OverfitCfg()
        o = FusedOverfitter(cfg, batch, flows, tracks, device=dev)
        o._clock.base_seed = 1234  # same softmin point samples in both runs
        with torch.no_grad():
            o.model.backbone.depth.copy_(1.0 + inp["depth"])
            o.model.backbone.weights.copy_(inp["wparam"])
        o.use_cuda_graph = graph
        losses = [float(o.training_step()[0]) for _ in range(steps)]
        return losses, o.model.backbone.depth.detach().clone(), o.model.backbone.weights.detach().clone(), len(o._graphs)

    la, da, wa, _ = run(False)
    lb, db, wb, ngraphs = run(True)
    assert ngraphs == 1
    tol = 1e-5 if full else 1e-7
    assert max(abs(x - y) for x, y in zip(la, lb)) <= tol * abs(la[0])
    assert rel_l2(db, da) <= tol and float((wb - wa).abs().max()) <= (1e-5 if full else 1e-6)


def test_early_moment_pass_of_a_sweep_step_matches_the_sequential_order():
    """An update step of the softmin stage accumulates the Procrustes moments beside the sweep, on the
    candidate-0 intrinsics, and rescales them to the focal length the sweep produced
    (fm_procrustes_moments + fm_overfit_step_args.moments_k4).  An evaluation step of the same state
    runs the moment pass after the sweep with the final intrinsics: same loss, same poses."""
    import bench
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows, Tracks
    dev = torch.device("cuda:0")
    f, h, w = 10, 72, 96
    inp = bench.synthetic_inputs(f, h, w, seed=3)
    batch = Batch(torch.zeros(1, f, 3, h, w, device=dev), torch.arange(f, device=dev)[None], ["s"], ["d"])
    flows = Flows(*(inp[k].to(dev) for k in ("fwd", "bwd", "fmask", "bmask")))
    tracks = [Tracks(xy, vis, s) for xy, vis, s in bench.synthetic_track_arrays(f, n_points=64, interval=3, radius=2)]
    o = FusedOverfitter(OverfitCfg(intrinsics="softmin", use_tracking=True, tracking_enable_after=0), batch, flows,
                        tracks, device=dev)
    with torch.no_grad():
        o.model.backbone.depth.copy_(1.0 + inp["depth"])
        o.model.backbone.weights.copy_(inp["wparam"])
    o.injected_indices = torch.randperm(h * w, generator=torch.Generator().manual_seed(5))[:512].to(dev)
    o.use_cuda_graph = False
    loss_eval, rt_eval = o.training_step(update=False)
    loss_eval, rt_eval = float(loss_eval), rt_eval.clone()
    loss_upd, rt_upd = o.training_step(update=True)
    assert abs(float(loss_upd) - loss_eval) <= 2e-6 * abs(loss_eval)
    assert float((rt_upd - rt_eval).abs().max()) <= 2e-6


def test_tracking_sweep_sharded_by_source_frame_adds_up():
    """fm_track_loss_fwd_sharded restricted to source frames [lo, hi): the head of the tracking
    workspace (loss sum, valid count, per-frame accumulators; what the ranks all-reduce) of two
    complementary shards adds up to the unsharded sweep's, with a shard whose depth pointer starts
    at its first source frame."""
    from flowmap_b200 import ops
    from flowmap_b200._lib import check, lib
    from flowmap_b200.types import Tracks
    dev = torch.device("cuda:0")
    f, h, w = 9, 24, 32
    g = torch.Generator().manual_seed(21)
    depth = (1.0 + 0.5 * torch.rand(1, f, h, w, generator=g)).to(dev)
    ext = torch.eye(4).repeat(1, f, 1, 1)
    ext[0, :, :3, 3] = 0.05 * torch.randn(f, 3, generator=g)
    ext = ext.to(dev).contiguous()
    s = (h * w) ** 0.5
    k4 = torch.tensor([0.9 * s / w, 0.9 * s / h, 0.5, 0.5]).expand(1, f, 4).contiguous().to(dev)
    tracks = [Tracks(torch.rand(1, f, 300, 2, generator=g).to(dev), (torch.rand(1, f, 300, generator=g) < 0.7).to(dev), 0),
              Tracks(torch.rand(1, 4, 70, 2, generator=g).to(dev), (torch.rand(1, 4, 70, generator=g) < 0.7).to(dev), 3)]
    pk = ops.PackedTracks(tracks, dev)
    L = lib()
    P = lambda t: t.data_ptr()  # noqa: E731
    st = torch.cuda.current_stream().cuda_stream
    head = L.fm_track_reduce_bytes(f) // 8

    def sweep(lo, hi, frame0):
        ws = torch.zeros(L.fm_track_workspace_bytes(f, pk.total), dtype=torch.uint8, device=dev)
        check(L.fm_track_loss_fwd_sharded(P(depth[:, frame0:]), P(k4), P(ext), P(pk.seg), pk.num_segments, pk.max_rows,
                                          pk.max_points, P(pk.xy), P(pk.vis), pk.total, 0, 0.01, 100.0, None, P(ws),
                                          f, h, w, frame0, lo, hi, 1, st), "fm_track_loss_fwd_sharded")
        torch.cuda.synchronize()
        return ws[:head * 8].view(torch.float64).clone()

    full = sweep(0, f, 0)
    parts = sweep(0, 4, 0) + sweep(4, f, 4)
    assert float(full[1]) > 100  # enough valid terms for the comparison to mean something
    assert float((parts - full).abs().max()) <= 1e-5 * float(full.abs().max())
