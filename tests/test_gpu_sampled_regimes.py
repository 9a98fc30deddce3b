"""The kernels that run on an explicit point set ("index mode") against the float64 oracle in the flow
regimes of real videos (oracle.flow_regime): the softmin focal-length sweep (fm_softmin_sweep_fwd /
_bwd, fm_softmin_focal / _bwd), the softmin stage of the fused step, and subsampled Procrustes.

The regimes change what the sweep does.  Under `scene` its gradient path is about half of frame 1's
depth gradient; under `leave` and `zoom` the softmin collapses onto the smallest candidate, and the
index-mode gathers clip at the image border.  Gradients are checked per frame, per pair and on the
one-pixel border band against max(1e-4, 3x the float32 oracle's own error in the same metric).

Every comparison hands the oracle the exact index tensor the kernels used, moved to the CPU."""
import pytest
import torch

from conftest import max_abs, rel_l2
from flow_regime_checks import border_band, check, errors, oracle_steps, start_point
from test_gpu_flow_regimes import KINDS

pytestmark = pytest.mark.gpu

SHAPES = [(1, 3, 96, 192),   # one video, the sweep's usual case
          (2, 3, 72, 136),   # a batched sweep (pretraining)
          (1, 3, 72, 133)]   # odd width
SHAPE_IDS = ["1x96x192", "2x72x136", "1x72x133"]
N_CAND = 60


@pytest.fixture(autouse=True)
def _threads():
    torch.set_num_threads(min(16, torch.get_num_threads()))


def _case(kind, b, f, h, w):
    """Regime inputs at the start point of test_gpu_flow_regimes (float64)."""
    from oracle import flowmap_oracle as O
    depth, fl, focal, _ = O.flow_regime(kind, f, h, w, seed=w, b=b)
    depth, focal = start_point(depth, focal, seed=w + 1)
    wparam = 0.01 * torch.randn(b, f - 1, h, w, generator=torch.Generator().manual_seed(w + 2), dtype=torch.float64)
    return depth, wparam, fl, focal


def _sweep_indices(npts, h, w):
    n = h * w if npts is None else npts
    return torch.randperm(h * w, generator=torch.Generator().manual_seed(n + w))[:n].cuda()


def _candidates(dt):
    return torch.linspace(0.5, 2.0, N_CAND, dtype=dt)


def _softmin(err, cand):
    """softmin((err - min) * 10) and f_hat = sum softmin_n f_n (intrinsics_softmin.py:126-131)."""
    sm = torch.softmax(-(err - err.min(dim=1, keepdim=True).values) * 10, dim=1)
    return sm, (sm * cand).sum(dim=1)


def _gpu_softmin(err, cand):
    """The same through k_softmin_focal."""
    from flowmap_b200._lib import check as lib_check, lib
    b, n = err.shape
    sm, fh = torch.empty_like(err), torch.empty(b, device=err.device)
    lib_check(lib().fm_softmin_focal(err.data_ptr(), cand.data_ptr(), n, b, sm.data_ptr(), fh.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream), "fm_softmin_focal")
    return sm, fh


def _oracle_sweep(depth, wparam, bwd, idx, dt, use_weights=True, g_err=None):
    """Oracle errors (b, n) in dtype `dt` [and, given the cotangent g_err, d / d depth and d / d wparam]."""
    from oracle import flowmap_oracle as O
    d = depth.to(dt, copy=True).requires_grad_(True)
    wp = wparam.to(dt, copy=True).requires_grad_(True)
    weights = torch.sigmoid(100.0 * wp) if use_weights else torch.ones_like(wp)
    err = O.softmin_errors(d, weights, bwd.to(dt), idx, _candidates(dt))
    if g_err is None:
        return err.detach().double()
    err.backward(g_err.to(dt))
    return err.detach().double(), d.grad.double(), wp.grad.double()


def _clear_of_kinks(depth, wparam, bwd, idx):
    """(b, n) mask of the candidates whose residuals all lie at least tau from zero, tau = 4x the float32
    oracle's largest residual error, with tau.  The sweep's error is an L1 norm: at a residual within
    rounding of zero, rounding picks the sign of its gradient, and one flipped sign on a candidate that
    carries a cotangent moves a whole frame's gradient (through that candidate's pose gradient) far past
    float32 noise.  A cotangent that is zero on every other candidate has no such ambiguity."""
    from oracle import flowmap_oracle as O
    weights = torch.sigmoid(100.0 * wparam)
    r64, r32 = (O.softmin_residuals(depth.to(dt), weights.to(dt), bwd.to(dt), idx, _candidates(dt)).double()
                for dt in (torch.float64, torch.float32))
    tau = 4 * float((r32 - r64).abs().max())
    return ~(r64.abs() < tau).any(dim=-1).any(dim=-1), tau


def _flow_loss_cotangent(depth, wparam, fl, idx):
    """d loss / d err of the float64 oracle's flow loss when K comes from the softmin over the sweep's
    errors: what the loss really sends back through the softmin."""
    from test_gpu_parity import _oracle_flow_step
    return _oracle_flow_step(depth, wparam, fl, softmin=(idx, _candidates(torch.float64)))[4]


def _fmt(x):
    return f"{x:.1e}"


@pytest.mark.parametrize("npts", [300, 8192, None], ids=["p300", "p8192", "all"])
@pytest.mark.parametrize("b,f,h,w", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("kind", KINDS)
def test_sweep_errors_vs_float64_oracle(kind, b, f, h, w, npts):
    """ops.softmin_errors (k_moments<1> -> k_sweep_scale_solve -> k_sweep<false>) and k_softmin_focal:
    every candidate's error relative to its own value, the softmin weights and f_hat; the all-pixel
    case also without correspondence weights."""
    from flowmap_b200 import ops
    depth, wparam, fl, _ = _case(kind, b, f, h, w)
    idx = _sweep_indices(npts, h, w)
    idx_cpu = idx.cpu()
    cand = _candidates(torch.float32).cuda()
    for use_weights in ((True, False) if npts is None else (True,)):
        e64 = _oracle_sweep(depth, wparam, fl.backward, idx_cpu, torch.float64, use_weights)
        e32 = _oracle_sweep(depth, wparam, fl.backward, idx_cpu, torch.float32, use_weights)
        wts = torch.sigmoid(100.0 * wparam.float().cuda()) if use_weights else None
        err = ops.softmin_errors(depth.float().cuda(), wts, fl.backward.float().cuda(), idx, cand)
        sm, fh = _gpu_softmin(err, cand)
        sm64, fh64 = _softmin(e64, _candidates(torch.float64))
        sm32, fh32 = _softmin(e32, _candidates(torch.float64))
        got = dict(err=float(((err.double().cpu() - e64) / e64).abs().max()),
                   softmin=max_abs(sm.cpu(), sm64), f_hat=max_abs(fh.cpu(), fh64))
        noise = dict(err=float(((e32 - e64) / e64).abs().max()), softmin=max_abs(sm32, sm64), f_hat=max_abs(fh32, fh64))
        label = f"sweep {kind} {b}x{f}x{h}x{w} {idx.numel()} pts{'' if use_weights else ' no weights'}"
        print(label, "f_hat", [_fmt(float(x)) for x in fh64], "max softmin", _fmt(float(sm64.max())),
              "| errors vs float64 oracle:", {k: _fmt(v) for k, v in got.items()},
              "| float32 oracle:", {k: _fmt(v) for k, v in noise.items()})
        # f_hat sums the softmin weights' errors with signs: the float32 oracle's f_hat error ranges over
        # 1e-7 - 2.4e-5 at these shapes depending on how they cancel, hence a floor above that range
        floors = dict(err=1e-6, softmin=1e-5, f_hat=3e-5)
        for key, floor in floors.items():
            assert got[key] <= max(floor, 3 * noise[key]), (label, key, got[key], noise[key])


@pytest.mark.parametrize("b,f,h,w", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("kind", KINDS)
def test_sweep_backward_vs_float64_oracle(kind, b, f, h, w):
    """fm_softmin_sweep_bwd (k_sweep<true> -> k_adjoint -> k_sweep_aggregate -> k_distribute<1>) on 300
    points, under three cotangents on the errors: a seeded random one, the same weighted by the softmin
    weights, and the one the flow loss sends through the softmin.  Each is restricted to the candidates
    without a residual at the L1 kink (_clear_of_kinks: 37 to all 60 per item here).  With 8192 points
    nearly every candidate has such residuals, so that size is covered by the fused softmin stage below.
    Checks: depth gradient of frames 0 and 1 (whole frame and border band) and weight gradient of pair 0
    against oracle autograd, exactly zero on frames >= 2, pairs >= 1 and off the index set, and with
    b = 2 every batch item's gradient from its own inputs only."""
    from flowmap_b200 import ops
    depth, wparam, fl, _ = _case(kind, b, f, h, w)
    cand = _candidates(torch.float32).cuda()
    band = border_band(h, w)
    d_in, bwd = depth.float().cuda(), fl.backward.float().cuda()

    def gpu(g_err, d0=d_in):
        d = d0.clone().requires_grad_(True)
        wp = wparam.float().cuda().requires_grad_(True)
        err = ops.softmin_errors(d, torch.sigmoid(100.0 * wp), bwd, idx, cand)
        err.backward(g_err.float().cuda())
        return err.detach(), d.grad.double().cpu(), wp.grad.double().cpu()

    idx = _sweep_indices(300, h, w)
    idx_cpu = idx.cpu()
    off_set = torch.ones(h * w, dtype=torch.bool)
    off_set[idx_cpu] = False
    clear, tau = _clear_of_kinks(depth, wparam, fl.backward, idx_cpu)
    sm64 = _softmin(_oracle_sweep(depth, wparam, fl.backward, idx_cpu, torch.float64), _candidates(torch.float64))[0]
    gen = torch.Generator().manual_seed(h + w)
    rand = torch.randn(b, N_CAND, generator=gen, dtype=torch.float64)
    on = f"on the {int(clear.sum())} of {b * N_CAND} candidates clear of zero by {tau:.0e}"
    cotangents = [(f"random cotangent {on}", clear * rand),
                  (f"softmin-weighted random cotangent {on}", clear * sm64 * rand),
                  (f"flow-loss cotangent {on}", clear * _flow_loss_cotangent(depth, wparam, fl, idx_cpu))]
    for name, g_err in cotangents:
        _, gd64, gw64 = _oracle_sweep(depth, wparam, fl.backward, idx_cpu, torch.float64, g_err=g_err)
        _, gd32, gw32 = _oracle_sweep(depth, wparam, fl.backward, idx_cpu, torch.float32, g_err=g_err)
        _, gd, gw = gpu(g_err)
        label = f"sweep bwd {kind} {b}x{f}x{h}x{w} {idx.numel()} pts, {name}"
        got, noise = {}, {}
        for i in range(b):
            for fr in (0, 1):
                for key, m in ((f"depth[{i},{fr}]", slice(None)), (f"depth_border[{i},{fr}]", band)):
                    got[key] = rel_l2(gd[i, fr][m], gd64[i, fr][m])
                    noise[key] = rel_l2(gd32[i, fr][m], gd64[i, fr][m])
            got[f"weights[{i},0]"] = rel_l2(gw[i, 0], gw64[i, 0])
            noise[f"weights[{i},0]"] = rel_l2(gw32[i, 0], gw64[i, 0])
        print(label, "errors vs float64 oracle:", {k: _fmt(v) for k, v in got.items()},
              "| float32 oracle:", {k: _fmt(v) for k, v in noise.items()})
        for key in got:
            assert got[key] <= max(1e-4, 3 * noise[key]), (label, key, got[key], noise[key])
        assert float(gd[:, 2:].abs().max()) == 0.0, (label, "depth gradient on frames >= 2")
        assert float(gw[:, 1:].abs().max()) == 0.0, (label, "weight gradient on pairs >= 1")
        assert float(gw[:, 0].reshape(b, h * w)[:, off_set].abs().sum()) == 0.0, \
            (label, "weight gradient off the index set")
        if b == 2:
            # item 1 without a cotangent: no gradient at all, item 0's unchanged
            g0 = g_err.clone()
            g0[1] = 0
            _, gd_0, gw_0 = gpu(g0)
            assert float(gd_0[1].abs().max()) == 0.0 and float(gw_0[1].abs().max()) == 0.0, label
            # (the weight gradient sums the candidates' terms in atomic order, with cancellation)
            assert rel_l2(gd_0[0], gd[0]) <= 1e-5 and rel_l2(gw_0[0], gw[0]) <= 1e-4, label
            # item 1 on other depths: item 0's errors and gradients unchanged
            other = d_in.clone()
            other[1] = d_in[0].flip(-1)
            err_a, gd_a, gw_a = gpu(g_err)
            err_b, gd_b, gw_b = gpu(g_err, other)
            assert max_abs(err_b[0].cpu(), err_a[0].cpu()) <= 1e-6 * float(err_a[0].abs().max()), label
            assert rel_l2(gd_b[0], gd_a[0]) <= 1e-5 and rel_l2(gw_b[0], gw_a[0]) <= 1e-4, label


def _index_set(name, h, w, f):
    from flowmap_b200.model import ExtrinsicsProcrustes, ExtrinsicsProcrustesCfg
    if name == "linspace":
        return ExtrinsicsProcrustes(ExtrinsicsProcrustesCfg("procrustes", 1000, False), f).select_indices(h, w, "cuda")
    if name == "randint":
        torch.manual_seed(h * w)
        return ExtrinsicsProcrustes(ExtrinsicsProcrustesCfg("procrustes", 1000, True), f).select_indices(h, w, "cuda")
    return torch.randperm(h * w, generator=torch.Generator().manual_seed(w))[:2000].cuda()


@pytest.mark.parametrize("points", ["linspace", "randint", "randperm"])
@pytest.mark.parametrize("b,f,h,w", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("kind", KINDS)
def test_subsampled_procrustes_vs_float64_oracle(kind, b, f, h, w, points):
    """ops.procrustes_poses on a point set (k_moments<1> / k_distribute<1>) + ops.flow_loss in the full
    and shared_focal modes: the reference's 1000 linspace points (built on CUDA, as it builds them),
    randint points with duplicates (randomize_points) and a randperm prefix.  The weight gradient is
    zero off the set, and a duplicated point carries its gradient once per occurrence, as the oracle's
    gather does."""
    from flowmap_b200 import ops
    depth, wparam, fl, focal = _case(kind, b, f, h, w)
    idx = _index_set(points, h, w, f)
    idx_cpu = idx.cpu()
    count = torch.bincount(idx_cpu, minlength=h * w)
    if points == "randint":
        assert int((count > 1).sum()) > 0, "no duplicated point"
    refs = oracle_steps(depth, wparam, fl, focal, indices=idx_cpu)
    noise = errors(refs[32], refs[64])
    d = depth.float().cuda().requires_grad_(True)
    wp = wparam.float().cuda().requires_grad_(True)
    foc = torch.tensor(focal, dtype=torch.float32, device="cuda", requires_grad=True)
    s = (h * w) ** 0.5
    half = torch.tensor(0.5, device="cuda")
    k4 = torch.stack((foc * s / w, foc * s / h, half, half)).expand(b, f, 4)
    flc = [t.float().cuda() for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)]
    rt = ops.procrustes_poses(d, torch.sigmoid(100.0 * wp), k4, flc[1], idx)
    ext = ops.pose_chain(rt.detach()).cpu()
    for mode in ("full", "shared_focal"):
        d.grad = wp.grad = foc.grad = None
        loss = ops.flow_loss(d, rt, k4, *flc, ops.mask_sum(flc[2], flc[3]), "huber", 0.01, 1000.0, mode)
        loss.backward(retain_graph=True)
        gw = wp.grad.cpu()
        out = dict(loss=float(loss), ext=ext, g_depth=d.grad.cpu(), g_w=gw, g_focal=float(foc.grad))
        label = f"procrustes {kind} {b}x{f}x{h}x{w} {points} {idx.numel()} pts {mode}"
        check(errors(out, refs[64]), noise, label, loss_tol=1e-4, pose_tol=2e-5, floor=1e-4)
        gw_flat = gw.reshape(b, f - 1, h * w)
        assert float(gw_flat[..., count == 0].abs().max()) == 0.0, (label, "weight gradient off the point set")
        dup = count > 1
        if bool(dup.any()):
            r64, r32 = (refs[k]["g_w"].reshape(b, f - 1, h * w)[..., dup] for k in (64, 32))
            e, n = rel_l2(gw_flat[..., dup], r64), rel_l2(r32, r64)
            print(label, f"duplicated points ({int(dup.sum())}): weight gradient error {e:.1e} | float32 oracle {n:.1e}")
            assert e <= max(1e-4, 3 * n), (label, "weight gradient at duplicated points", e, n)


FUSED_CASES = [("scene", None), ("leave", None), ("zoom", None), ("scene", 1000)]


# red: the global-RED backward
@pytest.mark.parametrize("kind,npts", FUSED_CASES,
                         ids=[f"{k}-red{'' if n is None else f'-pts{n}'}" for k, n in FUSED_CASES])
def test_fused_softmin_stage_vs_float64_oracle(kind, npts):
    """fm_overfit_step in the softmin stage with 8192 injected sweep points: one step without the update
    (loss, f_hat, poses, gradients per frame and pair), then 3 Adam steps against the oracle's
    trajectory.  The all-pixel update steps take the early moment pass (moments at the candidate-0
    intrinsics, rescaled inside the step), fuse the weight Adam of pairs >= 1 into the step and leave pair 0
    to the sweep's backward.  With 1000 Procrustes points the weight gradient is sparse and its Adam runs on
    its own."""
    from oracle import flowmap_oracle as O
    from flowmap_b200.overfit import FusedOverfitter, OverfitCfg
    from flowmap_b200.types import Batch, Flows, Tracks
    f, h, w = 6, 96, 192
    depth, fl, focal, ext = O.flow_regime(kind, f, h, w, seed=31)
    tracking = kind == "scene"
    tracks = O.scene_tracks(depth[0], ext, focal, [(0, f), (2, 3), (f - 2, 2)], n_points=600, seed=32) \
        if tracking else None
    depth, _ = start_point(depth, focal, seed=33)
    depth = depth[0]
    wparam = 0.01 * torch.randn(f - 1, h, w, generator=torch.Generator().manual_seed(34), dtype=torch.float64)
    sweep_idx = torch.randperm(h * w, generator=torch.Generator().manual_seed(35))[:8192].cuda()
    kw = dict(intrinsics="softmin", regression_after=None, procrustes_points=npts, use_tracking=tracking,
              tracking_enable_after=0)

    batch = Batch(torch.zeros(1, 1, 1, 1, 1).expand(1, f, 3, h, w), torch.arange(f)[None], ["s"], ["d"])
    o = FusedOverfitter(OverfitCfg(**kw), batch,
                        Flows(*(t.float() for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask))),
                        None if tracks is None else [Tracks(t.xy.float(), t.visibility, t.start_frame) for t in tracks])
    o.injected_indices = sweep_idx
    with torch.no_grad():
        o.model.backbone.depth.copy_(depth.float())
        o.model.backbone.weights.copy_(wparam.float())
    pts = None if o._indices is None else o._indices.cpu()

    def oracle(dt):
        st = O.OverfitOracle(O.OverfitConfig(**kw), f, h, w, dtype=dt)
        with torch.no_grad():
            st.depth.copy_(depth.to(dt))
            st.weights.copy_(wparam.to(dt))
        flows = O.Flows(*(t.to(dt) for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))
        trk = None if tracks is None else [O.Tracks(t.xy.to(dt), t.visibility, t.start_frame) for t in tracks]
        return st, lambda: st.training_step(flows, trk, softmin_indices=sweep_idx.cpu(), procrustes_idx=pts)

    def as_out(r):
        return dict(loss=r["loss"], ext=r["extrinsics"].double(), g_depth=r["grads"]["depth"].double(),
                    g_w=r["grads"]["weights"].double(), g_focal=None, fx=float(r["intrinsics"][0, 0, 0, 0]))

    st64, step64 = oracle(torch.float64)
    ref = [as_out(step64()) for _ in range(3)]
    step32 = oracle(torch.float32)[1]
    ref32 = [as_out(step32()) for _ in range(3)]
    noise = errors(ref32[0], ref[0])
    label = f"fused softmin {kind} {f}x{h}x{w}{' tracking' if tracking else ''}, " \
            f"{'all pixels' if npts is None else f'{npts} Procrustes points'}"

    loss, _ = o.training_step(update=False)
    gr = o.gradients()
    fx = float(o.intrinsics_k4()[0, 0])
    out = dict(loss=float(loss), ext=o.extrinsics().cpu(), g_depth=gr["depth"].cpu(), g_w=gr["weights"].cpu())
    e = errors(out, ref[0])
    # frames 0-1 and pair 0 carry the sweep's backward: name them
    for key, names in (("depth_frame", ("frame 0", "frame 1")), ("weights_pair", ("pair 0",))):
        for i, name in enumerate(names):
            print(label, f"{key} {name}: {e[key][i]:.1e} | float32 oracle {noise[key][i]:.1e}")
            assert e[key][i] <= max(1e-4, 3 * noise[key][i]), (label, name, e[key][i], noise[key][i])
    fx_err, fx_noise = abs(fx - ref[0]["fx"]), abs(ref32[0]["fx"] - ref[0]["fx"])
    print(label, f"fx {ref[0]['fx']:.6f}: error {fx_err:.1e} | float32 oracle {fx_noise:.1e}")
    assert fx_err <= max(1e-5, 3 * fx_noise), (label, "fx", fx_err, fx_noise)
    check(e, noise, label, loss_tol=1e-4, pose_tol=2e-5, floor=1e-4)

    for s in range(3):
        total, _ = o.training_step()
        l_err = abs(float(total) - ref[s]["loss"]) / abs(ref[s]["loss"])
        fx_err, fx_noise = abs(float(o.intrinsics_k4()[0, 0]) - ref[s]["fx"]), abs(ref32[s]["fx"] - ref[s]["fx"])
        print(label, f"Adam step {s}: loss error {l_err:.1e}, fx error {fx_err:.1e} | float32 oracle {fx_noise:.1e}")
        assert l_err <= 1e-4 and fx_err <= max(1e-5, 3 * fx_noise), (label, s, l_err, fx_err, fx_noise)
    d_err = rel_l2(o.model.backbone.depth.detach().cpu(), st64.depth.detach())
    upd = o.model.backbone.weights.detach().cpu().double() - wparam
    w_err = rel_l2(upd, st64.weights.detach() - wparam)
    print(label, f"after 3 Adam steps: depth {d_err:.1e}, weight update {w_err:.1e}")
    assert d_err <= 1e-5 and w_err <= 2e-2, (label, d_err, w_err)


@pytest.mark.parametrize("h,w", [(360, 640), (720, 1280), (360, 480)])
def test_procrustes_index_set_follows_the_reference_rule(h, w):
    """ExtrinsicsProcrustes.select_indices builds the reference's 1000 linspace points on the device, as
    extrinsics_procrustes.py does.  Whether the CPU's int64 linspace gives the same set is printed: the
    oracle comparisons hand the oracle the device's tensor either way."""
    from flowmap_b200.model import ExtrinsicsProcrustes, ExtrinsicsProcrustesCfg
    got = ExtrinsicsProcrustes(ExtrinsicsProcrustesCfg("procrustes", 1000, False), 3).select_indices(h, w, "cuda")
    want = torch.linspace(0, h * w - 1, 1000, dtype=torch.int64, device="cuda")
    assert got.dtype == torch.int64 and torch.equal(got, want)
    cpu = torch.linspace(0, h * w - 1, 1000, dtype=torch.int64)
    diff = int((got.cpu() != cpu).sum())
    print(f"{h}x{w}: device linspace differs from the CPU's in {diff} of 1000 indices")
