"""Checks the analytic forward/backward formulas that the CUDA kernels instantiate
(flowmap_b200/csrc/fm_pixel.cuh, fm_procrustes.cuh) by compiling the same headers with g++
and driving them serially on the CPU (tests/host_emulation/emu.cpp, test-only), against the
golden vectors of the reference.  Runs in the build container (no GPU)."""
import ctypes
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden, max_abs, rel_l2

EMU_DIR = ROOT / "tests" / "host_emulation"


@pytest.fixture(scope="module")
def emu():
    build = EMU_DIR / "_build"
    build.mkdir(exist_ok=True)
    so = build / "libemu.so"
    srcs = [EMU_DIR / "emu.cpp"] + sorted((ROOT / "flowmap_b200" / "csrc").glob("*.cuh"))
    if not so.exists() or any(s.stat().st_mtime > so.stat().st_mtime for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", str(so),
                               str(EMU_DIR / "emu.cpp")])
    lib = ctypes.CDLL(str(so))
    lib.emu_state_bytes.restype = ctypes.c_size_t
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def flow_pose_grad(flowacc, rt, B, F):
    """numpy twin of flow_pose_grad() in fm_kernels.cu."""
    g = np.zeros((B * (F - 1), 12))
    for pair in range(B * (F - 1)):
        bi, i = divmod(pair, F - 1)
        a = bi * F + i
        fa, fb = flowacc[a], flowacc[a + 1]
        R = rt[pair].reshape(3, 4)[:, :3].astype(np.float64)
        G = np.zeros((3, 4))
        G[:, :3] = fa[1:10].reshape(3, 3) + fb[13:22].reshape(3, 3)
        G[:, 3] = fb[22:25] - R @ fa[10:13]
        g[pair] = G.reshape(-1)
    return g


def flow_k4_grad(flowacc, B, F):
    g = np.zeros((B * F, 4))
    for fr in range(B * F):
        i = fr % F
        g[fr] = flowacc[fr, 25:29]
        if i > 0:
            g[fr] += flowacc[fr - 1, 29:33]
        if i < F - 1:
            g[fr] += flowacc[fr + 1, 33:37]
    return g


def _emulate(emu, depth, w, ff, fb, mf, mb, k4, indices, mapping, delta, weight, lean, focal_mode):
    """One flow-loss step through the per-pixel headers: Procrustes forward, the flow loss (k_flow's
    code, or k_flow_lean's with FOCAL = focal_mode), the pose gradient, the Procrustes backward.
    depth (B, F, H, W), w the weights (B, F-1, H, W), flows in their layouts, k4 (B*F, 4), all float32.
    Returns the loss, rt (B*(F-1), 12), the depth gradient, d loss / d weights, the intrinsics gradient
    (B*F, 4: flow_k4_grad's per-frame part plus the Procrustes backward's) and the flow loss's own depth
    gradient (`direct`)."""
    B, F_, H, W = depth.shape
    BP = B * (F_ - 1)
    rt = np.zeros((BP, 12), dtype=np.float32)
    state = np.zeros(BP * emu.emu_state_bytes(), dtype=np.uint8)
    idx = None if indices is None else np.ascontiguousarray(indices, dtype=np.int64)
    n_idx = 0 if idx is None else len(idx)
    emu.emu_procrustes_fwd(_p(depth), _p(k4), _p(fb), _p(w), _p(idx), n_idx, _p(rt), _p(state), B, F_, H, W)
    mask_sum = float(mf.astype(np.float64).sum() + mb.astype(np.float64).sum())
    g_depth = np.zeros_like(depth)
    flowacc = np.zeros((B * F_, 40), dtype=np.float64)
    if lean:
        emu.emu_flow_lean(_p(depth), _p(k4), _p(rt), _p(ff), _p(fb), _p(mf), _p(mb), ctypes.c_double(mask_sum),
                          mapping, ctypes.c_float(delta), ctypes.c_float(weight), focal_mode, _p(g_depth),
                          _p(flowacc), B, F_, H, W)
    else:
        emu.emu_flow(_p(depth), _p(k4), _p(rt), _p(ff), _p(fb), _p(mf), _p(mb), ctypes.c_double(mask_sum), mapping,
                     ctypes.c_float(delta), ctypes.c_float(weight), _p(g_depth), _p(flowacc), B, F_, H, W)
    g_rt = flow_pose_grad(flowacc, rt, B, F_)
    g_w = np.zeros_like(w)
    k4acc = np.zeros((B * F_, 4), dtype=np.float64)
    direct = g_depth.copy()
    emu.emu_procrustes_bwd(_p(depth), _p(k4), _p(fb), _p(w), _p(idx), n_idx, _p(state), _p(g_rt), _p(g_depth),
                           _p(g_w), _p(k4acc), B, F_, H, W)
    return dict(loss=flowacc[:, 0].sum(), rt=rt, g_depth=g_depth, g_w=g_w, direct=direct,
                g_k4=flow_k4_grad(flowacc, B, F_) + k4acc)


def _chain(rt, B, F_):
    """Camera-to-world extrinsics (B, F, 4, 4) of the relative poses, chained in float64 (the float32
    chain is checked on the GPU)."""
    ext = []
    for bi in range(B):
        P = [np.eye(4)]
        for i in range(F_ - 1):
            T = np.eye(4)
            T[:3] = rt[bi * (F_ - 1) + i].reshape(3, 4)
            P.append(P[-1] @ T)
        ext.append(np.stack(P))
    return np.stack(ext)


def _wparam_grad(g_w, wt):
    """d loss / d weight logits from d loss / d weights (weights = sigmoid(100 logits))."""
    return torch.as_tensor(g_w, dtype=torch.float64) * 100.0 * wt * (1 - wt)


def run_emulated_step(emu, g, mapping=0, focal=0.85, indices=None, delta=0.01, weight=1000.0,
                      lean=False):
    """One video of a golden case, K from one focal length; lean: k_flow_lean with FOCAL = true."""
    depth = np.ascontiguousarray(g["in_depth"], dtype=np.float32)
    F_, H, W = depth.shape
    wt = torch.sigmoid(100.0 * torch.as_tensor(g["in_wparam"], dtype=torch.float32))
    ff, fb, mf, mb = (np.ascontiguousarray(g[k], dtype=np.float32) for k in ("in_fwd", "in_bwd", "in_fmask", "in_bmask"))
    s = (H * W) ** 0.5
    k4 = np.tile(np.array([focal * s / W, focal * s / H, 0.5, 0.5], dtype=np.float32), (F_, 1))
    r = _emulate(emu, depth[None], wt.numpy(), ff, fb, mf, mb, k4, indices, mapping, delta, weight, lean, 1)
    g_focal = (r["g_k4"][:, 0] * s / W + r["g_k4"][:, 1] * s / H).sum()
    return dict(loss=r["loss"], extrinsics=_chain(r["rt"], 1, F_), g_depth=r["g_depth"][0],
                g_wparam=_wparam_grad(r["g_w"], wt.double()).numpy(), g_focal=g_focal, direct=r["direct"][0],
                rt=r["rt"])


CASES = [("flow_huber", 0, 0.85, None), ("flow_l1", 1, 0.85, None), ("flow_l2", 2, 0.85, None),
         ("flow_rough", 0, 1.3, None), ("flow_pts1000", 0, 0.85, 1000)]


@pytest.mark.parametrize("lean", [False, True])
@pytest.mark.parametrize("name,mapping,focal,npts", CASES)
def test_emulated_step_matches_reference(emu, name, mapping, focal, npts, lean):
    g64 = load_golden(name, f64=True)
    g32 = load_golden(name, f64=False)
    _, H, W = g64["in_depth"].shape
    idx = None if npts is None else torch.linspace(0, H * W - 1, npts, dtype=torch.int64).numpy()
    r = run_emulated_step(emu, g64, mapping=mapping, focal=focal, indices=idx, lean=lean)
    # float32 noise floor of the reference itself (float32 run vs float64 run of the reference)
    ref_noise_d = rel_l2(g32["g_depth"], g64["g_depth"])
    ref_noise_w = rel_l2(g32["g_wparam"], g64["g_wparam"])
    assert abs(r["loss"] - float(g64["loss"])) <= 2e-5 * abs(float(g64["loss"]))
    assert max_abs(r["extrinsics"], g64["extrinsics"]) <= 5e-6
    assert rel_l2(r["g_depth"], g64["g_depth"]) <= max(1e-4, 3 * ref_noise_d)
    assert rel_l2(r["g_wparam"], g64["g_wparam"]) <= max(1e-4, 3 * ref_noise_w)
    assert abs(r["g_focal"] - float(g64["g_focal"])) <= 1e-4 * abs(float(g64["g_focal"]))


@pytest.mark.parametrize("total,rounds,grid", [
    (33525, 1, 444), (33525, 9, 444), (134100, 37, 444),   # 149 pairs of 360x640 / 720x1280, 444 blocks
    (16762, 4, 444),                                        # one rank of an 8-way split at 720p
    (33525, 1, 396), (33525, 10, 396), (134100, 42, 396),  # the same on the H100 grid (132 SMs x 3)
    (16762, 5, 396),
    (7, 3, 5), (5, 8, 444), (1000, 1, 1), (4096, 16, 3), (0, 2, 4),
])
def test_item_decomposition_covers_every_item_once_and_is_balanced(emu, total, rounds, grid):
    """block_item_range of the persistent dense kernels (item_span in fm_math.cuh): the (round, block)
    spans tile the item list exactly, and the rotation between rounds keeps the blocks' totals within
    a couple of items of each other (one odd item per round, moved around)."""
    cover = np.zeros(max(total, 1), dtype=np.int32)
    minmax = np.zeros(2, dtype=np.int64)
    emu.emu_item_cover(ctypes.c_longlong(total), rounds, grid, _p(cover), _p(minmax))
    assert (cover[:total] == 1).all()
    if total >= grid * rounds:
        assert minmax[1] - minmax[0] <= 2


@pytest.mark.parametrize("mapping", [0, 1, 2], ids=["huber", "l1", "l2"])
def test_packed_two_point_term_equals_the_scalar_term(emu, mapping):
    """lean_term2 (two points as one float32x2 computation: k_flow_lean's pixel pairs, k_track_src's
    point pairs) against lean_term on each point, incl. a point behind the camera plane
    (z + eps == 0: the nan_to_num branch of projection.py:56) next to an ordinary one."""
    rng = np.random.default_rng(7)
    for case in range(200):
        D = rng.uniform(0.5, 2.0, 2).astype(np.float32)
        dirs = rng.normal(0, 0.3, (2, 3)).astype(np.float32)
        dirs[:, 2] = rng.uniform(0.7, 1.3, 2)
        off = rng.normal(0, 0.05, 3).astype(np.float32)
        if case % 10 == 0:  # first point exactly on the plane z + eps = 0
            dirs[0, 2] = 0.0
            off[2] = np.float32(-1e-5)
        k4 = np.array([0.9, 1.2, 0.5, 0.5], dtype=np.float32)
        xy = rng.uniform(0, 1, (2, 2)).astype(np.float32)
        fl = rng.normal(0, 0.01, (2, 2)).astype(np.float32)
        out, out2 = np.zeros(14, np.float32), np.zeros(14, np.float32)
        emu.emu_lean_terms(_p(D), _p(dirs), _p(off), _p(k4), _p(xy), _p(fl), mapping, ctypes.c_float(0.01), 36, 48,
                           _p(out), _p(out2))
        ok = np.isfinite(out)
        assert (np.isfinite(out2) == ok).all()
        assert np.allclose(out2[ok], out[ok], rtol=2e-6, atol=1e-7), (case, out, out2)


@pytest.fixture(scope="module")
def regime_cases():
    """Oracle results of the flow regimes, computed once per (regime, shape) for both kernel variants."""
    return {}


@pytest.mark.parametrize("lean", [False, True])
@pytest.mark.parametrize("f,h,w", [(4, 40, 64), (4, 38, 63)])
@pytest.mark.parametrize("kind", ["iid", "shift", "leave", "outliers", "zoom", "scene"])
def test_emulated_step_in_flow_regimes_vs_float64_oracle(emu, regime_cases, kind, f, h, w, lean):
    """The kernels' per-pixel code on flows with large coherent motion, taps that leave the frame,
    outliers, zoom and a large-motion rigid scene (oracle.flow_regime): bilinear_taps' clipping to the
    border and its adjoint, without any GPU scheduling.  Gradients within max(2e-5, 3x the float32
    oracle's error), the depth gradient also on the one-pixel border band."""
    from oracle import flowmap_oracle as O
    from flow_regime_checks import check, errors, oracle_steps, start_point
    key = (kind, f, h, w)
    if key not in regime_cases:
        depth, fl, focal, _ = O.flow_regime(kind, f, h, w, seed=3)
        depth, focal = start_point(depth, focal, seed=5)
        wparam = 0.01 * torch.randn(1, f - 1, h, w, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
        refs = oracle_steps(depth, wparam, fl, focal)
        g = {"in_depth": depth[0].numpy(), "in_wparam": wparam[0].numpy(), "in_fwd": fl.forward.numpy(),
             "in_bwd": fl.backward.numpy(), "in_fmask": fl.forward_mask.numpy(), "in_bmask": fl.backward_mask.numpy()}
        regime_cases[key] = (g, focal, refs, errors(refs[32], refs[64], per_item=False))
    g, focal, refs, noise = regime_cases[key]
    r = run_emulated_step(emu, g, focal=focal, lean=lean)
    out = dict(loss=r["loss"], ext=torch.as_tensor(r["extrinsics"]), g_depth=torch.as_tensor(r["g_depth"]),
               g_w=torch.as_tensor(r["g_wparam"]), g_focal=r["g_focal"])
    check(errors(out, refs[64], per_item=False), noise, f"{kind} {f}x{h}x{w} lean={lean}",
          loss_tol=1e-4, pose_tol=1e-5, floor=2e-5)


def run_emulated_step_k4(emu, depth, wparam, flows, k4, indices=None, lean=False):
    """One flow-loss step on b videos (b, f, h, w) under per-frame intrinsics k4 (b, f, 4).  lean:
    k_flow_lean's code with FOCAL = false (k_mode "const": the flow loss gives K no gradient), else
    k_flow's (k_mode "full").  g_k4 (b, f, 4)."""
    B, F_, H, W = depth.shape
    wt = torch.sigmoid(100.0 * wparam.float())
    f32 = lambda t: np.ascontiguousarray(t.numpy(), dtype=np.float32)  # noqa: E731
    r = _emulate(emu, f32(depth), f32(wt), f32(flows.forward), f32(flows.backward), f32(flows.forward_mask),
                 f32(flows.backward_mask), f32(k4), indices, 0, 0.01, 1000.0, lean, 0)
    return dict(loss=r["loss"], ext=torch.as_tensor(_chain(r["rt"], B, F_)), g_depth=torch.as_tensor(r["g_depth"]),
                g_w=_wparam_grad(r["g_w"], wt.double()), g_k4=torch.as_tensor(r["g_k4"]).reshape(B, F_, 4))


@pytest.fixture(scope="module")
def k4_cases():
    """Oracle results under per-frame intrinsics, computed once per (K regime, flows, points)."""
    return {}


@pytest.mark.parametrize("lean", [False, True], ids=["full", "lean-const"])
@pytest.mark.parametrize("points", [None, "linspace"], ids=["all", "pts300"])
@pytest.mark.parametrize("flows", ["shift", "scene"])
@pytest.mark.parametrize("kregime", ["offcentre", "zoom", "corner", "videos"])
def test_emulated_step_with_per_frame_intrinsics_vs_float64_oracle(emu, k4_cases, kregime, flows, points, lean):
    """The per-pixel code under the intrinsics of calibrated videos (flow_regime_checks.k4_regime): per-frame,
    off-centre, anisotropic K, a different K per video (B = 2), on the all-pixel and the index Procrustes
    paths.  A frame that reads its neighbour's K, or a principal point taken as 0.5, is wrong here and nowhere
    with the focal-length K of the other cases.  The intrinsics gradient is checked per video, frame and
    component: both routes that place it (flow_k4_grad's neighbour slots, distribute_point's kacc halves)."""
    from oracle import flowmap_oracle as O
    from flow_regime_checks import check, errors, k4_errors, k4_regime, k4_scene, oracle_steps_k4
    b, f, h, w = 2, 4, 24, 32
    key = (kregime, flows, points)
    if key not in k4_cases:
        k4 = k4_regime(kregime, b, f, h, w)
        if flows == "scene":
            depth, fl = k4_scene(k4, h, w, seed=11)
        else:
            depth, fl, _, _ = O.flow_regime(flows, f, h, w, seed=11, b=b)
        depth = depth * (1.0 + 0.02 * torch.randn(depth.shape, generator=torch.Generator().manual_seed(12),
                                                  dtype=torch.float64))
        # the kernels see float32 inputs: give the oracle the same values, so input rounding is not error
        depth, k4 = depth.float().double(), k4.float().double()
        fl = O.Flows(*(t.float().double() for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)))
        wparam = (0.01 * torch.randn(b, f - 1, h, w, generator=torch.Generator().manual_seed(13),
                                     dtype=torch.float64)).float().double()
        idx = None if points is None else torch.linspace(0, h * w - 1, 300, dtype=torch.int64)
        refs = oracle_steps_k4(depth, wparam, fl, k4, idx)
        k4_cases[key] = (depth, wparam, fl, k4, idx, refs)
    depth, wparam, fl, k4, idx, refs = k4_cases[key]
    r = run_emulated_step_k4(emu, depth, wparam, fl, k4, None if idx is None else idx.numpy(), lean)
    gk = "g_k4_const" if lean else "g_k4"
    noise = errors(refs[32], refs[64])
    noise.update(k4_errors(refs[32][gk], refs[64][gk], noise=True))
    errs = errors(dict(r, g_focal=None), refs[64])
    errs.update(k4_errors(r["g_k4"], refs[64][gk]))
    check(errs, noise, f"{kregime} {flows} {points} lean={lean}", loss_tol=1e-4, pose_tol=1e-5, floor=2e-5)


def _distribute_both(emu, depth, wt, fl, k4):
    """distribute_point<true> and <false> (the constant-intrinsics kernels' phase D2) on every pixel of one step's
    pose gradient: {kgrad: (g_db, g_w, taps, points whose kacc moved)}."""
    B, F_, H, W = depth.shape
    BP, N = B * (F_ - 1), H * W
    f32 = lambda t: np.ascontiguousarray(t.numpy(), dtype=np.float32)  # noqa: E731
    d, w, k = f32(depth), f32(wt), f32(k4)
    ff, fb, mf, mb = (f32(getattr(fl, n)) for n in ("forward", "backward", "forward_mask", "backward_mask"))
    rt = np.zeros((BP, 12), dtype=np.float32)
    state = np.zeros(BP * emu.emu_state_bytes(), dtype=np.uint8)
    emu.emu_procrustes_fwd(_p(d), _p(k), _p(fb), _p(w), None, 0, _p(rt), _p(state), B, F_, H, W)
    flowacc = np.zeros((B * F_, 40), dtype=np.float64)
    mask_sum = float(mf.astype(np.float64).sum() + mb.astype(np.float64).sum())
    emu.emu_flow(_p(d), _p(k), _p(rt), _p(ff), _p(fb), _p(mf), _p(mb), ctypes.c_double(mask_sum), 0,
                 ctypes.c_float(0.01), ctypes.c_float(1000.0), _p(np.zeros_like(d)), _p(flowacc), B, F_, H, W)
    g_rt = np.ascontiguousarray(flow_pose_grad(flowacc, rt, B, F_))
    out = {}
    for kgrad in (1, 0):
        g_db, g_w = np.zeros(BP * N, np.float32), np.zeros(BP * N, np.float32)
        taps = np.zeros(BP * N * 8, np.float32)
        moved = np.zeros(1, np.int64)
        emu.emu_distribute(_p(d), _p(k), _p(fb), _p(w), _p(state), _p(g_rt), kgrad, _p(g_db), _p(g_w), _p(taps),
                           _p(moved), B, F_, H, W)
        out[kgrad] = (g_db, g_w, taps, int(moved[0]))
    return out


DISTRIBUTE_CASES = ([("flows", kind, (1, 4, 40, 64)) for kind in ("iid", "shift", "leave", "outliers", "zoom", "scene")] +
                    [("flows", kind, (1, 4, 38, 63)) for kind in ("iid", "shift", "leave", "outliers", "zoom", "scene")] +
                    [(kregime, flows, (2, 4, 24, 32)) for kregime in ("offcentre", "zoom", "corner", "videos")
                     for flows in ("shift", "scene")])


@pytest.mark.parametrize("kregime,flows,shape", DISTRIBUTE_CASES,
                         ids=[f"{k}-{fl}-{'x'.join(map(str, s))}" for k, fl, s in DISTRIBUTE_CASES])
def test_constant_intrinsics_distribute_equals_k_carrying(emu, kregime, flows, shape):
    """distribute_point<false> (k_distribute*<false>, the constant-intrinsics step's phase D2) against <true> on
    the flow regimes (focal-length K) and the per-frame K regimes: the later frame's depth gradient, the weight
    gradient and every scattered tap (row, column, both values) are bit-identical, and the K accumulators are
    not touched (<true> moves them)."""
    from oracle import flowmap_oracle as O
    from flow_regime_checks import k4_regime, k4_scene
    b, f, h, w = shape
    if kregime == "flows":
        depth, fl, focal, _ = O.flow_regime(flows, f, h, w, seed=3)
        s = (h * w) ** 0.5
        k4 = torch.tensor([focal * s / w, focal * s / h, 0.5, 0.5], dtype=torch.float64).expand(b, f, 4)
    else:
        k4 = k4_regime(kregime, b, f, h, w)
        if flows == "scene":
            depth, fl = k4_scene(k4, h, w, seed=11)
        else:
            depth, fl, _, _ = O.flow_regime(flows, f, h, w, seed=11, b=b)
    wt = torch.sigmoid(100.0 * 0.01 * torch.randn(b, f - 1, h, w, generator=torch.Generator().manual_seed(4),
                                                  dtype=torch.float64))
    out = _distribute_both(emu, depth, wt, fl, k4.reshape(b * f, 4))
    assert out[1][3] > 0 and out[0][3] == 0, (out[1][3], out[0][3])
    for name, a, c in zip(("g_db", "g_w", "taps"), out[1][:3], out[0][:3]):
        assert np.isfinite(a).all() and np.abs(a).max() > 0, name
        assert np.array_equal(a.view(np.uint32), c.view(np.uint32)), (name, int((a != c).sum()))
