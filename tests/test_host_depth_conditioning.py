"""The kernels' per-pixel Procrustes and flow-loss code (fm_pixel.cuh, fm_procrustes.cuh, compiled with
g++ by test_host_emulation.py) on depth maps whose centre pixel is not typical of the frame, on depth
scales far from 1 and on weights that sit in one corner (oracle.depth_regime), against the float64
oracle.

The moment sums are taken of points shifted by a per-pair conditioning depth, and the covariance is
recovered from them by cancellation; the shift also sets the fixed-point scale of the backward's
scatter window.  A shift far from the depth of the weighted cloud (a far horizon or a speckle at the
image centre) costs the sums their significant bits.  This runs without a GPU."""
import pytest
import torch

from flow_regime_checks import check, errors, oracle_steps, start_point
from test_host_emulation import emu, run_emulated_step  # noqa: F401  (emu is a fixture)

KINDS = ["centre_far", "centre_far_weighted", "horizon", "centre_near", "scale_small", "scale_large",
         "corner_weights"]


@pytest.fixture(scope="module")
def depth_cases():
    """Oracle results per (regime, shape), computed once for both kernel variants."""
    return {}


@pytest.mark.parametrize("lean", [False, True])
@pytest.mark.parametrize("f,h,w", [(4, 40, 64), (4, 38, 63)])
@pytest.mark.parametrize("kind", KINDS)
def test_emulated_step_in_depth_regimes_vs_float64_oracle(emu, depth_cases, kind, f, h, w, lean):  # noqa: F811
    """Loss within 1e-4, poses within 1e-5 and every gradient (per frame, per pair, on the border band)
    within max(2e-5, 3x the float32 oracle's error).  Where the float32 oracle itself misses the loss or
    pose tolerance (the badly conditioned `centre_far_weighted`), those two are held to
    3x its error as well."""
    from oracle import flowmap_oracle as O
    key = (kind, f, h, w)
    if key not in depth_cases:
        depth, fl, focal, wparam = O.depth_regime(kind, f, h, w, seed=3)
        depth, focal = start_point(depth, focal, seed=5)
        refs = oracle_steps(depth, wparam, fl, focal)
        g = {"in_depth": depth[0].numpy(), "in_wparam": wparam[0].numpy(), "in_fwd": fl.forward.numpy(),
             "in_bwd": fl.backward.numpy(), "in_fmask": fl.forward_mask.numpy(), "in_bmask": fl.backward_mask.numpy()}
        depth_cases[key] = (g, focal, refs, errors(refs[32], refs[64]))
    g, focal, refs, noise = depth_cases[key]
    r = run_emulated_step(emu, g, focal=focal, lean=lean)
    out = dict(loss=r["loss"], ext=torch.as_tensor(r["extrinsics"]), g_depth=torch.as_tensor(r["g_depth"]),
               g_w=torch.as_tensor(r["g_wparam"]), g_focal=r["g_focal"])
    check(errors(out, refs[64]), noise, f"{kind} {f}x{h}x{w} lean={lean}", loss_tol=1e-4, pose_tol=1e-5,
          floor=2e-5, relative_fixed=True)
