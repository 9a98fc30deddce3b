"""The fixed-point scatter window of the Procrustes backward (k_distribute_window, W % 4 == 0)
against the float64 oracle on inputs that stress it: backward flows that pile the taps of a whole
tile onto a few cells, and correspondence weights far above 1 on a few pixels, whose tap values
lie beyond the range the pair's fixed-point scale covers and take the float fall-back."""
import pytest
import torch

from conftest import max_abs, rel_l2

pytestmark = pytest.mark.gpu


def _step_vs_oracle(depth, weights, fl):
    """One flow-loss step with the weights given directly (not as logits): loss, poses and the depth
    gradient of the CUDA path against the float64 oracle."""
    from oracle import flowmap_oracle as O
    from flowmap_b200 import ops
    b, f, h, w = depth.shape
    d64 = depth.clone().requires_grad_(True)
    k = O.intrinsics_from_focal(torch.tensor(0.85, dtype=torch.float64), h, w).expand(b, f, 3, 3)
    surf = O.unproject(O.pixel_grid(h, w, torch.float64), d64, k[:, :, None, None])
    ext_r = O.align_surfaces(surf, fl.backward, weights, torch.arange(h * w))
    loss_r = 1000.0 * O.flow_loss(surf, ext_r, k, fl, "huber", 0.01)
    loss_r.backward()
    d = depth.float().cuda().requires_grad_(True)
    s = (h * w) ** 0.5
    k4 = torch.tensor([0.85 * s / w, 0.85 * s / h, 0.5, 0.5], device="cuda").expand(b, f, 4).contiguous()
    flc = [t.float().cuda() for t in (fl.forward, fl.backward, fl.forward_mask, fl.backward_mask)]
    rt = ops.procrustes_poses(d, weights.float().cuda(), k4, flc[1], None)
    loss = ops.flow_loss(d, rt, k4, *flc, ops.mask_sum(flc[2], flc[3]), "huber", 0.01, 1000.0, "const")
    loss.backward()
    assert abs(float(loss) - float(loss_r)) <= 1e-4 * abs(float(loss_r))
    assert rel_l2(d.grad.cpu(), d64.grad) <= 1e-4
    assert max_abs(ops.pose_chain(rt).cpu(), ext_r.detach()) <= 1e-5


def _inputs(b, f, h, w, seed):
    from oracle import flowmap_oracle as O
    gen = torch.Generator().manual_seed(seed)
    depth = 1.0 + torch.rand(b, f, h, w, generator=gen, dtype=torch.float64)
    return gen, depth, O.synthetic_flows(f, h, w, seed=seed, dtype=torch.float64, b=b)


@pytest.mark.parametrize("b,f,h,w", [(1, 3, 64, 128), (1, 2, 72, 136)])
def test_taps_piled_onto_few_cells_vs_oracle(b, f, h, w):
    """Every pixel's backward flow points at 0.95 of the way to the centre of its 64 x 32 tile,
    so a tile's 2048 pixels add into a handful of cells of the window."""
    gen, depth, fl = _inputs(b, f, h, w, seed=11)
    ys = (torch.arange(h, dtype=torch.float64) + 0.5) / h
    xs = (torch.arange(w, dtype=torch.float64) + 0.5) / w
    cy = ((torch.arange(h) // 32) * 32 + 16).clamp(max=h - 1).double().add(0.5) / h
    cx = ((torch.arange(w) // 64) * 64 + 32).clamp(max=w - 1).double().add(0.5) / w
    bwd = torch.stack(torch.broadcast_tensors((0.95 * (cx - xs))[None, :], (0.95 * (cy - ys))[:, None]), -1)
    fl.backward = (bwd + 1e-4 * torch.randn(b, f - 1, h, w, 2, generator=gen, dtype=torch.float64)).contiguous()
    weights = torch.sigmoid(torch.randn(b, f - 1, h, w, generator=gen, dtype=torch.float64))
    _step_vs_oracle(depth, weights, fl)


@pytest.mark.parametrize("b,f,h,w", [(1, 3, 64, 128), (2, 2, 40, 100)])
def test_tap_values_beyond_the_fixed_point_range_vs_oracle(b, f, h, w):
    """One pixel in 64 carries a weight of 10^6 instead of about 1: the per-pair scale assumes
    weights up to 1, so these pixels' tap values exceed its range by far and are added as floats,
    next to the fixed-point sums of their neighbours in the same cells."""
    gen, depth, fl = _inputs(b, f, h, w, seed=12)
    weights = torch.sigmoid(torch.randn(b, f - 1, h, w, generator=gen, dtype=torch.float64))
    heavy = torch.rand(b, f - 1, h, w, generator=gen) < 1.0 / 64
    weights = torch.where(heavy, torch.full_like(weights, 1e6), weights)
    _step_vs_oracle(depth, weights, fl)
