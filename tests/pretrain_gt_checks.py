"""The oracle's pretraining step with ground-truth intrinsics (pretrain.py with model/intrinsics=ground_truth) on a
batch of B videos, shared by the CPU golden test (test_pretrain_gt_golden.py) and the GPU test
(test_gpu_ground_truth_surface.py).

As in pretrain_checks.pretrain_oracle, the batch's loss is 1000 x LossFlow with one mask sum M pooled over every
video, loss = sum_b num_b / (M or 1), evaluated one video at a time; K is given per video and per frame
(intrinsics_ground_truth.py), so there is no sweep and no focal length."""
import torch


def pretrain_gt_oracle(depths, weights, flows, intrinsics, procrustes_indices=None, mapping="huber",
                       dtype=torch.float64, use_weights=True, weight=1000.0, delta=0.01):
    """depths (B, F, H, W), weights (B, F-1, H, W), Flows of (B, F-1, ...) tensors and intrinsics (B, F, 3, 3)
    (any dtype: cast to `dtype` on the CPU); procrustes_indices the Procrustes point set (None: every pixel).
    Without correspondence weights the `weights` are replaced by ones (model.py:67-68) and get no gradient.

    Returns a dict of float64 CPU values: loss (float), share (B,) = weight x num_b / (M or 1), ext (B, F, 4, 4),
    g_depth (B, F, H, W), g_w (B, F-1, H, W) or None, mask_sum M (float)."""
    from oracle import flowmap_oracle as O
    b, f, h, w = depths.shape
    cpu = lambda t: t.detach().to("cpu", dtype)  # noqa: E731
    fl = [cpu(t) for t in (flows.forward, flows.backward, flows.forward_mask, flows.backward_mask)]
    m = float(fl[2].sum() + fl[3].sum())
    den = m if m != 0.0 else 1.0  # loss_flow.py:70 "valid_sum or 1"
    k_all = cpu(intrinsics)
    idx = torch.arange(h * w) if procrustes_indices is None else procrustes_indices.detach().cpu()
    xy = O.pixel_grid(h, w, dtype)
    out = {k: [] for k in ("share", "ext", "g_depth", "g_w")}
    for v in range(b):
        d = cpu(depths[v:v + 1]).requires_grad_(True)
        wt = cpu(weights[v:v + 1]).requires_grad_(True) if use_weights else torch.ones_like(cpu(weights[v:v + 1]))
        fv = O.Flows(*(t[v:v + 1] for t in fl))
        kf = k_all[v:v + 1]
        surf = O.unproject(xy, d, kf[:, :, None, None])
        ext = O.align_surfaces(surf, fv.backward, wt, idx)
        fwd = O.robust_map(O.forward_flow_positions(surf, ext, kf) - xy, fv.forward, h, w, mapping, delta)
        bwd = O.robust_map(O.backward_flow_positions(surf, ext, kf) - xy, fv.backward, h, w, mapping, delta)
        share = weight * ((fwd * fv.forward_mask).sum() + (bwd * fv.backward_mask).sum()) / den
        grads = torch.autograd.grad(share, [d, wt] if use_weights else [d], allow_unused=True)
        zero = lambda g, t: torch.zeros_like(t) if g is None else g  # noqa: E731
        out["share"].append(float(share.detach()))
        out["ext"].append(ext[0].detach().double())
        out["g_depth"].append(zero(grads[0], d)[0].double())
        if use_weights:
            out["g_w"].append(zero(grads[1], wt)[0].double())
    res = {"share": torch.tensor(out["share"], dtype=torch.float64), "ext": torch.stack(out["ext"]),
           "g_depth": torch.stack(out["g_depth"]), "g_w": torch.stack(out["g_w"]) if use_weights else None,
           "mask_sum": m}
    res["loss"] = float(res["share"].sum())
    return res
