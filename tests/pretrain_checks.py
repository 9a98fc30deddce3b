"""The oracle's pretraining step (pretrain.py, model_wrapper_pretrain.py) on a batch of B videos, shared by the
CPU golden test (test_pretrain_golden.py) and the GPU tests (test_gpu_pretrain_at_scale.py).

The batch's loss is 1000 x LossFlow: one mask sum M pooled over every video (loss_flow.py:31-70), so

    loss = sum_b num_b / (M or 1),   num_b = video b's masked flow-error sum,

and the sweep's sample is shared by all videos while each video gets its own softmin focal length
(intrinsics_softmin.py:84-131).  The sweep and the poses of video b depend only on video b's depths, weights
and flows, so the step is evaluated one video at a time, exactly: num_b / M is video b's share, and its
gradient is d share_b / d (depths_b, weights_b).  That keeps the CPU memory of a 16-video float64 step to one
video's."""
import torch


def pretrain_oracle(depths, weights, flows, sweep_indices, candidates, procrustes_indices=None, mapping="huber",
                    dtype=torch.float64, use_weights=True, weight=1000.0, delta=0.01):
    """depths (B, F, H, W), weights (B, F-1, H, W) and Flows of (B, F-1, ...) tensors (any dtype: cast to
    `dtype` on the CPU); sweep_indices (P,) the sweep's sample; candidates (N,) the candidate focal lengths;
    procrustes_indices the Procrustes point set (None: every pixel).  Without correspondence weights the
    `weights` are replaced by ones (model.py:67-68) and get no gradient.

    Returns a dict of float64 CPU values: loss (float), share (B,) = weight x num_b / (M or 1), focal (B,)
    (normalised focal lengths), k (B, 3, 3), ext (B, F, 4, 4), g_depth (B, F, H, W), g_w (B, F-1, H, W) or
    None, mask_sum M (float)."""
    from oracle import flowmap_oracle as O
    b, f, h, w = depths.shape
    cpu = lambda t: t.detach().to("cpu", dtype)  # noqa: E731
    fl = [cpu(t) for t in (flows.forward, flows.backward, flows.forward_mask, flows.backward_mask)]
    m = float(fl[2].sum() + fl[3].sum())
    den = m if m != 0.0 else 1.0  # loss_flow.py:70 "valid_sum or 1"
    cand = candidates.detach().to("cpu", dtype)
    sweep_indices = sweep_indices.detach().cpu()
    idx = torch.arange(h * w) if procrustes_indices is None else procrustes_indices.detach().cpu()
    xy = O.pixel_grid(h, w, dtype)
    out = {k: [] for k in ("share", "focal", "k", "ext", "g_depth", "g_w")}
    for v in range(b):
        d = cpu(depths[v:v + 1]).requires_grad_(True)
        wt = cpu(weights[v:v + 1]).requires_grad_(use_weights) if use_weights else torch.ones_like(cpu(weights[v:v + 1]))
        fv = O.Flows(*(t[v:v + 1] for t in fl))
        k, sm = O.softmin_focal(d, wt, fv.backward, sweep_indices, cand)
        kf = k[:, None].expand(1, f, 3, 3)
        surf = O.unproject(xy, d, kf[:, :, None, None])
        ext = O.align_surfaces(surf, fv.backward, wt, idx)
        fwd = O.robust_map(O.forward_flow_positions(surf, ext, kf) - xy, fv.forward, h, w, mapping, delta)
        bwd = O.robust_map(O.backward_flow_positions(surf, ext, kf) - xy, fv.backward, h, w, mapping, delta)
        share = weight * ((fwd * fv.forward_mask).sum() + (bwd * fv.backward_mask).sum()) / den
        grads = torch.autograd.grad(share, [d, wt] if use_weights else [d], allow_unused=True)
        zero = lambda g, t: torch.zeros_like(t) if g is None else g  # noqa: E731
        out["share"].append(float(share.detach()))
        out["focal"].append(float((sm * cand).sum().detach()))
        out["k"].append(k[0].detach().double())
        out["ext"].append(ext[0].detach().double())
        out["g_depth"].append(zero(grads[0], d)[0].double())
        if use_weights:
            out["g_w"].append(zero(grads[1], wt)[0].double())
    res = {"share": torch.tensor(out["share"], dtype=torch.float64),
           "focal": torch.tensor(out["focal"], dtype=torch.float64),
           "k": torch.stack(out["k"]), "ext": torch.stack(out["ext"]), "g_depth": torch.stack(out["g_depth"]),
           "g_w": torch.stack(out["g_w"]) if use_weights else None, "mask_sum": m}
    res["loss"] = float(res["share"].sum())
    return res
