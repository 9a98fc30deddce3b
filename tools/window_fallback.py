"""Fraction of the Procrustes-backward tap rows that miss the shared-memory window of
k_distribute_window and fall back to global REDs, computed on the host from the benchmark's flows
(window placement as in the kernel: tile + halo, shifted by the mean backward flow of 8 x 4 samples
of the tile, or by the flow at the tile centre for comparison).

  python tools/window_fallback.py [--tile 64 32] [--halo 16 12] [--shape 150 360 640] [--pairs 8]
"""
import argparse
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402


def smooth_flow(p, h, w, seed=100):
    g = torch.Generator().manual_seed(seed)
    coarse = 0.01 * torch.randn(p, 2, (h + 15) // 16 + 1, (w + 15) // 16 + 1, generator=g)
    up = torch.nn.functional.interpolate(coarse, size=(h, w), mode="bilinear", align_corners=True)
    return up.permute(0, 2, 3, 1).numpy()


def fallback_fraction(flow, tw, th, hx, hy, placement):
    """flow: (P, H, W, 2) backward flow in normalised units.  Returns missed / all scatter rows."""
    _, h, w, _ = flow.shape
    ww, wh = tw + 2 * hx, th + 2 * hy
    rows, cols = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    missed = total = 0
    for f in flow.astype(np.float32):
        px = np.clip(cols + f[..., 0] * w, 0, w - 1)  # bilinear_taps: (x + flx) W - .5, clipped
        py = np.clip(rows + f[..., 1] * h, 0, h - 1)
        x0 = np.floor(px).astype(np.int64)
        y0 = np.floor(py).astype(np.int64)
        y1 = np.minimum(y0 + 1, h - 1)
        for ty in range(0, h, th):
            for tx in range(0, w, tw):
                if placement == "mean":
                    sr = np.minimum(ty + (np.arange(32) >> 3) * (th // 4) + th // 8, h - 1)
                    sc = np.minimum(tx + (np.arange(32) & 7) * (tw // 8) + tw // 16, w - 1)
                    s = f[sr, sc].astype(np.float64).sum(0)
                else:  # the flow at the tile centre
                    s = 32.0 * f[min(ty + th // 2, h - 1), min(tx + tw // 2, w - 1)].astype(np.float64)
                shx = int(np.rint(np.clip(s[0] * w / 32 - 0.5, -w, w)))
                shy = int(np.rint(np.clip(s[1] * h / 32 - 0.5, -h, h)))
                wx0 = max(0, min((tx - hx + shx + 2) & ~3, w - ww))
                wy0 = max(0, min(ty - hy + shy, h - wh))
                sl = (slice(ty, ty + th), slice(tx, tx + tw))
                inx = (x0[sl] - wx0 >= 0) & (x0[sl] - wx0 < ww)
                for yy in (y0[sl], y1[sl]):
                    ok = inx & (yy - wy0 >= 0) & (yy - wy0 < wh)
                    missed += int((~ok).sum())
                    total += ok.size
    return missed / total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tile", type=int, nargs=2, default=(64, 32))
    ap.add_argument("--halo", type=int, nargs=2, default=(16, 12))
    ap.add_argument("--shape", type=int, nargs=3, default=(150, 360, 640))
    ap.add_argument("--pairs", type=int, default=8, help="frame pairs evaluated")
    a = ap.parse_args()
    f, h, w = a.shape
    p = min(a.pairs, f - 1)
    flows = {"iid": bench.synthetic_inputs(f, h, w, seed=0)["bwd"][0, :p].numpy(), "smooth": smooth_flow(p, h, w)}
    for kind, fl in flows.items():
        for placement in ("mean", "centre"):
            fr = fallback_fraction(fl, *a.tile, *a.halo, placement)
            print(f"{kind:6s} {placement:6s} tile {a.tile[0]}x{a.tile[1]} halo {a.halo[0]}x{a.halo[1]} "
                  f"at {h}x{w}: {100 * fr:.2f} % of tap rows fall back to REDs")


if __name__ == "__main__":
    main()
