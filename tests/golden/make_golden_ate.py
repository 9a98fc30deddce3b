"""Golden vectors for the trajectory metric (misc/ate.py:7-25 compute_ate), generated from the
UNMODIFIED reference (FLOWMAP_REFERENCE names the root of its checkout):

    python tests/golden/make_golden_ate.py

Runs the reference's flowmap.misc.ate.compute_ate (torch, jaxtyping, scipy) on seeded float32
trajectories and stores, per case <name>: the inputs (<name>__gt, <name>__pred), whether the
reference raised ValueError (<name>__raised), its outputs (<name>__ate, <name>__aligned_gt,
<name>__aligned_pred, float32) and the float64 disparity of the scipy.spatial.procrustes call it
makes (<name>__disparity), from which the float64 ATE is sqrt(disparity / (3 F)).
"""
from __future__ import annotations

import os
import sys
from pathlib import Path

import numpy as np
import torch

REF = os.environ.get("FLOWMAP_REFERENCE", "reference")
OUT = Path(__file__).resolve().parent
ROOT = OUT.parent.parent


def _rotation(g: torch.Generator) -> torch.Tensor:
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    return q * torch.sign(torch.linalg.det(q))


def _walk(g: torch.Generator, f: int, step: float = 0.1) -> torch.Tensor:
    return torch.cumsum(step * torch.randn(f, 3, generator=g, dtype=torch.float64), dim=0)


def cases() -> dict:
    g = torch.Generator().manual_seed(11)
    out = {}
    gt = _walk(g, 150)
    sim = 0.5 * gt @ _rotation(g).T + torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64)
    out["similarity"] = (gt, sim + 0.01 * torch.randn(150, 3, generator=g, dtype=torch.float64))
    out["mirrored"] = (gt, 3.0 * gt @ torch.diag(torch.tensor([1.0, 1.0, -1.0], dtype=torch.float64)) + 5.0)
    far = 1e4 + _walk(g, 150, step=0.08)
    out["far"] = (far, far @ _rotation(g).T * 2.0 + 0.01 * torch.randn(150, 3, generator=g, dtype=torch.float64))
    out["f2"] = (torch.randn(2, 3, generator=g, dtype=torch.float64), torch.randn(2, 3, generator=g, dtype=torch.float64))
    out["f3"] = (torch.randn(3, 3, generator=g, dtype=torch.float64), torch.randn(3, 3, generator=g, dtype=torch.float64))
    planar = _walk(g, 100)
    planar[:, 2] = 0.0
    out["planar_gt"] = (planar, _walk(g, 100) + planar)
    t = torch.arange(-40, 60, dtype=torch.float64) / 8.0  # exact float32 multiples of one direction
    line = t[:, None] * torch.tensor([1.0, 2.0, -2.0], dtype=torch.float64)
    out["collinear_pred"] = (_walk(g, 100), line)
    long = _walk(g, 2000)
    out["f2000"] = (long, long @ _rotation(g).T + 0.05 * torch.randn(2000, 3, generator=g, dtype=torch.float64))
    out["unrelated"] = (_walk(g, 150), _walk(g, 150))
    sys.path.insert(0, str(ROOT))
    from oracle.flowmap_oracle import consistent_scene
    _, _, _, ext = consistent_scene(40, 8, 12, seed=5, rotation=0.05, translation=0.1)
    cam = ext[0, :, :3, 3]
    out["scene"] = (cam, cam + 0.01 * torch.randn(40, 3, generator=g, dtype=torch.float64))
    out["zero_pred"] = (_walk(g, 150), torch.zeros(150, 3, dtype=torch.float64))
    return out


def main():
    sys.path.insert(0, REF)
    os.environ["PYTHONDONTWRITEBYTECODE"] = "1"
    sys.dont_write_bytecode = True
    from scipy.spatial import procrustes
    from flowmap.misc.ate import compute_ate

    store = {}
    for name, (gt, pred) in cases().items():
        gt, pred = gt.float(), pred.float()
        store[f"{name}__gt"], store[f"{name}__pred"] = gt.numpy(), pred.numpy()
        try:
            ate, al_gt, al_pred = compute_ate(gt, pred)
        except ValueError:
            store[f"{name}__raised"] = np.array(True)
            continue
        store[f"{name}__raised"] = np.array(False)
        store[f"{name}__ate"] = ate.numpy()
        store[f"{name}__aligned_gt"], store[f"{name}__aligned_pred"] = al_gt.numpy(), al_pred.numpy()
        store[f"{name}__disparity"] = np.array(procrustes(gt.numpy(), pred.numpy())[2], dtype=np.float64)
    store["names"] = np.array(list(cases()))
    np.savez_compressed(OUT / "ate.npz", **store)
    print("wrote ate.npz")


if __name__ == "__main__":
    main()
