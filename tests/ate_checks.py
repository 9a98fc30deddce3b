"""Shared checks of trajectory-ATE results against tests/golden/ate.npz (make_golden_ate.py)."""
import itertools

import numpy as np

from conftest import load_golden

ATE_RTOL, ATE_ATOL = 1e-6, 1e-9
ALIGNED_TOL = 1e-6


def golden_cases():
    g = load_golden("ate")
    out = {}
    for name in g["names"]:
        n = str(name)
        out[n] = {k.split("__", 1)[1]: v for k, v in g.items() if k.startswith(n + "__")}
    return out


def ate64(case) -> float:
    """The float64 ATE of the reference's scipy call: sqrt(disparity / (3 F))."""
    return float(np.sqrt(case["disparity"] / case["gt"].size))


def null_directions(aligned_gt, rel: float = 1e-6):
    """Unit 3-vectors n with aligned_gt @ n = 0 (planar / collinear / two-point ground truth)."""
    _, s, vt = np.linalg.svd(np.asarray(aligned_gt, dtype=np.float64))  # full_matrices: vt is 3 x 3
    s = np.concatenate([s, np.zeros(3 - len(s))])
    return [vt[i] for i in range(3) if s[i] <= rel * s[0]]


def check_case(name, case, ate, aligned_gt=None, aligned_pred=None):
    """ATE within 1e-6 relative or 1e-9 absolute of the float64 reference, aligned_gt within 1e-6,
    aligned_pred within 1e-6 up to a mirror along each null direction of aligned_gt (only there is
    it not unique)."""
    ref = ate64(case)
    assert abs(float(ate) - ref) <= max(ATE_RTOL * ref, ATE_ATOL), (name, float(ate), ref)
    if aligned_gt is not None:
        err = np.abs(np.asarray(aligned_gt, np.float64) - case["aligned_gt"]).max()
        assert err <= ALIGNED_TOL, (name, "aligned_gt", err)
    if aligned_pred is not None:
        ours = np.asarray(aligned_pred, np.float64)
        nulls = null_directions(case["aligned_gt"])
        best = np.inf
        for signs in itertools.product((1.0, -1.0), repeat=len(nulls)):
            m = np.eye(3)
            for sgn, n in zip(signs, nulls):
                if sgn < 0:
                    m = m @ (np.eye(3) - 2.0 * np.outer(n, n))
            best = min(best, np.abs(ours @ m - case["aligned_pred"]).max())
        assert best <= ALIGNED_TOL, (name, "aligned_pred", best)
