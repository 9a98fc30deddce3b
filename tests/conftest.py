"""pytest configuration: the `gpu` marker and shared helpers.

`-m "not gpu"` runs in the build container (no GPU): oracle vs golden vectors, host logic,
C-ABI symbol checks, world_size-2 gloo tests.  `-m gpu` runs on an H100 and checks the CUDA
path (called through the C ABI) against the oracle and the golden vectors.
"""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name: str, f64: bool = False) -> dict:
    path = GOLDEN / f"{name}{'_f64' if f64 else ''}.npz"
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


def rel_l2(a, b) -> float:
    a = torch.as_tensor(a, dtype=torch.float64).flatten()
    b = torch.as_tensor(b, dtype=torch.float64).flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def max_abs(a, b) -> float:
    a = torch.as_tensor(a, dtype=torch.float64)
    b = torch.as_tensor(b, dtype=torch.float64)
    return float((a - b).abs().max())
