"""In-tree build of the CUDA library for sm_90a (no torch extension machinery: the
library is a plain C-ABI .so, see include/flowmap_b200.h)."""
from __future__ import annotations

import shutil
import subprocess
from pathlib import Path

CSRC = Path(__file__).resolve().parent / "csrc"
SOURCES = ["fm_kernels.cu", "fm_io.cu"]
HEADERS = ["fm_math.cuh", "fm_procrustes.cuh", "fm_ate.cuh", "fm_pixel.cuh", "fm_host.h"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "--expt-extended-lambda", "-Xcompiler", "-fPIC", "-shared"]


def needs_build() -> bool:
    so = CSRC / "libflowmap_b200.so"
    if not so.exists():
        return True
    deps = [CSRC / s for s in SOURCES + HEADERS]
    deps.append(CSRC.parent.parent / "include" / "flowmap_b200.h")
    return any(d.stat().st_mtime > so.stat().st_mtime for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    so = CSRC / "libflowmap_b200.so"
    if not force and not needs_build():
        return so
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cmd = [nvcc, *NVCC_FLAGS, "-o", str(so), *[str(CSRC / s) for s in SOURCES]]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.check_call(cmd, cwd=str(CSRC))
    return so
