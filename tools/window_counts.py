"""Where the tap rows of the Procrustes backward's scatter window go, counted on the GPU by a
counting build of the library (-DFM_WIN_COUNT, not the default): into the fixed-point window, to the
float fall-back because a value is out of the fixed-point range, or to the float fall-back because
the row lies outside the window.

  cd flowmap_b200/csrc && mkdir -p ab && nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 \\
      --expt-extended-lambda -Xcompiler -fPIC -shared -DFM_WIN_COUNT -o ab/count.so fm_kernels.cu fm_io.cu
  python tools/window_counts.py flowmap_b200/csrc/ab/count.so
"""
import ctypes
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import ab_libs  # noqa: E402
from flowmap_b200 import _lib as libmod  # noqa: E402


def main():
    L = libmod.load_library(ROOT / sys.argv[1])
    L.fm_window_counts.restype = ctypes.c_int
    L.fm_window_counts.argtypes = [ctypes.c_void_p]
    buf = (ctypes.c_ulonglong * 3)()
    for key in [(150, 360, 640, "iid"), (150, 360, 640, "smooth"), (5, 72, 96, "leave")]:
        c = ab_libs.OpsCase(*key)
        c.fwd(L)
        c.flow(L)
        torch.cuda.synchronize()
        assert L.fm_window_counts(buf) == 0  # reset
        c.bwd(L)
        torch.cuda.synchronize()
        assert L.fm_window_counts(buf) == 0
        window, out_of_range, outside = list(buf)
        total = window + out_of_range + outside
        print(json.dumps({"case": list(key), "tap_rows": total, "window": window, "out_of_range": out_of_range,
                          "outside_window": outside, "out_of_range_share": out_of_range / total,
                          "outside_share": outside / total}), flush=True)
        del c
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
