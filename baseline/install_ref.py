"""Stage the UNMODIFIED reference for `bench.py --impl reference` (SURVEY.md 8(c)).

The reference cannot be pip-installed offline (hydra / lightning / dacite are absent and the
`flowmap` namespace package declares no build backend), so this script copies the reference's
own Python package -- `flowmap/` as it lies, minus `third_party/` (RAFT / GMFlow / CoTracker /
COLMAP code the optimisation hot path never imports) -- from a checkout of the reference into the
git-ignored `baseline/_ref/`.  Nothing under baseline/_ref is product source or is imported by
flowmap_b200; only `bench.py --impl reference` and the `reference_cuda_eager` leg of the GPU arm
import it, and both skip it when it is absent.

    python baseline/install_ref.py /path/to/flowmap-checkout
"""
from __future__ import annotations

import shutil
import sys
from pathlib import Path

DST = Path(__file__).resolve().parent / "_ref"


def install(reference: Path, verbose: bool = True) -> bool:
    src = Path(reference) / "flowmap"
    if not src.is_dir():
        if verbose:
            print(f"{src} not found: keeping whatever is in {DST}")
        return (DST / "flowmap" / "model" / "model.py").exists()
    if DST.exists():
        shutil.rmtree(DST)
    shutil.copytree(src, DST / "flowmap",
                    ignore=shutil.ignore_patterns("third_party", "__pycache__", "*.pyc"))
    n = sum(1 for _ in (DST / "flowmap").rglob("*.py"))
    (DST / "README").write_text(
        "Unmodified copy of the reference's flowmap/ package (minus third_party/), staged by "
        "baseline/install_ref.py for the reference arm of bench.py.  Git-ignored; not product code.\n")
    if verbose:
        print(f"staged {n} reference modules under {DST}")
    return True


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    sys.exit(0 if install(Path(sys.argv[1])) else 1)
