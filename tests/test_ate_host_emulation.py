"""The trajectory-ATE math that k_trajectory_ate instantiates (flowmap_b200/csrc/fm_ate.cuh), compiled
with g++ and run serially on the CPU (tests/host_emulation/ate_emu.cpp, test-only), against the
reference's compute_ate on tests/golden/ate.npz."""
import ctypes
import subprocess

import numpy as np
import pytest

from ate_checks import check_case, golden_cases
from conftest import ROOT

EMU_DIR = ROOT / "tests" / "host_emulation"
CASES = golden_cases()


@pytest.fixture(scope="module")
def emu():
    build = EMU_DIR / "_build"
    build.mkdir(exist_ok=True)
    so = build / "libate_emu.so"
    srcs = [EMU_DIR / "ate_emu.cpp"] + sorted((ROOT / "flowmap_b200" / "csrc").glob("*.cuh"))
    if not so.exists() or any(s.stat().st_mtime > so.stat().st_mtime for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", str(so),
                               str(EMU_DIR / "ate_emu.cpp")])
    return ctypes.CDLL(str(so))


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_trajectory_ate_matches_reference(emu, name):
    c = CASES[name]
    gt = np.ascontiguousarray(c["gt"], dtype=np.float32)
    pred = np.ascontiguousarray(c["pred"], dtype=np.float32)
    ate = np.zeros(1, dtype=np.float64)
    al_gt, al_pred = np.zeros_like(gt), np.zeros_like(pred)
    status = emu.emu_trajectory_ate(_p(gt), _p(pred), gt.shape[0], _p(ate), _p(al_gt), _p(al_pred))
    assert status == int(bool(c["raised"]))
    if c["raised"]:
        assert np.isnan(ate[0])
        return
    check_case(name, c, ate[0], al_gt, al_pred)
