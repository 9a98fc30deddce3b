"""The fixed-point encoding of the Procrustes backward's scatter window (fix_exponent, fix_encode,
fix_decode in flowmap_b200/csrc/fm_math.cuh), compiled from the same header with g++ and checked
on the CPU: the precision it promises, the int32 headroom of a tile's sums, and which values take
the float fall-back."""
import ctypes
import subprocess

import numpy as np
import pytest

from conftest import ROOT

EMU_DIR = ROOT / "tests" / "host_emulation"
TILE_PIXELS = 2048  # kWinTW * kWinTH: the most nonzero adds one window cell receives per tile


@pytest.fixture(scope="module")
def fx():
    build = EMU_DIR / "_build"
    build.mkdir(exist_ok=True)
    so = build / "libfixwin.so"
    srcs = [EMU_DIR / "fixwin.cpp", ROOT / "flowmap_b200" / "csrc" / "fm_math.cuh"]
    if not so.exists() or any(s.stat().st_mtime > so.stat().st_mtime for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", str(so),
                               str(EMU_DIR / "fixwin.cpp")])
    lib = ctypes.CDLL(str(so))
    lib.fixwin_exponent.restype = ctypes.c_int
    lib.fixwin_exponent.argtypes = [ctypes.c_float]
    lib.fixwin_pow2.restype = ctypes.c_float
    lib.fixwin_pow2.argtypes = [ctypes.c_int]
    lib.fixwin_decode.restype = ctypes.c_float
    lib.fixwin_decode.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_float]
    return lib


def encode(fx, v, s):
    v = np.ascontiguousarray(v, dtype=np.float32)
    hi, lo, ok = (np.zeros(v.size, np.int32) for _ in range(3))
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    fx.fixwin_encode(p(v), v.size, ctypes.c_float(s), p(hi), p(lo), p(ok))
    return hi.astype(np.int64), lo.astype(np.int64), ok.astype(bool)


@pytest.mark.parametrize("T", [1e-12, 3.7e-5, 0.5, 1.0, 1.5, 6.0e3, 2.2e9, 1e30])
def test_exponent_maps_the_estimate_below_2_24(fx, T):
    e = fx.fixwin_exponent(T)
    assert fx.fixwin_pow2(e) == 2.0 ** e and fx.fixwin_pow2(-e) == 2.0 ** -e
    assert 2.0 ** 23 <= np.float32(T) * 2.0 ** e < 2.0 ** 24


@pytest.mark.parametrize("T", [0.0, -1.0, float("nan"), float("inf")])
def test_exponent_of_a_degenerate_estimate_is_zero(fx, T):
    assert fx.fixwin_exponent(T) == 0


@pytest.mark.parametrize("T", [2.0e-3, 1.0, 7.5e4])
def test_encoding_is_exact_or_within_half_a_unit(fx, T):
    """x = v 2^e is represented as hi 2^16 + lo with |hi| <= 2^19, lo in [0, 2^16]; values with
    |x| >= 2^24 exactly, smaller ones within half a unit (plus 2^-9 for negative x above -2^16,
    which is rounded twice)."""
    e = fx.fixwin_exponent(T)
    s = 2.0 ** e
    rng = np.random.default_rng(1)
    mag = T * 2.0 ** rng.uniform(-30, 11, 200_000)  # from far below T up to the top of the range
    v = (rng.choice([-1.0, 1.0], mag.size) * mag).astype(np.float32)
    # edge cases: zero, exact multiples of 2^16 units (hi may come out one lower with lo = 2^16),
    # values next to powers of two, and next to the range limit
    units = np.array([0.0, -0.0, 65536.0, -65536.0, 3 * 65536.0, -(2.0 ** 30), 2.0 ** 24, -(2.0 ** 24),
                      2.0 ** 35 * (1 - 2.0 ** -24), -(2.0 ** 35) * (1 - 2.0 ** -24), 0.5, -0.5, 1.5, -32767.5])
    near = np.concatenate([np.nextafter(units, np.inf), np.nextafter(units, -np.inf)])
    v = np.concatenate([v, ((units / s).astype(np.float32)), (near / s).astype(np.float32)])
    hi, lo, ok = encode(fx, v, s)
    assert ok.all()
    assert (lo >= 0).all() and (lo <= 65536).all()
    assert (np.abs(hi) <= 2 ** 19).all()
    x = v.astype(np.float64) * s
    err = np.abs(hi * 65536 + lo - x)
    big = np.abs(x) >= 2.0 ** 24
    assert (err[big] == 0).all()
    assert err.max() <= 0.5 + 2.0 ** -9


@pytest.mark.parametrize("T", [2.0e-3, 1.0, 7.5e4])
def test_tile_sums_decode_to_the_float64_sum(fx, T):
    """TILE_PIXELS values added into one cell as the kernel adds them (int32 sums of hi and lo),
    decoded once: within n half units of the float64 sum plus one float32 rounding."""
    e = fx.fixwin_exponent(T)
    s, inv = 2.0 ** e, 2.0 ** -e
    rng = np.random.default_rng(2)
    for trial in range(50):
        scale = T * 2.0 ** rng.uniform(-12, 3)
        v = (scale * rng.standard_normal(TILE_PIXELS)).astype(np.float32)
        hi, lo, ok = encode(fx, v, s)
        assert ok.all()
        sh, sl = int(hi.sum()), int(lo.sum())
        assert -2 ** 31 <= sh < 2 ** 31 and 0 <= sl < 2 ** 31
        got = fx.fixwin_decode(sh, sl, inv)
        ref = float(v.astype(np.float64).sum())
        bound = TILE_PIXELS * (0.5 + 2.0 ** -9) * inv + abs(ref) * 2.0 ** -24
        assert abs(got - ref) <= bound, (trial, got, ref)


def test_a_full_tile_at_the_range_limit_does_not_overflow(fx):
    """TILE_PIXELS adds of the largest magnitude that still encodes, of either sign: the int32 sums
    stay in range and decode to the exact total."""
    s, inv = 2.0 ** 10, 2.0 ** -10
    top = np.float32(np.nextafter(np.float32(2.0 ** 35), np.float32(0)) / s)
    for sign in (1.0, -1.0):
        v = np.full(TILE_PIXELS, sign * top, np.float32)
        hi, lo, ok = encode(fx, v, s)
        assert ok.all()
        sh, sl = int(hi.sum()), int(lo.sum())
        assert -2 ** 31 <= sh < 2 ** 31 and 0 <= sl < 2 ** 31
        assert fx.fixwin_decode(sh, sl, inv) == np.float32(TILE_PIXELS * np.float64(v[0]))


def test_out_of_range_and_non_finite_values_fall_back(fx):
    s = 2.0 ** 10
    limit = 2.0 ** 35 / s
    v = np.array([limit, -limit, 3 * limit, -1e38, np.inf, -np.inf, np.nan], np.float32)
    _, _, ok = encode(fx, v, s)
    assert not ok.any()
    _, _, ok = encode(fx, np.array([np.nextafter(np.float32(limit), np.float32(0))], np.float32), s)
    assert ok.all()
