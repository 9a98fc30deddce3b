// Host build of the fixed-point window encoding (fm_math.cuh: fix_exponent / fix_pow2 /
// fix_encode / fix_decode), driven from tests/test_fixed_point_window.py.  Test-only.
#include "../../flowmap_b200/csrc/fm_math.cuh"

extern "C" {

int fixwin_exponent(float T) { return fm::fix_exponent(T); }

float fixwin_pow2(int e) { return fm::fix_pow2(e); }

// Encodes v[0..n) with scale s; ok[i] = 1 where the value encodes, 0 where it falls back.
void fixwin_encode(const float* v, int n, float s, int* hi, int* lo, int* ok) {
  for (int i = 0; i < n; ++i) {
    int h = 0, l = 0;
    ok[i] = fm::fix_encode(v[i], s, h, l) ? 1 : 0;
    hi[i] = h;
    lo[i] = l;
  }
}

float fixwin_decode(int hi, int lo, float inv_s) { return fm::fix_decode(hi, lo, inv_s); }

}  // extern "C"
