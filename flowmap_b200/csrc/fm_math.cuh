// Per-pixel geometry of the FlowMap hot path, written once as host+device inline code.
//
// The CUDA kernels in fm_kernels.cu call these from device code; tests/host_emulation
// compiles the very same header with g++ to check the analytic gradients against the
// oracle on a machine without a GPU (test infrastructure -- the shipped library has
// no CPU path).  All semantics follow SURVEY.md Appendix A; citations are to the
// reference's flowmap/...
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define FM_HD __host__ __device__ __forceinline__
#else
#define FM_HD inline
#endif

namespace fm {

struct K4 {  // normalised intrinsics [[fx 0 cx][0 fy cy][0 0 1]] (intrinsics/common.py:6-20)
  float fx, fy, cx, cy;
};

struct Rt {  // rigid 3x4 [R | t], row-major R
  float r[9];
  float t[3];
};

enum Mapping : int { MAP_HUBER = 0, MAP_L1 = 1, MAP_L2 = 2 };

// Reciprocal / reciprocal square root: ONE MUFU instruction on the device (<= 1-2 ulp), plain C on
// the host (tests/host_emulation).  The flush-to-zero forms are used on purpose: the default
// forms wrap the MUFU in a denormal range fix-up (compare, select, two scalings) that costs more
// issue slots than the operation itself.  Consequences: a denormal argument counts as 0
// (rcp -> inf, which the callers' nan_to_num path handles like the division by zero it is), and
// fm_rsqrt callers compare against kTinyNorm2 instead of 0.
constexpr float kTinyNorm2 = 1e-30f;  // squared residual norms below this are treated as exactly 0
FM_HD float fm_rcp(float v) {
#if defined(__CUDA_ARCH__)
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
  return r;
#else
  return 1.0f / v;
#endif
}
FM_HD float fm_rsqrt(float v) {
#if defined(__CUDA_ARCH__)
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
  return r;
#else
  return 1.0f / sqrtf(v);
#endif
}
FM_HD float fm_fma(float a, float b, float c) {
#if defined(__CUDA_ARCH__)
  return __fmaf_rn(a, b, c);
#else
  return fmaf(a, b, c);
#endif
}

// Pairs of float32: the lean flow kernel processes two neighbouring pixels per lane-pair with
// these.  sm_90 has no packed float32 instructions, so each operation is two scalar IEEE-rounded
// ones; the explicit _rn forms keep the compiler from contracting a mul and an add into one FMA,
// so every component is rounded exactly as the host form (tests/host_emulation) rounds it.
struct F2 {
  float x, y;
};
FM_HD F2 f2(float a, float b) { F2 r; r.x = a; r.y = b; return r; }
FM_HD F2 f2s(float a) { F2 r; r.x = a; r.y = a; return r; }
FM_HD F2 f2_fma(F2 a, F2 b, F2 c) {
#if defined(__CUDA_ARCH__)
  return f2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
#else
  return f2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
#endif
}
FM_HD F2 f2_mul(F2 a, F2 b) {
#if defined(__CUDA_ARCH__)
  return f2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
#else
  return f2(a.x * b.x, a.y * b.y);
#endif
}
FM_HD F2 f2_add(F2 a, F2 b) {
#if defined(__CUDA_ARCH__)
  return f2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
#else
  return f2(a.x + b.x, a.y + b.y);
#endif
}
FM_HD F2 f2_sub(F2 a, F2 b) { return f2_add(a, f2(-b.x, -b.y)); }
FM_HD F2 f2_neg(F2 a) { return f2(-a.x, -a.y); }

constexpr float kProjEps = 1e-5f;   // projection.py:52
constexpr float kProjInf = 1e8f;    // projection.py:53

// ---------------------------------------------------------------------------------
// Pixel grid (projection.py:93-113): x = (col + .5) / W, y = (row + .5) / H.
// ---------------------------------------------------------------------------------
FM_HD float pix_x(int c, int W) { return ((float)c + 0.5f) / (float)W; }
FM_HD float pix_y(int r, int H) { return ((float)r + 0.5f) / (float)H; }

// Same value as (i + .5) / n, correctly rounded, from a precomputed inv_n = 1 / n: one
// Newton correction of the quotient with an exact FMA remainder (three instructions
// instead of an IEEE division).
FM_HD float pix_coord(int i, float n, float inv_n) {
  const float a = (float)i + 0.5f;
  const float q = a * inv_n;
  const float r = fm_fma(-q, n, a);
  return fm_fma(r, inv_n, q);
}

// Per-frame camera constants: K and the reciprocals of the focal lengths.
struct Cam {
  float fx, fy, cx, cy, ifx, ify;
};
FM_HD Cam make_cam(const K4& k) {
  Cam c;
  c.fx = k.fx; c.fy = k.fy; c.cx = k.cx; c.cy = k.cy;
  c.ifx = 1.0f / k.fx;
  c.ify = 1.0f / k.fy;
  return c;
}

// Ray of K^-1 [x y 1]^T with z = 1 (projection.py:84-87).
FM_HD void ray_of(float x, float y, const Cam& k, float& rx, float& ry) {
  rx = (x - k.cx) * k.ifx;
  ry = (y - k.cy) * k.ify;
}

// ---------------------------------------------------------------------------------
// Bilinear tap set of grid_sample(bilinear, border, align_corners=False) at a
// normalised location (ex, ey) (projection.py:235-241; SURVEY A.3).  Follows ATen's
// unnormalise -> clip -> floor sequence.  Out-of-range taps get weight 0 and a clamped
// (in-bounds) index, so callers may load unconditionally.
// ---------------------------------------------------------------------------------
// Work decomposition of the persistent dense kernels (see block_item_range in fm_kernels.cu):
// `total` items, walked in `rounds` consecutive slices; a slice is cut into `grid` contiguous parts
// of q or q + 1 items.  The parts with the extra item are handed out round-robin ACROSS the rounds
// (round r starts where round r - 1 stopped), so that over all rounds the blocks' totals differ by
// at most two items.  Every item belongs to exactly one (round, block).
struct ItemSpan { long long i0, i1; };
FM_HD ItemSpan item_span(long long total, int rounds, int round, int block, int grid) {
  const long long len = (total + rounds - 1) / rounds;
  long long s0 = len * round, s1 = s0 + len;
  if (s0 > total) s0 = total;
  if (s1 > total) s1 = total;
  const long long g = grid;
  const long long first = ((long long)round * (len % g)) % g;  // block that takes part 0 of this slice
  const long long part = ((long long)block - first + g) % g;
  const long long q = (s1 - s0) / g, extra = (s1 - s0) % g;
  ItemSpan r;
  r.i0 = s0 + part * q + (part < extra ? part : extra);
  r.i1 = r.i0 + q + (part < extra ? 1 : 0);
  return r;
}

struct Taps {
  int x0, y0, x1, y1;      // clamped tap coordinates
  float fx0, fy0;          // x0 / y0 as floats (they fall out of the floor computation)
  float w00, w01, w10, w11;  // weights: w{row}{col}: (y0,x0) (y0,x1) (y1,x0) (y1,x1)
};

struct GridDims {
  int H, W;
  float Hf, Wf, invH, invW;
};
FM_HD GridDims make_grid(int H, int W) {
  GridDims g;
  g.H = H; g.W = W; g.Hf = (float)H; g.Wf = (float)W;
  g.invH = 1.0f / (float)H; g.invW = 1.0f / (float)W;
  return g;
}

// floor() of a value in [0, 2^22) together with its integer, on the FP32 add pipe: adding
// 1.5 * 2^23 to (v - .5) rounds to the nearest integer; a tie (v an exact integer) may pick
// v - 1 with fraction 1, which is the same point of the (continuous) bilinear interpolant.
FM_HD int floor_pos(float v, float& frac, float& fl) {
  const float magic = 12582912.0f;  // 1.5 * 2^23
  const float m = (v - 0.5f) + magic;
  fl = m - magic;
  frac = v - fl;
#if defined(__CUDA_ARCH__)
  return __float_as_int(m) - 0x4B400000;
#else
  return (int)fl;
#endif
}

// ---------------------------------------------------------------------------------
// Fixed-point accumulation in two int32 channels (the shared-memory scatter window of
// k_distribute_window: 32-bit integer adds are native shared-memory atomics on sm_90, float adds
// are compare-and-swap loops).  A value v is represented by x = v * 2^e rounded to an integer
// x = hi * 2^16 + lo, |hi| < 2^19, lo in [0, 2^16].  The exponent e is chosen per frame pair so
// that an estimate T of the pair's largest value maps to [2^23, 2^24): values with |v| >= T are
// then encoded exactly as float32 rounds them, smaller ones within half a float32 ulp at T (one
// unit 2^-e; a negative x above -2^16 is rounded twice, which adds at most 2^-9 of a unit).  Sums
// of the integers are exact and independent of the order of the adds.
// ---------------------------------------------------------------------------------
constexpr float kFixLimit = 34359738368.0f;  // 2^35: |x| below this encodes, anything else falls back

// e with T * 2^e in [2^23, 2^24), clamped so that 2^e and 2^-e are normal floats.  T <= 0 or
// non-finite gives e = 0 (then every value is 0 or takes the fall-back).
FM_HD int fix_exponent(float T) {
  if (!(T > 0.0f && T <= 3.0e38f)) return 0;
  int ex;
  frexpf(T, &ex);  // T = m 2^ex, m in [.5, 1)
  const int e = 24 - ex;
  return e < -120 ? -120 : (e > 120 ? 120 : e);
}

// 2^e as a float for |e| <= 126.
FM_HD float fix_pow2(int e) {
  const uint32_t bits = (uint32_t)(127 + e) << 23;
  float f;
  memcpy(&f, &bits, 4);
  return f;
}

// Encodes v with scale s = 2^e.  Returns false (hi = lo = 0) when |v s| >= 2^35 or v is not
// finite: the caller adds such a value as a float.  Branch-free, so that the kernel keeps hi / lo
// in registers.  Both roundings run on the FP32 add pipe as in floor_pos: hi = floor(x / 2^16) (an
// exact integer x / 2^16 may give hi one lower, with lo = 2^16), lo = rint(x - hi 2^16).
FM_HD bool fix_encode(float v, float s, int& hi, int& lo) {
  const bool ok = fabsf(v * s) < kFixLimit;
  const float x = ok ? v * s : 0.0f;
  const float magic = 12582912.0f;  // 1.5 * 2^23
  const float mh = (x * (1.0f / 65536.0f) - 0.5f) + magic;  // |x / 2^16 - .5| < 2^22
  const float fh = mh - magic;
  const float ml = (x - fh * 65536.0f) + magic;
#if defined(__CUDA_ARCH__)
  hi = __float_as_int(mh) - 0x4B400000;
  lo = __float_as_int(ml) - 0x4B400000;
#else
  hi = (int)fh;
  lo = (int)(ml - magic);
#endif
  return ok;
}

// Sum of encoded values -> float with one rounding (the product with 2^-e is exact).
FM_HD float fix_decode(int hi, int lo, float inv_s) {
  return (float)((long long)hi * 65536 + lo) * inv_s;
}

FM_HD Taps bilinear_taps(float ex, float ey, const GridDims& g) {
  // unnormalise (align_corners=False): ((2e - 1 + 1) * n - 1) / 2 = e * n - .5, then clip
  float px = fm_fma(ex, g.Wf, -0.5f);
  float py = fm_fma(ey, g.Hf, -0.5f);
  px = fminf(g.Wf - 1.0f, fmaxf(px, 0.0f));
  py = fminf(g.Hf - 1.0f, fmaxf(py, 0.0f));
  float tx, ty;
  Taps t;
  t.x0 = floor_pos(px, tx, t.fx0);
  t.y0 = floor_pos(py, ty, t.fy0);
  t.x1 = t.x0 + 1;
  t.y1 = t.y0 + 1;
  float wx1 = tx, wx0 = 1.0f - tx, wy1 = ty, wy0 = 1.0f - ty;
  if (t.x1 > g.W - 1) { t.x1 = g.W - 1; wx1 = 0.0f; }
  if (t.y1 > g.H - 1) { t.y1 = g.H - 1; wy1 = 0.0f; }
  t.w00 = wy0 * wx0;
  t.w01 = wy0 * wx1;
  t.w10 = wy1 * wx0;
  t.w11 = wy1 * wx1;
  return t;
}

// Bilinear sample of the xyz image D*ray(K) of a frame (NOT interp(D)*ray(e)): returns
// q = (qx, qy, qz).  `D` points at the frame's (H, W) depth.
// Rays through the tap centres: ((i + .5) / n - c) / f as ONE fma per axis on the float tap index
// with per-frame constants (the compiler hoists them out of the pixel loop), the second tap one
// step further.  A clamped second tap (x1 == x0) carries weight 0, so its ray never matters.  The
// rays only enter weighted sums, where one ulp is far below the float32 noise floor.
FM_HD void tap_rays(const Taps& t, const GridDims& g, const Cam& k, float& rx0, float& ry0,
                    float& rx1, float& ry1) {
  const float ax = g.invW * k.ifx, bx = (0.5f * g.invW - k.cx) * k.ifx;
  const float ay = g.invH * k.ify, by = (0.5f * g.invH - k.cy) * k.ify;
  rx0 = fm_fma(t.fx0, ax, bx);
  ry0 = fm_fma(t.fy0, ay, by);
  rx1 = rx0 + ax;
  ry1 = ry0 + ay;
}

// `load(o)` returns the frame's depth at linear offset o = row * W + col.
template <typename Load>
FM_HD void sample_surface(const Taps& t, const GridDims& g, const Cam& k, Load load, float& qx,
                          float& qy, float& qz) {
  const int r0 = t.y0 * g.W, r1 = t.y1 * g.W;
  float d00 = load(r0 + t.x0), d01 = load(r0 + t.x1);
  float d10 = load(r1 + t.x0), d11 = load(r1 + t.x1);
  float a00 = t.w00 * d00, a01 = t.w01 * d01, a10 = t.w10 * d10, a11 = t.w11 * d11;
  float rx0, rx1, ry0, ry1;
  tap_rays(t, g, k, rx0, ry0, rx1, ry1);
  qx = (a00 + a10) * rx0 + (a01 + a11) * rx1;
  qy = (a00 + a01) * ry0 + (a10 + a11) * ry1;
  qz = (a00 + a01) + (a10 + a11);
}

// ---------------------------------------------------------------------------------
// Projection u = X / (X_z + eps) on all three components, nan_to_num, then K
// (projection.py:49-58; SURVEY A.2).  Returns uv and keeps what the adjoint needs.
// ---------------------------------------------------------------------------------
struct Proj {
  float u[3];      // after nan_to_num
  float inv;       // 1 / (z + eps)
  bool all_finite; // common case: every component finite, gradient passes everywhere
  bool finite[3];  // (only meaningful when !all_finite)
  float uvx, uvy;
};

FM_HD float nan_to_num1(float v, bool& fin) {
  if (v != v) { fin = false; return 0.0f; }
  if (v > 3.0e38f) { fin = false; return kProjInf; }
  if (v < -3.0e38f) { fin = false; return -kProjInf; }
  fin = true;
  return v;
}

FM_HD Proj project_point(float X, float Y, float Z, const Cam& k) {
  Proj p;
  float den = Z + kProjEps;
  p.inv = fm_rcp(den);  // den == 0 -> inf, products below -> +-inf / nan as the division would
  p.u[0] = X * p.inv;
  p.u[1] = Y * p.inv;
  p.u[2] = Z * p.inv;
  // one test for the common case; inf/nan components (z + eps == 0, overflow) take the
  // nan_to_num branch (projection.py:56)
  p.all_finite = (fabsf(p.u[0]) <= 3.0e38f) & (fabsf(p.u[1]) <= 3.0e38f) & (fabsf(p.u[2]) <= 3.0e38f);
  if (!p.all_finite) {
    p.u[0] = nan_to_num1(p.u[0], p.finite[0]);
    p.u[1] = nan_to_num1(p.u[1], p.finite[1]);
    p.u[2] = nan_to_num1(p.u[2], p.finite[2]);
  }
  p.uvx = k.fx * p.u[0] + k.cx * p.u[2];
  p.uvy = k.fy * p.u[1] + k.cy * p.u[2];
  return p;
}

// Adjoint of project_point: given d(uv), returns d(X, Y, Z) and accumulates dK.
FM_HD void project_point_adj(const Proj& p, float X, float Y, float Z, const Cam& k, float duvx,
                             float duvy, float& dX, float& dY, float& dZ, float& dfx, float& dfy,
                             float& dcx, float& dcy) {
  dfx += duvx * p.u[0];
  dfy += duvy * p.u[1];
  dcx += duvx * p.u[2];
  dcy += duvy * p.u[2];
  float du0 = k.fx * duvx;
  float du1 = k.fy * duvy;
  float du2 = k.cx * duvx + k.cy * duvy;
  if (!p.all_finite) {
    if (!p.finite[0]) du0 = 0.0f;
    if (!p.finite[1]) du1 = 0.0f;
    if (!p.finite[2]) du2 = 0.0f;
  }
  dX = du0 * p.inv;
  dY = du1 * p.inv;
  // d/dZ of (X, Y, Z) / (Z + eps):  (du2 - du . u) / (Z + eps) on the finite components
  dZ = (du2 - (du0 * X + du1 * Y + du2 * Z) * p.inv) * p.inv;
}

// ---------------------------------------------------------------------------------
// Robust mapping of the aspect-corrected residual (mapping.py:9-43, mapping_huber.py:19-34,
// mapping_l1.py:16-20, mapping_l2.py:16-21).  Returns the loss value and writes
// d(loss)/d(r) for the *uncorrected* residual components (aspect folded in).
// ax = W / sqrt(HW), ay = H / sqrt(HW).
// ---------------------------------------------------------------------------------
struct RobustCfg {
  int mapping;
  float delta, inv_delta, ax, ay;
};
FM_HD RobustCfg make_robust(int mapping, float delta, int H, int W) {
  RobustCfg c;
  const float sc = sqrtf((float)H * (float)W);
  c.mapping = mapping;
  c.delta = delta;
  c.inv_delta = delta > 0.0f ? 1.0f / delta : 0.0f;
  c.ax = (float)W / sc;
  c.ay = (float)H / sc;
  return c;
}

FM_HD float robust_map(float rx, float ry, const RobustCfg& c, float& gx, float& gy) {
  const float sx = rx * c.ax, sy = ry * c.ay;
  const float n2 = sx * sx + sy * sy;
  if (c.mapping == MAP_L2) {
    gx = sx * c.ax;
    gy = sy * c.ay;
    return 0.5f * n2;
  }
  // norm has subgradient 0 at the origin; rsqrt(0) = inf is masked out
  const float inv_n = n2 > kTinyNorm2 ? fm_rsqrt(n2) : 0.0f;
  const float n = n2 * inv_n;
  float k = inv_n, val = n;                       // l1: n ; d/ds = s / n
  if (c.mapping == MAP_HUBER) {                   // huber_loss(n, 0, delta) / delta
    const bool quad = n <= c.delta;
    k = quad ? c.inv_delta : inv_n;
    val = quad ? 0.5f * n2 * c.inv_delta : n - 0.5f * c.delta;
  }
  gx = sx * k * c.ax;
  gy = sy * k * c.ay;
  return val;
}

}  // namespace fm
