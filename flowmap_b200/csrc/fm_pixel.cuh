// Per-pixel bodies of the three pixel-parallel phases, host+device.
//
// fm_kernels.cu instantiates these with __ldg loads and red.global atomics;
// tests/host_emulation instantiates the same code with plain loads/adds on the CPU to
// check the analytic gradients against the oracle without a GPU (test-only).
#pragma once
#include <string.h>

#include "fm_procrustes.cuh"

namespace fm {

// Geometry of pair (a, b = a + 1).
struct PairGeom {
  Cam ka, kb;
  GridDims grid;
  float z0;  // conditioning shift (0, 0, z0) applied to p and q before accumulation
};

// The conditioning shift z0 of a pair: the mean of the later frame's depth over a fixed grid of
// kShiftGrid x kShiftGrid pixels, weighted by the pair's correspondence weights (unweighted if
// those sum to zero).  The moment sums cancel down to the covariance, so z0 has to be close to the
// depth of the weighted cloud: one pixel is not (the image centre of a forward-moving video is the
// far horizon, hundreds of times the foreground depth, at weight ~0).  Computed once per forward
// and stored; the solve, the backward and the sweep's candidates read the stored value.
constexpr int kShiftGrid = 32;
constexpr int kShiftSamples = kShiftGrid * kShiftGrid;

// Pixel (linear index) of sample i: cell centres of a kShiftGrid x kShiftGrid grid over the frame.
FM_HD int shift_sample(int i, int H, int W) {
  const int gy = i / kShiftGrid, gx = i - gy * kShiftGrid;
  const int r = (int)(((long long)(2 * gy + 1) * H) / (2 * kShiftGrid));
  const int c = (int)(((long long)(2 * gx + 1) * W) / (2 * kShiftGrid));
  return r * W + c;
}

// z0 from the sums over `count` samples of w * depth, w and depth, rounded to 4 significant bits.  z0
// only has to lie near the cloud's depth; a coarse value is also the same for weights that differ in
// their last bits (the fused step's sigmoid and torch's, or two runs that differ by float atomics), so
// the paths and runs round the moment sums identically.
FM_HD float shift_from_sums(double swz, double sw, double sz, int count = kShiftSamples) {
  const double z = sw > 0.0 ? swz / sw : sz / count;
  if (!isfinite(z)) return 0.0f;
  int e;
  const double m = frexp(z, &e);
  return (float)ldexp(round(m * 16.0) / 16.0, e);
}

// Later point p (frame b, pixel (r, c)) and earlier point q (frame a sampled at
// xy + backward flow), both shifted by (0, 0, z0).  projection.py:222-242.
template <typename LoadA>
FM_HD void point_pq(const PairGeom& g, float x, float y, float db, float flx, float fly,
                    LoadA load_a, float* p, float* q, Taps& t) {
  float rx, ry;
  ray_of(x, y, g.kb, rx, ry);
  p[0] = db * rx;
  p[1] = db * ry;
  p[2] = db - g.z0;
  t = bilinear_taps(x + flx, y + fly, g.grid);
  float qx, qy, qz;
  sample_surface(t, g.grid, g.ka, load_a, qx, qy, qz);
  q[0] = qx;
  q[1] = qy;
  q[2] = qz - g.z0;
}

// acc[16] += (w, w p, w q, w q p^T)   (procrustes.py:23-32 on sufficient statistics)
FM_HD void moments_add(float* acc, float w, const float* p, const float* q) {
  acc[0] += w;
  const float wp0 = w * p[0], wp1 = w * p[1], wp2 = w * p[2];
  acc[1] += wp0;
  acc[2] += wp1;
  acc[3] += wp2;
  acc[4] += w * q[0];
  acc[5] += w * q[1];
  acc[6] += w * q[2];
  for (int a = 0; a < 3; ++a) {
    acc[7 + a * 3 + 0] += q[a] * wp0;
    acc[7 + a * 3 + 1] += q[a] * wp1;
    acc[7 + a * 3 + 2] += q[a] * wp2;
  }
}

// ---------------------------------------------------------------------------------
// Phase C.  Accumulator slots per frame k:
//  0        loss numerator (already scaled by weight / mask_sum)
//  1..9     forward term of pair (k, k+1): A[l][m] = sum (s - t)_l dY_m      (dR)
//  10..12   forward term: b = sum dY                                        (dt = -R b)
//  13..21   backward term of pair (k-1, k): sum dX_l s_m                    (dR)
//  22..24   backward term: sum dX                                           (dt)
//  25..28   dK_k through the unprojection ray (fx fy cx cy)
//  29..32   dK_{k+1} through the forward-term projection
//  33..36   dK_{k-1} through the backward-term projection
// ---------------------------------------------------------------------------------
constexpr int kFlowVals = 37;

struct FlowFrame {
  Cam kk, kn, kp;  // intrinsics of frames k, k+1, k-1
  Rt tf, tb;      // [R|t] of pair (k, k+1) and of pair (k-1, k)
  bool hasF, hasB;
};

// One pixel of frame k: forward term (loss_flow.py:47-56 with projection.py:143-162) and
// backward term (loss_flow.py:59-68 with projection.py:165-184) in the pair-local form of
// SURVEY A.6.  Returns the direct (pose-detached) depth gradient.
template <bool HASF, bool HASB>
FM_HD float flow_pixel(const FlowFrame& f, float x, float y, float D, float ffx, float ffy, float mf,
                       float fbx, float fby, float mb, float g, const RobustCfg& rc, float* acc) {
  float rx, ry;
  ray_of(x, y, f.kk, rx, ry);
  const float s0 = D * rx, s1 = D * ry, s2 = D;
  float ds0 = 0.f, ds1 = 0.f, ds2 = 0.f;
  if (HASF) {  // Y = R^T (s - t), projected with K_{k+1}
    const float d0 = s0 - f.tf.t[0], d1 = s1 - f.tf.t[1], d2 = s2 - f.tf.t[2];
    const float* R = f.tf.r;
    const float Y0 = R[0] * d0 + R[3] * d1 + R[6] * d2;
    const float Y1 = R[1] * d0 + R[4] * d1 + R[7] * d2;
    const float Y2 = R[2] * d0 + R[5] * d1 + R[8] * d2;
    const Proj pr = project_point(Y0, Y1, Y2, f.kn);
    float gx, gy;
    const float l = robust_map((pr.uvx - x) - ffx, (pr.uvy - y) - ffy, rc, gx, gy);
    const float wgt = g * mf;
    acc[0] += wgt * l;
    float dY0, dY1, dY2;
    project_point_adj(pr, Y0, Y1, Y2, f.kn, wgt * gx, wgt * gy, dY0, dY1, dY2, acc[29], acc[30],
                      acc[31], acc[32]);
    acc[1] += d0 * dY0; acc[2] += d0 * dY1; acc[3] += d0 * dY2;
    acc[4] += d1 * dY0; acc[5] += d1 * dY1; acc[6] += d1 * dY2;
    acc[7] += d2 * dY0; acc[8] += d2 * dY1; acc[9] += d2 * dY2;
    acc[10] += dY0; acc[11] += dY1; acc[12] += dY2;
    ds0 += R[0] * dY0 + R[1] * dY1 + R[2] * dY2;
    ds1 += R[3] * dY0 + R[4] * dY1 + R[5] * dY2;
    ds2 += R[6] * dY0 + R[7] * dY1 + R[8] * dY2;
  }
  if (HASB) {  // X = R s + t, projected with K_{k-1}
    const float* R = f.tb.r;
    const float X0 = R[0] * s0 + R[1] * s1 + R[2] * s2 + f.tb.t[0];
    const float X1 = R[3] * s0 + R[4] * s1 + R[5] * s2 + f.tb.t[1];
    const float X2 = R[6] * s0 + R[7] * s1 + R[8] * s2 + f.tb.t[2];
    const Proj pr = project_point(X0, X1, X2, f.kp);
    float gx, gy;
    const float l = robust_map((pr.uvx - x) - fbx, (pr.uvy - y) - fby, rc, gx, gy);
    const float wgt = g * mb;
    acc[0] += wgt * l;
    float dX0, dX1, dX2;
    project_point_adj(pr, X0, X1, X2, f.kp, wgt * gx, wgt * gy, dX0, dX1, dX2, acc[33], acc[34],
                      acc[35], acc[36]);
    acc[13] += dX0 * s0; acc[14] += dX0 * s1; acc[15] += dX0 * s2;
    acc[16] += dX1 * s0; acc[17] += dX1 * s1; acc[18] += dX1 * s2;
    acc[19] += dX2 * s0; acc[20] += dX2 * s1; acc[21] += dX2 * s2;
    acc[22] += dX0; acc[23] += dX1; acc[24] += dX2;
    ds0 += R[0] * dX0 + R[3] * dX1 + R[6] * dX2;
    ds1 += R[1] * dX0 + R[4] * dX1 + R[7] * dX2;
    ds2 += R[2] * dX0 + R[5] * dX1 + R[8] * dX2;
  }
  // s = D * (rx, ry, 1), rx = (x - cx) / fx
  const float e0 = ds0 * f.kk.ifx, e1 = ds1 * f.kk.ify;
  acc[25] -= e0 * s0;
  acc[26] -= e1 * s1;
  acc[27] -= e0 * D;
  acc[28] -= e1 * D;
  return ds0 * rx + ds1 * ry + ds2;
}

// ---------------------------------------------------------------------------------
// Phase C, lean form (intrinsics are constant or one shared focal length).  Uses
//   Y = R^T (s - t) = D * m + c,  m = R^T ray, c = -R^T t      (forward term)
//   X = R s + t     = D * n + t,  n = R ray                    (backward term)
// so the direct depth gradient is dY . m (+ dX . n), and the pose gradient is accumulated
// as 6-DOF twists in the local frames (only the tangent part of dL/d[R|t] survives the
// Procrustes adjoint, SURVEY A.10): forward term  aF += Y x dY, bF += dY  (world twist =
// -R aF, -R bF), backward term  aB += (D n) x dX, bB += dX.  With a shared focal length
// (fx = f W'/..., fy likewise, principal point fixed) d/df needs ONE accumulator:
//   f * dL/df = sum (du . u)_{xy}  -  D (dY . m - (R dY)_z)  -  D (dX . n - (R^T dX)_z).
// Slots: 0 loss | 1-3 aF | 4-6 bF | 7-9 aB | 10-12 bB | 13 f * dL/df.
// ---------------------------------------------------------------------------------
constexpr int kFlowLeanVals = 14;

struct FlowFrameLean {
  Cam kk, kn, kp;
  float rtF[9], cF[3], r2F[3];  // R_F^T (row-major), -R_F^T t_F, row 2 of R_F
  float rB[9], tB[3], c2B[3];   // R_B, t_B, column 2 of R_B
};

FM_HD void fill_lean(FlowFrameLean& f, const Rt* tf, const Rt* tb) {
  if (tf) {
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) f.rtF[i * 3 + j] = tf->r[j * 3 + i];
      f.cF[i] = -(tf->r[0 * 3 + i] * tf->t[0] + tf->r[1 * 3 + i] * tf->t[1] + tf->r[2 * 3 + i] * tf->t[2]);
      f.r2F[i] = tf->r[2 * 3 + i];
    }
  }
  if (tb) {
    for (int i = 0; i < 9; ++i) f.rB[i] = tb->r[i];
    for (int i = 0; i < 3; ++i) { f.tB[i] = tb->t[i]; f.c2B[i] = tb->r[i * 3 + 2]; }
  }
}

// One reprojection term of the lean kernel, written with explicit FMAs (the compiler only
// contracts a*b+c patterns, not the sum-of-products / accumulate chains used here).
//   P = D * dir + off ; uv = K (P / (P_z + eps)) ; residual vs flow ; robust map ; adjoint.
// Outputs dP (gradient w.r.t. the camera-space point), su = fx duvx u0 + fy duvy u1 and the
// masked, scaled loss contribution.
struct LeanTerm {
  float P0, P1, P2, d0, d1, d2, su, loss, uvx, uvy;
};

// Everything after the projection quotients u = P / (P_z + eps).  ALLFIN: all three are finite
// (the common case): no nan_to_num, no per-component flags; the rare case runs its own copy of
// the tail (keeping three rarely-used flags alive through this code costs more instructions
// than the arithmetic they guard).
template <bool ALLFIN>
FM_HD void lean_term_tail(LeanTerm& t, float u0, float u1, float u2, float inv, const Cam& k, float x,
                          float y, float flx, float fly, float wgt, const RobustCfg& rc) {
  bool f0 = true, f1 = true, f2 = true;
  if (!ALLFIN) {
    u0 = nan_to_num1(u0, f0);
    u1 = nan_to_num1(u1, f1);
    u2 = nan_to_num1(u2, f2);
  }
  const float uvx = fm_fma(k.fx, u0, k.cx * u2), uvy = fm_fma(k.fy, u1, k.cy * u2);
  t.uvx = uvx;
  t.uvy = uvy;
  // robust map of the aspect-corrected residual (mapping.py:35-43)
  const float sx = ((uvx - x) - flx) * rc.ax, sy = ((uvy - y) - fly) * rc.ay;
  const float n2 = fm_fma(sx, sx, sy * sy);
  float kx, ky, val;
  if (rc.mapping == MAP_L2) {
    kx = rc.ax; ky = rc.ay; val = 0.5f * n2;
  } else {
    const float inv_n = n2 > kTinyNorm2 ? fm_rsqrt(n2) : 0.0f;
    const float n = n2 * inv_n;
    float kk = inv_n;
    val = n;
    if (rc.mapping == MAP_HUBER) {
      const bool quad = n <= rc.delta;
      kk = quad ? rc.inv_delta : inv_n;
      val = quad ? (0.5f * rc.inv_delta) * n2 : n - 0.5f * rc.delta;
    }
    kx = kk * rc.ax; ky = kk * rc.ay;
  }
  t.loss = wgt * val;
  const float duvx = (wgt * sx) * kx, duvy = (wgt * sy) * ky;
  float du0 = k.fx * duvx, du1 = k.fy * duvy, du2 = fm_fma(k.cx, duvx, k.cy * duvy);
  t.su = fm_fma(du0, u0, du1 * u1);
  if (!ALLFIN) {  // nan_to_num passes no gradient through replaced components
    if (!f0) du0 = 0.0f;
    if (!f1) du1 = 0.0f;
    if (!f2) du2 = 0.0f;
  }
  t.d0 = du0 * inv;
  t.d1 = du1 * inv;
  const float dot = fm_fma(du0, t.P0, fm_fma(du1, t.P1, du2 * t.P2));
  t.d2 = fm_fma(-dot, inv, du2) * inv;
}

FM_HD LeanTerm lean_term(float D, float dir0, float dir1, float dir2, float off0, float off1,
                         float off2, const Cam& k, float x, float y, float flx, float fly, float wgt,
                         const RobustCfg& rc) {
  LeanTerm t;
  t.P0 = fm_fma(D, dir0, off0);
  t.P1 = fm_fma(D, dir1, off1);
  t.P2 = fm_fma(D, dir2, off2);
  const float inv = fm_rcp(t.P2 + kProjEps);
  const float u0 = t.P0 * inv, u1 = t.P1 * inv, u2 = t.P2 * inv;
  // one test for the common all-finite case: a NaN or an infinity anywhere fails the comparison
  if ((fabsf(u0) + fabsf(u1)) + fabsf(u2) <= 3.0e38f) lean_term_tail<true>(t, u0, u1, u2, inv, k, x, y, flx, fly, wgt, rc);
  else lean_term_tail<false>(t, u0, u1, u2, inv, k, x, y, flx, fly, wgt, rc);
  return t;
}

template <bool HASF, bool HASB, bool FOCAL>
FM_HD float flow_pixel_lean(const FlowFrameLean& f, float x, float y, float D, float ffx, float ffy,
                            float mf, float fbx, float fby, float mb, float g, const RobustCfg& rc,
                            float* acc) {
  float rx, ry;
  ray_of(x, y, f.kk, rx, ry);
  float gD = 0.f;
  if (HASF) {
    const float m0 = fm_fma(f.rtF[0], rx, fm_fma(f.rtF[1], ry, f.rtF[2]));
    const float m1 = fm_fma(f.rtF[3], rx, fm_fma(f.rtF[4], ry, f.rtF[5]));
    const float m2 = fm_fma(f.rtF[6], rx, fm_fma(f.rtF[7], ry, f.rtF[8]));
    const LeanTerm t = lean_term(D, m0, m1, m2, f.cF[0], f.cF[1], f.cF[2], f.kn, x, y, ffx, ffy, g * mf, rc);
    acc[0] += t.loss;
    const float gd = fm_fma(t.d0, m0, fm_fma(t.d1, m1, t.d2 * m2));
    gD = gd;
    acc[1] = fm_fma(t.P1, t.d2, fm_fma(-t.P2, t.d1, acc[1]));
    acc[2] = fm_fma(t.P2, t.d0, fm_fma(-t.P0, t.d2, acc[2]));
    acc[3] = fm_fma(t.P0, t.d1, fm_fma(-t.P1, t.d0, acc[3]));
    acc[4] += t.d0; acc[5] += t.d1; acc[6] += t.d2;
    if (FOCAL) {
      const float dz = fm_fma(f.r2F[0], t.d0, fm_fma(f.r2F[1], t.d1, f.r2F[2] * t.d2));
      acc[13] += fm_fma(-D, gd - dz, t.su);
    }
  }
  if (HASB) {
    const float n0 = fm_fma(f.rB[0], rx, fm_fma(f.rB[1], ry, f.rB[2]));
    const float n1 = fm_fma(f.rB[3], rx, fm_fma(f.rB[4], ry, f.rB[5]));
    const float n2 = fm_fma(f.rB[6], rx, fm_fma(f.rB[7], ry, f.rB[8]));
    const LeanTerm t = lean_term(D, n0, n1, n2, f.tB[0], f.tB[1], f.tB[2], f.kp, x, y, fbx, fby, g * mb, rc);
    acc[0] += t.loss;
    const float gd = fm_fma(t.d0, n0, fm_fma(t.d1, n1, t.d2 * n2));
    gD += gd;
    // (X - t) x dX with X - t = D n
    const float e0 = D * n0, e1 = D * n1, e2 = D * n2;
    acc[7] = fm_fma(e1, t.d2, fm_fma(-e2, t.d1, acc[7]));
    acc[8] = fm_fma(e2, t.d0, fm_fma(-e0, t.d2, acc[8]));
    acc[9] = fm_fma(e0, t.d1, fm_fma(-e1, t.d0, acc[9]));
    acc[10] += t.d0; acc[11] += t.d1; acc[12] += t.d2;
    if (FOCAL) {
      const float dz = fm_fma(f.c2B[0], t.d0, fm_fma(f.c2B[1], t.d1, f.c2B[2] * t.d2));
      acc[13] += fm_fma(-D, gd - dz, t.su);
    }
  }
  return gD;
}

// ---------------------------------------------------------------------------------
// Two-pixel (F2, fm_math.cuh) form of lean_term / flow_pixel_lean: the two pixels are
// neighbours in a row, so they share y, the per-frame constants and every control decision
// except the per-pixel selects (finite test, Huber branch).
// ---------------------------------------------------------------------------------
struct LeanTerm2 {
  F2 P0, P1, P2, d0, d1, d2, su, loss, uvx, uvy;
};
struct Cam2 {  // two cameras side by side (the same one twice for two pixels of one frame)
  F2 fx, fy, cx, cy;
};
FM_HD Cam2 cam2(const Cam& a, const Cam& b) {
  Cam2 c;
  c.fx = f2(a.fx, b.fx); c.fy = f2(a.fy, b.fy); c.cx = f2(a.cx, b.cx); c.cy = f2(a.cy, b.cy);
  return c;
}

// Everything after the projection quotients u = P / (P_z + eps).  ALLFIN: all six quotients are
// finite (the common case): no nan_to_num, no per-component flags -- keeping six rarely-used
// predicates alive through this code costs more instructions than the arithmetic they guard, so
// the rare case gets its own copy of the tail instead.
template <bool ALLFIN>
FM_HD void lean_term2_tail(LeanTerm2& t, F2 u0, F2 u1, F2 u2, F2 inv, const Cam2& k, F2 x, F2 y, F2 flx,
                           F2 fly, F2 wgt, const RobustCfg& rc) {
  bool fx0 = true, fx1 = true, fx2 = true, fy0 = true, fy1 = true, fy2 = true;
  if (!ALLFIN) {  // nan_to_num branch (projection.py:56), per component
    u0.x = nan_to_num1(u0.x, fx0); u1.x = nan_to_num1(u1.x, fx1); u2.x = nan_to_num1(u2.x, fx2);
    u0.y = nan_to_num1(u0.y, fy0); u1.y = nan_to_num1(u1.y, fy1); u2.y = nan_to_num1(u2.y, fy2);
  }
  const F2 uvx = f2_fma(k.fx, u0, f2_mul(k.cx, u2));
  const F2 uvy = f2_fma(k.fy, u1, f2_mul(k.cy, u2));
  t.uvx = uvx;
  t.uvy = uvy;
  const F2 sx = f2_mul(f2_sub(f2_sub(uvx, x), flx), f2s(rc.ax));
  const F2 sy = f2_mul(f2_sub(f2_sub(uvy, y), fly), f2s(rc.ay));
  const F2 n2 = f2_fma(sx, sx, f2_mul(sy, sy));
  F2 kx, ky, val;
  if (rc.mapping == MAP_L2) {
    kx = f2s(rc.ax); ky = f2s(rc.ay); val = f2_mul(f2s(0.5f), n2);
  } else {
    const F2 inv_n = f2(n2.x > kTinyNorm2 ? fm_rsqrt(n2.x) : 0.0f, n2.y > kTinyNorm2 ? fm_rsqrt(n2.y) : 0.0f);
    const F2 n = f2_mul(n2, inv_n);
    F2 kk = inv_n;
    val = n;
    if (rc.mapping == MAP_HUBER) {
      const F2 vq = f2_mul(f2s(0.5f * rc.inv_delta), n2), vl = f2_sub(n, f2s(0.5f * rc.delta));
      const bool qx = n.x <= rc.delta, qy = n.y <= rc.delta;
      kk = f2(qx ? rc.inv_delta : inv_n.x, qy ? rc.inv_delta : inv_n.y);
      val = f2(qx ? vq.x : vl.x, qy ? vq.y : vl.y);
    }
    kx = f2_mul(kk, f2s(rc.ax)); ky = f2_mul(kk, f2s(rc.ay));
  }
  t.loss = f2_mul(wgt, val);
  const F2 duvx = f2_mul(f2_mul(wgt, sx), kx), duvy = f2_mul(f2_mul(wgt, sy), ky);
  F2 du0 = f2_mul(k.fx, duvx), du1 = f2_mul(k.fy, duvy);
  F2 du2 = f2_fma(k.cx, duvx, f2_mul(k.cy, duvy));
  t.su = f2_fma(du0, u0, f2_mul(du1, u1));
  if (!ALLFIN) {
    if (!fx0) du0.x = 0.0f;
    if (!fx1) du1.x = 0.0f;
    if (!fx2) du2.x = 0.0f;
    if (!fy0) du0.y = 0.0f;
    if (!fy1) du1.y = 0.0f;
    if (!fy2) du2.y = 0.0f;
  }
  t.d0 = f2_mul(du0, inv);
  t.d1 = f2_mul(du1, inv);
  const F2 dot = f2_fma(du0, t.P0, f2_fma(du1, t.P1, f2_mul(du2, t.P2)));
  t.d2 = f2_mul(f2_fma(f2_neg(dot), inv, du2), inv);
}

FM_HD LeanTerm2 lean_term2(F2 D, F2 dir0, F2 dir1, F2 dir2, F2 off0, F2 off1, F2 off2, const Cam2& k,
                           F2 x, F2 y, F2 flx, F2 fly, F2 wgt, const RobustCfg& rc) {
  LeanTerm2 t;
  t.P0 = f2_fma(D, dir0, off0);
  t.P1 = f2_fma(D, dir1, off1);
  t.P2 = f2_fma(D, dir2, off2);
  const F2 den = f2_add(t.P2, f2s(kProjEps));
  const F2 inv = f2(fm_rcp(den.x), fm_rcp(den.y));
  const F2 u0 = f2_mul(t.P0, inv), u1 = f2_mul(t.P1, inv), u2 = f2_mul(t.P2, inv);
  // one test per pixel: a NaN or an infinity anywhere makes the sum fail the comparison
  const bool okx = (fabsf(u0.x) + fabsf(u1.x)) + fabsf(u2.x) <= 3.0e38f;
  const bool oky = (fabsf(u0.y) + fabsf(u1.y)) + fabsf(u2.y) <= 3.0e38f;
  if (okx && oky) lean_term2_tail<true>(t, u0, u1, u2, inv, k, x, y, flx, fly, wgt, rc);
  else lean_term2_tail<false>(t, u0, u1, u2, inv, k, x, y, flx, fly, wgt, rc);
  return t;
}

// Two neighbouring pixels (x.x, x.y) of one row; acc holds kFlowLeanVals packed accumulators
// (the two lanes are added together when the thread is done).  Returns the two depth gradients.
template <bool HASF, bool HASB, bool FOCAL>
FM_HD F2 flow_pixel_lean2(const FlowFrameLean& f, F2 x, float y, F2 D, F2 ffx, F2 ffy, F2 mf, F2 fbx,
                          F2 fby, F2 mb, float g, const RobustCfg& rc, F2* acc) {
  const F2 rx = f2_mul(f2_sub(x, f2s(f.kk.cx)), f2s(f.kk.ifx));
  const float ry = (y - f.kk.cy) * f.kk.ify;
  F2 gD = f2s(0.f);
  if (HASF) {
    // m = R^T ray: the y / constant part is shared by the two pixels
    const F2 m0 = f2_fma(f2s(f.rtF[0]), rx, f2s(fm_fma(f.rtF[1], ry, f.rtF[2])));
    const F2 m1 = f2_fma(f2s(f.rtF[3]), rx, f2s(fm_fma(f.rtF[4], ry, f.rtF[5])));
    const F2 m2 = f2_fma(f2s(f.rtF[6]), rx, f2s(fm_fma(f.rtF[7], ry, f.rtF[8])));
    const LeanTerm2 t = lean_term2(D, m0, m1, m2, f2s(f.cF[0]), f2s(f.cF[1]), f2s(f.cF[2]),
                                   cam2(f.kn, f.kn), x, f2s(y), ffx, ffy, f2_mul(f2s(g), mf), rc);
    acc[0] = f2_add(acc[0], t.loss);
    const F2 gd = f2_fma(t.d0, m0, f2_fma(t.d1, m1, f2_mul(t.d2, m2)));
    gD = gd;
    acc[1] = f2_fma(t.P1, t.d2, f2_fma(f2_neg(t.P2), t.d1, acc[1]));
    acc[2] = f2_fma(t.P2, t.d0, f2_fma(f2_neg(t.P0), t.d2, acc[2]));
    acc[3] = f2_fma(t.P0, t.d1, f2_fma(f2_neg(t.P1), t.d0, acc[3]));
    acc[4] = f2_add(acc[4], t.d0); acc[5] = f2_add(acc[5], t.d1); acc[6] = f2_add(acc[6], t.d2);
    if (FOCAL) {
      const F2 dz = f2_fma(f2s(f.r2F[0]), t.d0, f2_fma(f2s(f.r2F[1]), t.d1, f2_mul(f2s(f.r2F[2]), t.d2)));
      acc[13] = f2_add(acc[13], f2_fma(f2_neg(D), f2_sub(gd, dz), t.su));
    }
  }
  if (HASB) {
    const F2 n0 = f2_fma(f2s(f.rB[0]), rx, f2s(fm_fma(f.rB[1], ry, f.rB[2])));
    const F2 n1 = f2_fma(f2s(f.rB[3]), rx, f2s(fm_fma(f.rB[4], ry, f.rB[5])));
    const F2 n2 = f2_fma(f2s(f.rB[6]), rx, f2s(fm_fma(f.rB[7], ry, f.rB[8])));
    const LeanTerm2 t = lean_term2(D, n0, n1, n2, f2s(f.tB[0]), f2s(f.tB[1]), f2s(f.tB[2]),
                                   cam2(f.kp, f.kp), x, f2s(y), fbx, fby, f2_mul(f2s(g), mb), rc);
    acc[0] = f2_add(acc[0], t.loss);
    const F2 gd = f2_fma(t.d0, n0, f2_fma(t.d1, n1, f2_mul(t.d2, n2)));
    gD = f2_add(gD, gd);
    const F2 e0 = f2_mul(D, n0), e1 = f2_mul(D, n1), e2 = f2_mul(D, n2);
    acc[7] = f2_fma(e1, t.d2, f2_fma(f2_neg(e2), t.d1, acc[7]));
    acc[8] = f2_fma(e2, t.d0, f2_fma(f2_neg(e0), t.d2, acc[8]));
    acc[9] = f2_fma(e0, t.d1, f2_fma(f2_neg(e1), t.d0, acc[9]));
    acc[10] = f2_add(acc[10], t.d0); acc[11] = f2_add(acc[11], t.d1); acc[12] = f2_add(acc[12], t.d2);
    if (FOCAL) {
      const F2 dz = f2_fma(f2s(f.c2B[0]), t.d0, f2_fma(f2s(f.c2B[1]), t.d1, f2_mul(f2s(f.c2B[2]), t.d2)));
      acc[13] = f2_add(acc[13], f2_fma(f2_neg(D), f2_sub(gd, dz), t.su));
    }
  }
  return gD;
}

// Lean accumulators of frame `frame` -> the standard slot layout (kFlowVals) that the pose /
// intrinsics reductions read.  rtF / rtB: [R|t] (3x4 row-major, float) of pair (frame, frame+1)
// / (frame-1, frame) or NULL; f_of_frame: the shared focal length expressed through this
// frame's fx (f = fx * W / sqrt(HW)); W_over_s = W / sqrt(HW).
template <typename T>
FM_HD void lean_to_standard(const T* lean, const float* rtF, const float* rtB, double focal,
                            double W_over_s, bool focal_mode, T* out) {
  for (int i = 0; i < kFlowVals; ++i) out[i] = (T)0;
  out[0] = lean[0];
  if (rtF) {  // world twist a = -R aF, ambient dR = 1/2 [a]x R ; slots 10-12 feed dt = -R b
    double a[3];
    for (int i = 0; i < 3; ++i)
      a[i] = -((double)rtF[i * 4 + 0] * lean[1] + (double)rtF[i * 4 + 1] * lean[2] + (double)rtF[i * 4 + 2] * lean[3]);
    for (int c = 0; c < 3; ++c) {
      const double r0 = rtF[0 * 4 + c], r1 = rtF[1 * 4 + c], r2 = rtF[2 * 4 + c];
      out[1 + 0 * 3 + c] = (T)(0.5 * (-a[2] * r1 + a[1] * r2));
      out[1 + 1 * 3 + c] = (T)(0.5 * (a[2] * r0 - a[0] * r2));
      out[1 + 2 * 3 + c] = (T)(0.5 * (-a[1] * r0 + a[0] * r1));
    }
    out[10] = lean[4]; out[11] = lean[5]; out[12] = lean[6];
  }
  if (rtB) {
    const double a[3] = {(double)lean[7], (double)lean[8], (double)lean[9]};
    for (int c = 0; c < 3; ++c) {
      const double r0 = rtB[0 * 4 + c], r1 = rtB[1 * 4 + c], r2 = rtB[2 * 4 + c];
      out[13 + 0 * 3 + c] = (T)(0.5 * (-a[2] * r1 + a[1] * r2));
      out[13 + 1 * 3 + c] = (T)(0.5 * (a[2] * r0 - a[0] * r2));
      out[13 + 2 * 3 + c] = (T)(0.5 * (-a[1] * r0 + a[0] * r1));
    }
    out[22] = lean[10]; out[23] = lean[11]; out[24] = lean[12];
  }
  // dL/df booked as an equivalent dL/dfx (fx = f * sqrt(HW) / W) of this frame
  if (focal_mode) out[25] = (T)((double)lean[13] / focal * W_over_s);
}

// ---------------------------------------------------------------------------------
// Phase D2: per-point adjoints of the Procrustes inputs.  `scatter(row, x0, v0, v1)` adds
// v0 / v1 into the earlier frame's depth gradient at columns x0 / x0 + 1 of a row; returns the aligned later-frame depth gradient and
// the weight gradient.  kacc[0..3] += dK_a (through q), kacc[4..7] += dK_b (through p); KGRAD = false
// (constant intrinsics) leaves kacc alone.
// ---------------------------------------------------------------------------------
template <bool KGRAD = true, typename LoadA, typename Scatter>
FM_HD void distribute_point(const PairGeom& g, const PairAdjoint& ad, float x, float y, float db,
                            float w, float flx, float fly, LoadA load_a, Scatter scatter,
                            float& g_db, float& g_w, float* kacc) {
  float p[3], q[3];
  Taps t;
  point_pq(g, x, y, db, flx, fly, load_a, p, q, t);
  const float dp[3] = {p[0] - ad.pbar[0], p[1] - ad.pbar[1], p[2] - ad.pbar[2]};
  const float dq[3] = {q[0] - ad.qbar[0], q[1] - ad.qbar[1], q[2] - ad.qbar[2]};
  float pb[3], qb[3];
  point_adjoint(ad, w, dp, dq, g_w, pb, qb);
  // p = db * (rx, ry, 1)
  float rx, ry;
  ray_of(x, y, g.kb, rx, ry);
  g_db = pb[0] * rx + pb[1] * ry + pb[2];
  if (KGRAD) {
    const float eb0 = pb[0] * g.kb.ifx, eb1 = pb[1] * g.kb.ify;
    kacc[4] -= eb0 * p[0];
    kacc[5] -= eb1 * p[1];
    kacc[6] -= eb0 * db;
    kacc[7] -= eb1 * db;
  }
  // q = sum_n w_n D_n (rx_n, ry_n, 1): scatter into the four taps of the earlier frame
  float rx0, ry0, rx1, ry1;
  tap_rays(t, g.grid, g.ka, rx0, ry0, rx1, ry1);
  const float b00 = qb[0] * rx0 + qb[1] * ry0 + qb[2];
  const float b01 = qb[0] * rx1 + qb[1] * ry0 + qb[2];
  const float b10 = qb[0] * rx0 + qb[1] * ry1 + qb[2];
  const float b11 = qb[0] * rx1 + qb[1] * ry1 + qb[2];
  // one call per tap row: (row y, x0, value at x0, value at x0 + 1); a clamped x1 has weight 0
  scatter(t.y0, t.x0, t.w00 * b00, t.w01 * b01);
  scatter(t.y1, t.x0, t.w10 * b10, t.w11 * b11);
  if (KGRAD) {
    const float qz_true = q[2] + g.z0;
    const float ea0 = qb[0] * g.ka.ifx, ea1 = qb[1] * g.ka.ify;
    kacc[0] -= ea0 * q[0];
    kacc[1] -= ea1 * q[1];
    kacc[2] -= ea0 * qz_true;
    kacc[3] -= ea1 * qz_true;
  }
}

// Order of magnitude of the largest tap value distribute_point scatters for a pair, from its
// constants alone (an estimate, not a bound): a tap value is a bilinear weight times
// qb . (rx, ry, 1) with qb = w (Cbar dp + ad.qb), w <= 1, |dp| of the order of the depth times a
// ray (the conditioning depth z0, the weighted cloud's mean depth, stands in for the depth), and no ray component larger than R, the
// largest over the image of either frame.
FM_HD float ray_bound(const Cam& k) {
  return fmaxf(fmaxf(fabsf(k.cx), fabsf(1.0f - k.cx)) * fabsf(k.ifx),
               fmaxf(fabsf(k.cy), fabsf(1.0f - k.cy)) * fabsf(k.ify));
}
FM_HD float tap_magnitude(const PairAdjoint& ad, const PairGeom& g) {
  float c = 0.0f, q = 0.0f;
  for (int i = 0; i < 9; ++i) c = fmaxf(c, fabsf(ad.cbar[i]));
  for (int i = 0; i < 3; ++i) q = fmaxf(q, fabsf(ad.qb[i]));
  const float R = fmaxf(1.0f, fmaxf(ray_bound(g.ka), ray_bound(g.kb)));
  return R * (3.0f * c * fabsf(g.z0) * R + q);
}

}  // namespace fm

// ---------------------------------------------------------------------------------
// Track reprojection (projection.py:255-298 + loss_tracking.py:28-61): one source sample
// (world point Xw) seen from target frame ft.  Returns validity and the robust loss; on
// request the adjoint pieces.
// ---------------------------------------------------------------------------------
namespace fm {

struct Pose {  // camera-to-world [R | t]
  float r[9];
  float t[3];
};

FM_HD bool in_unit_square(float x, float y) { return x >= 0.f && x < 1.f && y >= 0.f && y < 1.f; }

// Y = R_ft^T (Xw - t_ft); uv = project(K_ft, Y).  valid = base_valid & uv in [0,1)^2
// (projection.py:294-296: the *predicted* target position decides).
FM_HD bool track_term(const Pose& pt, const Cam& kt, const float* Xw, float gx_, float gy_,
                      bool base_valid, const RobustCfg& rc, float& loss, float* dvec, float* Yout,
                      Proj& pr, float& gux, float& guy) {
  const float d0 = Xw[0] - pt.t[0], d1 = Xw[1] - pt.t[1], d2 = Xw[2] - pt.t[2];
  const float Y0 = pt.r[0] * d0 + pt.r[3] * d1 + pt.r[6] * d2;
  const float Y1 = pt.r[1] * d0 + pt.r[4] * d1 + pt.r[7] * d2;
  const float Y2 = pt.r[2] * d0 + pt.r[5] * d1 + pt.r[8] * d2;
  pr = project_point(Y0, Y1, Y2, kt);
  const bool valid = base_valid && in_unit_square(pr.uvx, pr.uvy);
  loss = robust_map(pr.uvx - gx_, pr.uvy - gy_, rc, gux, guy);
  dvec[0] = d0; dvec[1] = d1; dvec[2] = d2;
  Yout[0] = Y0; Yout[1] = Y1; Yout[2] = Y2;
  return valid;
}

}  // namespace fm
