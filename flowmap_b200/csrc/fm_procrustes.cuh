// Weighted-Procrustes solve and its adjoint on per-pair moment sums, in float64.
//
// Restates flowmap/model/procrustes.py:7-51 (align_rigid) on sufficient statistics:
// the CUDA moment kernel accumulates sum(w), sum(w p), sum(w q), sum(w q p^T) over the
// selected points (shifted by a per-pair constant for conditioning), this file turns
// them into [R | t] and, for the backward pass, turns dL/d[R | t] into the per-pair
// constants from which every per-point adjoint is a closed form (SURVEY A.7).
#pragma once
#include "fm_math.cuh"

namespace fm {

constexpr int kNumMoments = 16;  // sw, mp[3], mq[3], M[9] (M[a*3+b] = sum w q_a p_b)

// Saved per-pair state of the forward solve (float64), consumed by the adjoint.
struct PairState {
  double sw;        // sum of weights
  double inv;       // 1 / (sw + 1e-8)
  double pbar[3];   // centroid of shifted p (includes the (1-kappa) shift term)
  double qbar[3];
  double mp[3];     // raw shifted first moments
  double mq[3];
  double U[9];      // proper (det +1) left basis, columns u1 u2 u1xu2 (row-major)
  double V[9];      // proper right basis, columns v1 v2 v1xv2 (row-major)
  double sig[3];    // sigma1, sigma2, signed sigma3 = u3^T C v3
  double R[9];
  double shift[3];  // c0, the constant subtracted from p and q before accumulation
};

// Per-pair constants for the distribution kernel (float32 is enough: they multiply
// per-point quantities that are themselves float32).
struct PairAdjoint {
  float cbar[9];   // dL/dC
  float pb[3];     // dL/dpbar_total / (sw + eps)
  float qb[3];     // dL/dqbar_total / (sw + eps)
  float pbar[3];   // shifted centroids (so the kernel forms p' - pbar, q' - qbar)
  float qbar[3];
  float shift[3];
  float wconst;    // constant added to every point's weight adjoint (aggregated sweeps only)
};

FM_HD void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}
FM_HD double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// Any unit vector orthogonal to a (|a| = 1).
FM_HD void any_orthogonal(const double* a, double* o) {
  double ax = fabs(a[0]), ay = fabs(a[1]), az = fabs(a[2]);
  double e[3] = {0, 0, 0};
  if (ax <= ay && ax <= az) e[0] = 1; else if (ay <= az) e[1] = 1; else e[2] = 1;
  cross3(a, e, o);
  double n = sqrt(dot3(o, o));
  o[0] /= n; o[1] /= n; o[2] /= n;
}

// One-sided (Hestenes) Jacobi SVD of a 3x3, column-major working copies.  On return the
// columns of `a` are sigma_i u_i and the columns of `v` the right singular vectors,
// unsorted.  a[c][r] layout: a[c*3 + r].
FM_HD void jacobi_svd3(double* a, double* v) {
  for (int i = 0; i < 9; ++i) v[i] = (i % 4 == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 30; ++sweep) {
    bool rotated = false;
    for (int pi = 0; pi < 3; ++pi) {
      int p = pi == 2 ? 1 : 0, q = pi == 0 ? 1 : 2;  // (0,1) (0,2) (1,2)
      double* ap = a + 3 * p; double* aq = a + 3 * q;
      double alpha = dot3(ap, ap), beta = dot3(aq, aq), gamma = dot3(ap, aq);
      if (gamma == 0.0 || fabs(gamma) <= 1e-17 * sqrt(alpha * beta)) continue;
      rotated = true;
      double zeta = (beta - alpha) / (2.0 * gamma);
      double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
      double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
      double* vp = v + 3 * p; double* vq = v + 3 * q;
      for (int r = 0; r < 3; ++r) {
        double x = ap[r], y = aq[r];
        ap[r] = c * x - s * y; aq[r] = s * x + c * y;
        x = vp[r]; y = vq[r];
        vp[r] = c * x - s * y; vq[r] = s * x + c * y;
      }
    }
    if (!rotated) break;
  }
}

// Solve one pair.  `m` holds the 16 shifted moment sums, `shift` the constant c0.
// Writes the float32 [R | t] (3x4 row-major) and the saved state.
FM_HD void procrustes_solve(const double* m, const double* shift, float* rt_out, PairState& st) {
  st.sw = m[0];
  st.inv = 1.0 / (st.sw + 1e-8);               // procrustes.py:23
  const double kappa = st.sw * st.inv;
  double C[9];
  for (int i = 0; i < 3; ++i) {
    st.mp[i] = m[1 + i];
    st.mq[i] = m[4 + i];
    st.shift[i] = shift[i];
    // centroid of the true points minus the shift: inv*m' - (1-kappa) c0
    st.pbar[i] = st.inv * st.mp[i] - (1.0 - kappa) * shift[i];
    st.qbar[i] = st.inv * st.mq[i] - (1.0 - kappa) * shift[i];
  }
  // C = sum w (q - qbar)(p - pbar)^T on the raw weights (procrustes.py:28-32).
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b)
      C[a * 3 + b] = m[7 + a * 3 + b] - st.qbar[a] * st.mp[b] - st.mq[a] * st.pbar[b] +
                     st.sw * st.qbar[a] * st.pbar[b];

  // SVD (procrustes.py:35).  Work column-major.
  double a[9], v[9];
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) a[c * 3 + r] = C[r * 3 + c];
  jacobi_svd3(a, v);
  double n[3] = {sqrt(dot3(a, a)), sqrt(dot3(a + 3, a + 3)), sqrt(dot3(a + 6, a + 6))};
  int i0 = 0, i1 = 1, i2 = 2;  // sort descending
  if (n[i0] < n[i1]) { int t = i0; i0 = i1; i1 = t; }
  if (n[i0] < n[i2]) { int t = i0; i0 = i2; i2 = t; }
  if (n[i1] < n[i2]) { int t = i1; i1 = i2; i2 = t; }
  double u1[3], u2[3], u3[3], v1[3], v2[3], v3[3];
  for (int r = 0; r < 3; ++r) { v1[r] = v[i0 * 3 + r]; v2[r] = v[i1 * 3 + r]; }
  if (n[i0] > 0.0) {
    for (int r = 0; r < 3; ++r) u1[r] = a[i0 * 3 + r] / n[i0];
  } else {  // C == 0: any rotation is optimal; take the identity bases
    u1[0] = 1; u1[1] = 0; u1[2] = 0; v1[0] = 1; v1[1] = 0; v1[2] = 0;
    v2[0] = 0; v2[1] = 1; v2[2] = 0;
  }
  bool rank1 = !(n[i1] > 1e-300 && n[i1] > 1e-14 * n[i0]);
  if (!rank1) {
    double d = 0;
    for (int r = 0; r < 3; ++r) { u2[r] = a[i1 * 3 + r] / n[i1]; }
    d = dot3(u2, u1);
    for (int r = 0; r < 3; ++r) u2[r] -= d * u1[r];
    double nn = sqrt(dot3(u2, u2));
    for (int r = 0; r < 3; ++r) u2[r] /= nn;
  } else {
    if (n[i0] > 0.0) any_orthogonal(u1, u2); else { u2[0] = 0; u2[1] = 1; u2[2] = 0; }
  }
  cross3(u1, u2, u3);
  cross3(v1, v2, v3);
  for (int r = 0; r < 3; ++r) {
    st.U[r * 3 + 0] = u1[r]; st.U[r * 3 + 1] = u2[r]; st.U[r * 3 + 2] = u3[r];
    st.V[r * 3 + 0] = v1[r]; st.V[r * 3 + 1] = v2[r]; st.V[r * 3 + 2] = v3[r];
  }
  // signed third singular value: u3^T C v3 (= d * sigma3 of procrustes.py:38)
  double cv[3] = {C[0] * v3[0] + C[1] * v3[1] + C[2] * v3[2],
                  C[3] * v3[0] + C[4] * v3[1] + C[5] * v3[2],
                  C[6] * v3[0] + C[7] * v3[1] + C[8] * v3[2]};
  st.sig[0] = n[i0];
  st.sig[1] = rank1 ? 0.0 : n[i1];
  st.sig[2] = dot3(u3, cv);
  // R = U diag(1, 1, d) Vt with d fixing the handedness == U' V'^T for proper U', V'.
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      st.R[r * 3 + c] = u1[r] * v1[c] + u2[r] * v2[c] + u3[r] * v3[c];
  // t = qbar - R pbar on the TRUE centroids (procrustes.py:42): pbar_true = pbar' + c0.
  for (int r = 0; r < 3; ++r) {
    double t = st.qbar[r] + shift[r];
    for (int c = 0; c < 3; ++c) t -= st.R[r * 3 + c] * (st.pbar[c] + shift[c]);
    rt_out[r * 4 + 0] = (float)st.R[r * 3 + 0];
    rt_out[r * 4 + 1] = (float)st.R[r * 3 + 1];
    rt_out[r * 4 + 2] = (float)st.R[r * 3 + 2];
    rt_out[r * 4 + 3] = (float)t;
  }
}

// Adjoint of the solve.  g_rt is dL/d[R | t] (3x4 row-major, float64).
FM_HD void procrustes_adjoint(const PairState& st, const double* g_rt, PairAdjoint& out) {
  double gt[3] = {g_rt[3], g_rt[7], g_rt[11]};
  double G[9];
  double ptrue[3] = {st.pbar[0] + st.shift[0], st.pbar[1] + st.shift[1], st.pbar[2] + st.shift[2]};
  // t = qbar - R pbar  =>  dR += -gt pbar^T, dqbar = gt, dpbar = -R^T gt
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) G[r * 3 + c] = g_rt[r * 4 + c] - gt[r] * ptrue[c];
  double qbar_bar[3] = {gt[0], gt[1], gt[2]};
  double pbar_bar[3];
  for (int c = 0; c < 3; ++c)
    pbar_bar[c] = -(st.R[0 * 3 + c] * gt[0] + st.R[1 * 3 + c] * gt[1] + st.R[2 * 3 + c] * gt[2]);
  // Q = U^T G V ; Z_ij = Q_ij / (s_i + s_j) ; Cbar = U (Z - Z^T) V^T   (SURVEY A.7)
  double UG[9], Q[9];
  for (int i = 0; i < 3; ++i)
    for (int c = 0; c < 3; ++c)
      UG[i * 3 + c] = st.U[0 * 3 + i] * G[0 * 3 + c] + st.U[1 * 3 + i] * G[1 * 3 + c] +
                      st.U[2 * 3 + i] * G[2 * 3 + c];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      Q[i * 3 + j] = UG[i * 3 + 0] * st.V[0 * 3 + j] + UG[i * 3 + 1] * st.V[1 * 3 + j] +
                     UG[i * 3 + 2] * st.V[2 * 3 + j];
  double A[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      if (i == j) { A[i * 3 + j] = 0.0; continue; }
      double den = st.sig[i] + st.sig[j];
      A[i * 3 + j] = (Q[i * 3 + j] - Q[j * 3 + i]) / den;
    }
  double UA[9], Cb[9];
  for (int r = 0; r < 3; ++r)
    for (int j = 0; j < 3; ++j)
      UA[r * 3 + j] = st.U[r * 3 + 0] * A[0 * 3 + j] + st.U[r * 3 + 1] * A[1 * 3 + j] +
                      st.U[r * 3 + 2] * A[2 * 3 + j];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      Cb[r * 3 + c] = UA[r * 3 + 0] * st.V[c * 3 + 0] + UA[r * 3 + 1] * st.V[c * 3 + 1] +
                      UA[r * 3 + 2] * st.V[c * 3 + 2];
  // Centroid terms of C: qbar_bar += -Cbar sum w (p - pbar), pbar_bar += -Cbar^T sum w (q - qbar)
  double sp[3], sq[3];
  for (int i = 0; i < 3; ++i) {
    sp[i] = st.mp[i] - st.sw * st.pbar[i];
    sq[i] = st.mq[i] - st.sw * st.qbar[i];
  }
  for (int r = 0; r < 3; ++r) {
    qbar_bar[r] -= Cb[r * 3 + 0] * sp[0] + Cb[r * 3 + 1] * sp[1] + Cb[r * 3 + 2] * sp[2];
    pbar_bar[r] -= Cb[0 * 3 + r] * sq[0] + Cb[1 * 3 + r] * sq[1] + Cb[2 * 3 + r] * sq[2];
  }
  for (int i = 0; i < 9; ++i) out.cbar[i] = (float)Cb[i];
  for (int i = 0; i < 3; ++i) {
    out.pb[i] = (float)(pbar_bar[i] * st.inv);
    out.qb[i] = (float)(qbar_bar[i] * st.inv);
    out.pbar[i] = (float)st.pbar[i];
    out.qbar[i] = (float)st.qbar[i];
    out.shift[i] = (float)st.shift[i];
  }
  out.wconst = 0.0f;
}

// Per-point adjoints given the pair constants: dp' = p' - pbar', dq' = q' - qbar'.
FM_HD void point_adjoint(const PairAdjoint& a, float w, const float* dp, const float* dq, float& wbar,
                         float* pbar, float* qbar) {
  // Cbar dp and Cbar^T dq
  float cp[3], cq[3];
  for (int r = 0; r < 3; ++r) {
    cp[r] = a.cbar[r * 3 + 0] * dp[0] + a.cbar[r * 3 + 1] * dp[1] + a.cbar[r * 3 + 2] * dp[2];
    cq[r] = a.cbar[0 * 3 + r] * dq[0] + a.cbar[1 * 3 + r] * dq[1] + a.cbar[2 * 3 + r] * dq[2];
  }
  wbar = dq[0] * cp[0] + dq[1] * cp[1] + dq[2] * cp[2] + a.pb[0] * dp[0] + a.pb[1] * dp[1] +
         a.pb[2] * dp[2] + a.qb[0] * dq[0] + a.qb[1] * dq[1] + a.qb[2] * dq[2] + a.wconst;
  for (int r = 0; r < 3; ++r) {
    pbar[r] = w * (cq[r] + a.pb[r]);
    qbar[r] = w * (cp[r] + a.qb[r]);
  }
}

}  // namespace fm
