// Absolute trajectory error of a predicted camera trajectory against ground truth, with the
// semantics of scipy.spatial.procrustes, which flowmap/misc/ate.py:7-25 (compute_ate) calls:
//
//   1. centre both point sets on their mean;
//   2. divide each by its Frobenius norm (a norm of exactly 0 is scipy's ValueError "Input matrices
//      must contain >1 unique points": status 1);
//   3. SVD of mtx1^T mtx2 = U S V^T, R = U V^T (scipy.linalg.orthogonal_procrustes: the determinant
//      is NOT fixed, a mirrored trajectory aligns exactly), s = sigma1 + sigma2 + sigma3;
//   4. aligned_pred = s * mtx2 R^T;
//   5. ate = sqrt(mean((mtx1 - aligned_pred)^2)), summed term by term (the closed form 1 - s^2
//      cancels when the fit is good).
//
// Everything is float64.  The function is written for `lanes` cooperating callers (the threads of
// one CUDA block, or one host thread): each takes the points lane, lane + lanes, ... and `red`
// sums a small vector over all callers in place, so that every caller sees the same totals.
#pragma once
#include "fm_procrustes.cuh"

namespace fm {

// One trajectory of F points; coordinate c of point i is gt[i * gt_stride + c] and
// pred[i * pred_stride + c * pred_cstride] (pred_cstride 4: the translations of (F, 4, 4) poses).
struct AtePoints {
  const float* gt;
  const float* pred;
  int gt_stride, pred_stride, pred_cstride, F;
};

// Returns 0, or 1 where scipy raises (ate = NaN).  aligned_gt / aligned_pred ((F,3) float32) may
// be NULL.  Every caller returns the same status and ate; each writes the aligned rows of its points.
template <class Red>
FM_HD int trajectory_ate(const AtePoints& x, int lane, int lanes, Red& red, double& ate, float* aligned_gt,
                         float* aligned_pred) {
  const int F = x.F;
  // 1. means
  double mean[6] = {0, 0, 0, 0, 0, 0};
  for (int i = lane; i < F; i += lanes)
    for (int c = 0; c < 3; ++c) {
      mean[c] += (double)x.gt[(size_t)i * x.gt_stride + c];
      mean[3 + c] += (double)x.pred[(size_t)i * x.pred_stride + c * x.pred_cstride];
    }
  red(mean, 6);
  for (int c = 0; c < 6; ++c) mean[c] /= (double)F;
  auto centred = [&](int i, double* a, double* b) {
    for (int c = 0; c < 3; ++c) {
      a[c] = (double)x.gt[(size_t)i * x.gt_stride + c] - mean[c];
      b[c] = (double)x.pred[(size_t)i * x.pred_stride + c * x.pred_cstride] - mean[3 + c];
    }
  };
  // 2. Frobenius norms
  double nrm[2] = {0, 0};
  for (int i = lane; i < F; i += lanes) {
    double a[3], b[3];
    centred(i, a, b);
    nrm[0] += dot3(a, a);
    nrm[1] += dot3(b, b);
  }
  red(nrm, 2);
  if (nrm[0] == 0.0 || nrm[1] == 0.0) {
    ate = NAN;
    return 1;
  }
  const double n1 = sqrt(nrm[0]), n2 = sqrt(nrm[1]);
  auto scaled = [&](int i, double* a, double* b) {
    centred(i, a, b);
    for (int c = 0; c < 3; ++c) { a[c] /= n1; b[c] /= n2; }
  };
  // 3. M = mtx1^T mtx2, kept column-major for jacobi_svd3 (m[c * 3 + r] = M[r][c])
  double m[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = lane; i < F; i += lanes) {
    double a[3], b[3];
    scaled(i, a, b);
    for (int c = 0; c < 3; ++c)
      for (int r = 0; r < 3; ++r) m[c * 3 + r] += a[r] * b[c];
  }
  red(m, 9);
  double v[9];
  jacobi_svd3(m, v);  // columns of m: sigma_i u_i, columns of v: v_i
  double sig[3] = {sqrt(dot3(m, m)), sqrt(dot3(m + 3, m + 3)), sqrt(dot3(m + 6, m + 6))};
  int o[3] = {0, 1, 2};  // descending
  if (sig[o[0]] < sig[o[1]]) { int t = o[0]; o[0] = o[1]; o[1] = t; }
  if (sig[o[0]] < sig[o[2]]) { int t = o[0]; o[0] = o[2]; o[2] = t; }
  if (sig[o[1]] < sig[o[2]]) { int t = o[1]; o[1] = o[2]; o[2] = t; }
  // Left singular vectors from the data; where sigma_i vanishes (rank-deficient M: F = 2, a planar or
  // collinear set) any completion to an orthonormal basis is optimal, and none changes the ATE.
  double u[9];  // u + 3k: the left vector of column o[k]
  const double tiny = 1e-14 * sig[o[0]];
  if (sig[o[0]] > 0.0) {
    for (int r = 0; r < 3; ++r) u[r] = m[o[0] * 3 + r] / sig[o[0]];
  } else {
    u[0] = 1; u[1] = 0; u[2] = 0;
  }
  if (sig[o[1]] > tiny && sig[o[1]] > 0.0) {
    for (int r = 0; r < 3; ++r) u[3 + r] = m[o[1] * 3 + r] / sig[o[1]];
  } else {
    any_orthogonal(u, u + 3);
  }
  if (sig[o[2]] > tiny && sig[o[2]] > 0.0) {
    for (int r = 0; r < 3; ++r) u[6 + r] = m[o[2] * 3 + r] / sig[o[2]];
  } else {
    cross3(u, u + 3, u + 6);
  }
  double R[9];  // R = U V^T = sum_k u_k v_k^T (row-major)
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      R[r * 3 + c] = u[r] * v[o[0] * 3 + c] + u[3 + r] * v[o[1] * 3 + c] + u[6 + r] * v[o[2] * 3 + c];
  const double s = sig[0] + sig[1] + sig[2];
  // 4.-5. aligned prediction s * R b, squared residuals
  double d2[1] = {0};
  for (int i = lane; i < F; i += lanes) {
    double a[3], b[3];
    scaled(i, a, b);
    for (int r = 0; r < 3; ++r) {
      const double p = s * (R[r * 3 + 0] * b[0] + R[r * 3 + 1] * b[1] + R[r * 3 + 2] * b[2]);
      const double e = a[r] - p;
      d2[0] += e * e;
      if (aligned_gt) aligned_gt[(size_t)i * 3 + r] = (float)a[r];
      if (aligned_pred) aligned_pred[(size_t)i * 3 + r] = (float)p;
    }
  }
  red(d2, 1);
  ate = sqrt(d2[0] / (3.0 * F));
  return 0;
}

}  // namespace fm
