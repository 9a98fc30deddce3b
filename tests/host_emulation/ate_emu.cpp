// TEST INFRASTRUCTURE -- never loaded by flowmap_b200.
//
// Serial host driver for the trajectory-ATE math in flowmap_b200/csrc/fm_ate.cuh (the function
// k_trajectory_ate runs with one block per trajectory), compiled with g++ by
// tests/test_ate_host_emulation.py into tests/host_emulation/_build/ (git-ignored).
#include "../../flowmap_b200/csrc/fm_ate.cuh"

using namespace fm;

namespace {
struct SerialSum {  // one caller: its partial sums are the totals
  void operator()(double*, int) {}
};
}  // namespace

extern "C" {

// gt / pred (F, 3) float32; returns the status, writes the float64 ATE and the aligned sets.
int emu_trajectory_ate(const float* gt, const float* pred, int F, double* ate, float* aligned_gt,
                       float* aligned_pred) {
  AtePoints x;
  x.gt = gt;
  x.pred = pred;
  x.gt_stride = 3;
  x.pred_stride = 3;
  x.pred_cstride = 1;
  x.F = F;
  SerialSum red;
  return trajectory_ate(x, 0, 1, red, *ate, aligned_gt, aligned_pred);
}

}  // extern "C"
