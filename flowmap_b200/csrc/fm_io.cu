// sm_90a kernels + C ABI for the stages either side of the optimisation hot path (SURVEY 8(f)
// rank 4): the flow-side preprocessing that builds `Flows` (consistency masks, rescaling) and the
// point-cloud part of the COLMAP export.  One-off, HBM-bound elementwise work: one thread per
// output pixel, coalesced stores, gathers through the read-only path.
#include <cuda_runtime.h>

#include "../../include/flowmap_b200.h"
#include "fm_host.h"
#include "fm_math.cuh"

namespace {

using namespace fm;
using fm_host::fail_msg;

constexpr int kIoThreads = 256;

// flow_predictor.py:60-82.  grid = (pixel blocks, B * (F - 1)).  Frames are planar (3, H, W).
// reverse = 0: colour of frame i at the pixel vs frame i+1 at pixel + flow (forward flow);
// reverse = 1: frame i+1 vs frame i (the backward flow of pair i, i.e. what the reference gets by
// flipping the video, predicting, and flipping the result back, :92-99).
__global__ void __launch_bounds__(kIoThreads)
k_consistency_mask(const float* __restrict__ videos, const float* __restrict__ flow, float* __restrict__ mask,
                   int F, int H, int W, int reverse) {
  const int N = H * W;
  const int pair = blockIdx.y, b = pair / (F - 1), i = pair - b * (F - 1);
  const float* src = videos + ((size_t)b * F + i + (reverse ? 1 : 0)) * 3 * N;
  const float* tgt = videos + ((size_t)b * F + i + (reverse ? 0 : 1)) * 3 * N;
  const float2* fl = reinterpret_cast<const float2*>(flow) + (size_t)pair * N;
  const GridDims grid = make_grid(H, W);
  for (int px = blockIdx.x * kIoThreads + threadIdx.x; px < N; px += gridDim.x * kIoThreads) {
    const int r = px / W, c = px - r * W;
    const float2 f = __ldg(fl + px);
    // grid_sample(align_corners=False): pixel position = x * W - .5, zero padding
    const float fx = (pix_coord(c, grid.Wf, grid.invW) + f.x) * (float)W - 0.5f;
    const float fy = (pix_coord(r, grid.Hf, grid.invH) + f.y) * (float)H - 0.5f;
    const float x0f = floorf(fx), y0f = floorf(fy);
    const float tx = fx - x0f, ty = fy - y0f;
    float delta = 0.f;
    // positions far outside (or NaN) have no tap inside the image
    const bool any = fx > -1.f && fx < (float)W && fy > -1.f && fy < (float)H;
    const int x0 = any ? (int)x0f : 0, y0 = any ? (int)y0f : 0;
    const bool in_x0 = any && x0 >= 0, in_x1 = any && x0 + 1 <= W - 1;
    const bool in_y0 = any && y0 >= 0, in_y1 = any && y0 + 1 <= H - 1;
    const float w00 = (in_x0 && in_y0) ? (1.f - tx) * (1.f - ty) : 0.f;
    const float w01 = (in_x1 && in_y0) ? tx * (1.f - ty) : 0.f;
    const float w10 = (in_x0 && in_y1) ? (1.f - tx) * ty : 0.f;
    const float w11 = (in_x1 && in_y1) ? tx * ty : 0.f;
    const int xa = max(x0, 0), xb = min(x0 + 1, W - 1), ya = max(y0, 0), yb = min(y0 + 1, H - 1);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float* t = tgt + (size_t)ch * N;
      const float s = w00 * __ldg(t + ya * W + xa) + w01 * __ldg(t + ya * W + xb) +
                      w10 * __ldg(t + yb * W + xa) + w11 * __ldg(t + yb * W + xb);
      delta = fmaxf(delta, fabsf(__ldg(src + (size_t)ch * N + px) - s));
    }
    const float m = 1.f - delta, m2 = m * m, m4 = m2 * m2;
    mask[(size_t)pair * N + px] = m4 * m4;
  }
}

// F.interpolate(mode="bilinear", align_corners=False), channels-last images (items, H, W, C):
// source index = (dst + .5) * (in / out) - .5, clamped below at 0 (flow_predictor.py:40-58).
struct AxisTap { int i0, i1; float t; };
__device__ __forceinline__ AxisTap axis_tap(int dst, float scale, int n_in) {
  // separate multiply / subtract (no FMA contraction): the same roundings as ATen's CPU kernel
  float s = __fsub_rn(__fmul_rn(scale, (float)dst + 0.5f), 0.5f);
  s = s < 0.f ? 0.f : s;
  AxisTap a;
  a.i0 = min((int)s, n_in - 1);
  a.i1 = min(a.i0 + 1, n_in - 1);
  a.t = s - (float)a.i0;
  return a;
}

template <int C>
__global__ void __launch_bounds__(kIoThreads)
k_resize_bilinear(const float* __restrict__ in, float* __restrict__ out, int Hi, int Wi, int Ho, int Wo) {
  const int item = blockIdx.y;
  const float sh = (float)Hi / (float)Ho, sw = (float)Wi / (float)Wo;
  const float* I = in + (size_t)item * Hi * Wi * C;
  float* O = out + (size_t)item * Ho * Wo * C;
  for (int px = blockIdx.x * kIoThreads + threadIdx.x; px < Ho * Wo; px += gridDim.x * kIoThreads) {
    const int r = px / Wo, c = px - r * Wo;
    const AxisTap y = axis_tap(r, sh, Hi), x = axis_tap(c, sw, Wi);
#pragma unroll
    for (int ch = 0; ch < C; ++ch) {
      const float v00 = __ldg(I + ((size_t)y.i0 * Wi + x.i0) * C + ch), v01 = __ldg(I + ((size_t)y.i0 * Wi + x.i1) * C + ch);
      const float v10 = __ldg(I + ((size_t)y.i1 * Wi + x.i0) * C + ch), v11 = __ldg(I + ((size_t)y.i1 * Wi + x.i1) * C + ch);
      const float top = (1.f - x.t) * v00 + x.t * v01, bot = (1.f - x.t) * v10 + x.t * v11;
      O[(size_t)px * C + ch] = (1.f - y.t) * top + y.t * bot;
    }
  }
}

// export/colmap.py:84-101: world-space point per pixel, X = R (z K^-1 [x y 1]) + t.
__global__ void __launch_bounds__(kIoThreads)
k_world_points(const float* __restrict__ depth, const float* __restrict__ k4, const float* __restrict__ ext,
               float* __restrict__ xyz, int H, int W) {
  const int N = H * W, frame = blockIdx.y;
  const float4 kk = __ldg(reinterpret_cast<const float4*>(k4) + frame);
  const float* P = ext + (size_t)frame * 16;
  float R[9], t[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    R[i * 3 + 0] = __ldg(P + i * 4 + 0); R[i * 3 + 1] = __ldg(P + i * 4 + 1); R[i * 3 + 2] = __ldg(P + i * 4 + 2);
    t[i] = __ldg(P + i * 4 + 3);
  }
  const GridDims grid = make_grid(H, W);
  const float ifx = 1.f / kk.x, ify = 1.f / kk.y;
  for (int px = blockIdx.x * kIoThreads + threadIdx.x; px < N; px += gridDim.x * kIoThreads) {
    const int r = px / W, c = px - r * W;
    const float z = __ldg(depth + (size_t)frame * N + px);
    const float X = (pix_coord(c, grid.Wf, grid.invW) - kk.z) * ifx * z, Y = (pix_coord(r, grid.Hf, grid.invH) - kk.w) * ify * z;
    float* o = xyz + ((size_t)frame * N + px) * 3;
    o[0] = R[0] * X + R[1] * Y + R[2] * z + t[0];
    o[1] = R[3] * X + R[4] * Y + R[5] * z + t[1];
    o[2] = R[6] * X + R[7] * Y + R[8] * z + t[2];
  }
}

int io_blocks(long long n) {
  long long nb = (n + kIoThreads * 4 - 1) / (kIoThreads * 4);
  return (int)(nb < 1 ? 1 : (nb > 65535 ? 65535 : nb));
}

}  // namespace

extern "C" {

int fm_consistency_mask(const float* videos, const float* flow, float* mask, int B, int F, int H, int W,
                        int reverse, void* stream) {
  if (!videos || !flow || !mask || B < 1 || F < 2 || H < 1 || W < 1 || (long long)H * W > (1ll << 30))
    return fail_msg("fm_consistency_mask: bad arguments");
  dim3 grid(io_blocks((long long)H * W), B * (F - 1));
  k_consistency_mask<<<grid, kIoThreads, 0, (cudaStream_t)stream>>>(videos, flow, mask, F, H, W, reverse ? 1 : 0);
  FM_CHECK_LAUNCH("fm_consistency_mask");
  return 0;
}

int fm_resize_bilinear(const float* in, float* out, int items, int Hin, int Win, int Hout, int Wout,
                       int channels, void* stream) {
  if (!in || !out || items < 1 || Hin < 1 || Win < 1 || Hout < 1 || Wout < 1 ||
      (long long)Hout * Wout > (1ll << 30) || items > 65535)
    return fail_msg("fm_resize_bilinear: bad arguments");
  dim3 grid(io_blocks((long long)Hout * Wout), items);
  cudaStream_t s = (cudaStream_t)stream;
  if (channels == 1) k_resize_bilinear<1><<<grid, kIoThreads, 0, s>>>(in, out, Hin, Win, Hout, Wout);
  else if (channels == 2) k_resize_bilinear<2><<<grid, kIoThreads, 0, s>>>(in, out, Hin, Win, Hout, Wout);
  else if (channels == 3) k_resize_bilinear<3><<<grid, kIoThreads, 0, s>>>(in, out, Hin, Win, Hout, Wout);
  else return fail_msg("fm_resize_bilinear: channels must be 1, 2 or 3");
  FM_CHECK_LAUNCH("fm_resize_bilinear");
  return 0;
}

int fm_world_points(const float* depth, const float* k4, const float* extrinsics, float* xyz, int F, int H,
                    int W, void* stream) {
  if (!depth || !k4 || !extrinsics || !xyz || F < 1 || F > 65535 || H < 1 || W < 1 ||
      (long long)H * W > (1ll << 30))
    return fail_msg("fm_world_points: bad arguments");
  dim3 grid(io_blocks((long long)H * W), F);
  k_world_points<<<grid, kIoThreads, 0, (cudaStream_t)stream>>>(depth, k4, extrinsics, xyz, H, W);
  FM_CHECK_LAUNCH("fm_world_points");
  return 0;
}

}  // extern "C"
