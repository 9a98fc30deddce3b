// sm_90a kernels + C ABI of the FlowMap optimisation hot path (see include/flowmap_b200.h).
//
// Roofline: everything here is pointwise + reduction work over (frame, H, W) tensors --
// HBM-bound, no tensor cores.  Per frame pair the algorithmic traffic is 32 B per
// pair-pixel + 8 B per frame-pixel (SURVEY 8(d)).
//
// Version-1 structure (one launch per phase over all pairs):
//   k_pair_shift   phase A0 per-pair conditioning shift: weighted mean depth of 32 x 32 samples
//   k_moments      phase A  weighted moment sums per pair (bilinear gather of the earlier
//                           frame at xy + backward flow), fp32 per thread -> fp64 block
//                           reduction -> fp64 atomics                (projection.py:213-249)
//   k_solve        phase B  16 moments -> C -> Jacobi SVD -> [R|t], saved state
//                                                                    (procrustes.py:7-51)
//   k_flow         phase C  per frame: forward term of pair k and backward term of pair
//                           k-1 share the unprojected point; loss, direct depth gradient
//                           (plain store), pose / intrinsics partial sums
//                                                  (loss_flow.py:31-70, projection.py:116-184)
//   k_adjoint      phase D1 pose gradient -> per-pair adjoint constants (SURVEY A.7)
//   k_distribute   phase D2 per-point adjoints: aligned add into the later frame,
//                           bilinear scatter into the earlier frame, weight gradient.  All
//                           pixels, W % 4 == 0: k_distribute_window, 2-D tiles whose scatter
//                           is accumulated in a shared-memory window of the earlier frame and
//                           flushed with coalesced 16-byte REDs; other widths:
//                           k_distribute_dense, one RED per tap row
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>

#include "../../include/flowmap_b200.h"
#include "fm_ate.cuh"
#include "fm_host.h"
#include "fm_pixel.cuh"

namespace fm_host {
namespace {
thread_local char g_err[512] = "";
unsigned long long g_launches = 0;  // kernels launched by this library (bench evidence only)
}  // namespace
int fail(const char* what, cudaError_t e) {
  snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
  return 1;
}
int fail_msg(const char* what) {
  snprintf(g_err, sizeof(g_err), "%s", what);
  return 2;
}
void count_launch() { __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED); }
const char* last_error() { return g_err; }
unsigned long long launches() { return __atomic_load_n(&g_launches, __ATOMIC_RELAXED); }
}  // namespace fm_host

namespace {

using namespace fm;

using fm_host::fail;
using fm_host::fail_msg;

constexpr int kThreads = 256;
constexpr int kFlowAcc = 40;  // per-frame accumulator slots of k_flow

// ---------------------------------------------------------------- workspace layout
struct Workspace {
  double* moments;   // [BP][16]
  double* flowacc;   // [BF][kFlowAcc]
  double* k4acc;     // [BF][4]
  double* loss;      // [4]
  PairState* state;  // [BP]
  PairAdjoint* adj;  // [BP]
  float* zshift;     // [BP] conditioning shift of the moment pass (k_pair_shift)
  float* pshift;     // [BP][3] conditioning shift of explicit point sets (k_points_shift)
  size_t bytes;
};

__host__ __device__ inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

Workspace carve(void* base, int B, int F) {
  const size_t BP = (size_t)B * (F - 1), BF = (size_t)B * F;
  char* p = (char*)base;
  size_t off = 0;
  Workspace w;
  w.moments = (double*)(p + off); off = align_up(off + BP * kNumMoments * sizeof(double), 256);
  w.flowacc = (double*)(p + off); off = align_up(off + BF * kFlowAcc * sizeof(double), 256);
  w.k4acc = (double*)(p + off); off = align_up(off + BF * 4 * sizeof(double), 256);
  w.loss = (double*)(p + off); off = align_up(off + 4 * sizeof(double), 256);
  w.state = (PairState*)(p + off); off = align_up(off + BP * sizeof(PairState), 256);
  w.adj = (PairAdjoint*)(p + off); off = align_up(off + BP * sizeof(PairAdjoint), 256);
  w.zshift = (float*)(p + off); off = align_up(off + BP * sizeof(float), 256);
  w.pshift = (float*)(p + off); off = align_up(off + BP * 3 * sizeof(float), 256);
  w.bytes = off;
  return w;
}

// ---------------------------------------------------------------- small device helpers
__device__ __forceinline__ K4 load_k4(const float* k4, int frame) {
  const float4 v = __ldg(reinterpret_cast<const float4*>(k4) + frame);
  K4 k; k.fx = v.x; k.fy = v.y; k.cx = v.z; k.cy = v.w;
  return k;
}

__device__ __forceinline__ Rt load_rt(const float* rt, int pair) {
  Rt t;
  const float* s = rt + (size_t)pair * 12;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    t.r[r * 3 + 0] = __ldg(s + r * 4 + 0);
    t.r[r * 3 + 1] = __ldg(s + r * 4 + 1);
    t.r[r * 3 + 2] = __ldg(s + r * 4 + 2);
    t.t[r] = __ldg(s + r * 4 + 3);
  }
  return t;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum of NV per-thread float values, atomically added (fp64) to dst[0..NV).
// Per-thread partials cover at most a few dozen pixels, so the float32 warp tree adds no
// visible error; the cross-warp and cross-block sums run in float64.
// smem must hold NV * (kThreads / 32) doubles.
template <int NV, int NT = kThreads>
__device__ __forceinline__ void block_accumulate(const float* vals, double* dst, double* smem) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = NT / 32;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float s = warp_sum_f(vals[i]);
    if (lane == 0) smem[i * NW + warp] = (double)s;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NV; i += NT) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < NW; ++w) s += smem[i * NW + w];
    if (s != 0.0) atomicAdd(dst + i, s);
  }
  __syncthreads();
}

template <int NV>
__device__ __forceinline__ void block_accumulate_d(const double* vals, double* dst, double* smem) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = kThreads / 32;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    double s = warp_sum(vals[i]);
    if (lane == 0) smem[i * NW + warp] = s;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NV; i += kThreads) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < NW; ++w) s += smem[i * NW + w];
    if (s != 0.0) atomicAdd(dst + i, s);
  }
  __syncthreads();
}

// Fire-and-forget float add (RED.E.ADD.F32); no return value, no warp aggregation code.
__device__ __forceinline__ void red_add(float* addr, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}

__device__ __forceinline__ void red_add4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d)
               : "memory");
}

// Adds v0 / v1 at columns x0 / x0 + 1 of a row.  With 16-byte aligned rows (ALIGNED) the pair
// goes out as ONE vector RED on the aligned group of four floats that contains x0 unless it
// straddles two groups: one RED instruction instead of two for scattered taps (tools/red_bench.cu
// times the two forms).
template <bool ALIGNED>
__device__ __forceinline__ void red_pair(float* row, int x0, int W, float v0, float v1) {
  const int k = x0 & 3;
  if (ALIGNED && k != 3) {
    red_add4(row + (x0 - k), k == 0 ? v0 : 0.f, k == 0 ? v1 : (k == 1 ? v0 : 0.f),
             k == 1 ? v1 : (k == 2 ? v0 : 0.f), k == 2 ? v1 : 0.f);
  } else {
    red_add(row + x0, v0);
    if (x0 + 1 < W) red_add(row + x0 + 1, v1);
  }
}

// Correspondence weight from its stored form: the weight itself (sens == 0) or the logit of
// BackboneExplicitDepth (backbone_explicit_depth.py:40): w = sigmoid(sens * logit).
__device__ __forceinline__ float weight_of(float stored, float sens) {
  if (sens == 0.f) return stored;
  // exp(-sens * stored) as ONE MUFU.EX2 (flush-to-zero form: no denormal range fix-up around it;
  // an underflowing exponential gives w = 1, as it should)
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * sens * stored));
  return fm_rcp(1.0f + e);
}

// Keeps a frame's base pointer as ONE 64-bit value: without this the compiler re-associates
// depth + (frame offset + tap offset) and spends a 64-bit add + two LEAs on every gathered tap
// instead of one IMAD.WIDE on the finished pointer.
__device__ __forceinline__ const float* opaque_ptr(const float* p) {
  asm volatile("" : "+l"(p));
  return p;
}

// Same for a 32-bit value (a shared-space base address the compiler would otherwise re-derive from
// %cluster_ctarank at every use).
__device__ __forceinline__ unsigned opaque_u32(unsigned v) {
  asm volatile("" : "+r"(v));
  return v;
}

// Software prefetch into L2 (no register, no scoreboard): streaming operands are requested a couple
// of chunks ahead so that the demand loads find them on chip.
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// Load the 4 (or 1) values a thread owns.
template <int VEC>
__device__ __forceinline__ void load_vec(const float* p, float* out) {
  if (VEC == 4) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(p));
    out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w;
  } else {
    out[0] = __ldg(p);
  }
}
template <int VEC>
__device__ __forceinline__ void load_vec2(const float* p, float* out) {  // 2 * VEC floats
  if (VEC == 4) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p));
    const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    out[0] = a.x; out[1] = a.y; out[2] = a.z; out[3] = a.w;
    out[4] = b.x; out[5] = b.y; out[6] = b.z; out[7] = b.w;
  } else {
    const float2 a = __ldg(reinterpret_cast<const float2*>(p));
    out[0] = a.x; out[1] = a.y;
  }
}

// Work decomposition of the dense (all-pixel) kernels: an item is one chunk of kThreads * VEC
// consecutive pixels of one unit (a frame pair, or a frame); ONE 1-D grid of SMs x CTAs-per-SM blocks,
// each taking a contiguous range of items.  No partial last wave (the 2-D grids of round 1 ended in a
// 9 %..70 % full one), and a block's per-unit constants change at most a couple of times.
struct ItemRange { int i0, i1; };
__device__ __forceinline__ ItemRange block_item_range(long long total) {
  const ItemSpan sp = item_span(total, 1, 0, (int)blockIdx.x, (int)gridDim.x);
  ItemRange r;
  r.i0 = (int)sp.i0;
  r.i1 = (int)sp.i1;
  return r;
}
// The same decomposition applied to each of `rounds` consecutive slices of the item list (all blocks
// share slice 0, then slice 1, ...).  The gathers / REDs of the Procrustes kernels touch a band of rows
// around a block's position; with one round the resident blocks sit in as many different places as there
// are blocks, and at 720p those bands (grid x band x row bytes x 2 arrays) no longer fit in L2.
// With more rounds the blocks advance together through
// a few frame pairs and share their bands.  Blocks are rotated between rounds so that the odd chunk of
// an uneven split does not always land on the same block.
__device__ __forceinline__ ItemRange block_item_range(long long total, int rounds, int round) {
  const ItemSpan sp = item_span(total, rounds, round, (int)blockIdx.x, (int)gridDim.x);
  ItemRange r;
  r.i0 = (int)sp.i0;
  r.i1 = (int)sp.i1;
  return r;
}

// Thread -> pixel mapping inside a chunk of kThreads * 4 pixels of the dense Procrustes kernels; a
// thread always owns 4 consecutive pixels of a row (128-bit streaming loads / stores).
//   LX == 0 (strip): a warp is a 128-pixel strip of one row (linear order).
//   LX  > 0 (patch): a chunk is 8 warp tiles of (4 LX) x (32 / LX) pixels: LX lanes side by side,
//                    32 / LX rows.  The flow-displaced taps of one gather / RED instruction then fall
//                    into fewer distinct 128-byte lines.  Needs W % (4 LX) == 0 and H % (32 / LX) == 0.
template <int LX>
struct PatchSite {
  int base;     // linear index of the thread's first pixel
  int r, c0;    // its row / column
  bool inside;  // the warp tile exists (the last chunk of a frame may be partial)
};
template <int LX>
__device__ __forceinline__ PatchSite<LX> patch_site(int chunk, int W, int tiles_x, int tiles) {
  constexpr int kRows = 32 / LX;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int wt = chunk * (kThreads / 32) + warp;
  const int band = wt / tiles_x, tx = wt - band * tiles_x;
  PatchSite<LX> s;
  s.inside = wt < tiles;
  s.r = band * kRows + lane / LX;
  s.c0 = tx * (4 * LX) + 4 * (lane % LX);
  s.base = s.r * W + s.c0;
  return s;
}

// ================================================================== phase A: moments
// Where the data of (virtual) pair `pair` lives.  Normally item == batch element and the
// strides are the dense ones; the focal-length sweep (intrinsics_softmin.py:84-109) runs
// `cand` virtual items per batch element that all read the SAME depth / flow / weights
// (and accumulate into the same gradients) but have their own intrinsics, poses and moments.
struct PairLayout {
  int F;     // frames per item
  int cand;  // virtual items per batch element (1 = none)
  long long depth_bs, flow_bs, weight_bs;  // element strides between batch elements
};
struct PairAddr {
  int k4_frame_a;          // row of k4 for the earlier frame (virtual frame index)
  long long depth_a;       // element offset of the earlier frame's depth
  long long flow, weight;  // element offsets of the pair's flow / weights
};
__host__ __device__ inline PairLayout dense_layout(int F, int H, int W) {
  PairLayout l;
  const long long N = (long long)H * W;
  l.F = F; l.cand = 1; l.depth_bs = F * N; l.flow_bs = (F - 1) * N * 2; l.weight_bs = (F - 1) * N;
  return l;
}
__device__ __forceinline__ PairAddr pair_addr(const PairLayout& l, int pair, int N) {
  const int item = pair / (l.F - 1), i = pair - item * (l.F - 1);
  const int rb = item / l.cand;
  PairAddr a;
  a.k4_frame_a = item * l.F + i;
  a.depth_a = rb * l.depth_bs + (long long)i * N;
  a.flow = rb * l.flow_bs + (long long)i * N * 2;
  a.weight = rb * l.weight_bs + (long long)i * N;
  return a;
}
// z0: the pair's stored conditioning shift (the forward reads it from Workspace::zshift, the
// backward from its PairAdjoint, which the solve filled from the same value).
__device__ __forceinline__ PairGeom pair_geom(const float* k4, const PairAddr& pa, int H, int W, float z0) {
  PairGeom g;
  g.ka = make_cam(load_k4(k4, pa.k4_frame_a));
  g.kb = make_cam(load_k4(k4, pa.k4_frame_a + 1));
  g.grid = make_grid(H, W);
  g.z0 = z0;
  return g;
}

// The conditioning shift of every moment pair (shift_sample / shift_from_sums in fm_pixel.cuh): one
// block per pair, kShiftSamples gathers of the later frame's depth and the pair's weights.
__global__ void __launch_bounds__(kThreads)
k_pair_shift(const float* __restrict__ depth, const float* __restrict__ weights, float wsens,
             float* __restrict__ zshift, PairLayout lay, int H, int W) {
  __shared__ double smem[3][kThreads / 32];
  const int pair = blockIdx.x, N = H * W;
  const PairAddr pa = pair_addr(lay, pair, N);
  const float* db = depth + pa.depth_a + N;
  const float* wt = weights ? weights + pa.weight : nullptr;
  double s[3] = {0.0, 0.0, 0.0};  // w z, w, z
  for (int i = threadIdx.x; i < kShiftSamples; i += kThreads) {
    const int j = shift_sample(i, H, W);
    const double z = (double)__ldg(db + j), w = wt ? (double)weight_of(__ldg(wt + j), wsens) : 1.0;
    s[0] += w * z; s[1] += w; s[2] += z;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double v = warp_sum(s[k]);
    if (lane == 0) smem[k][warp] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t[3] = {0.0, 0.0, 0.0};
    for (int k = 0; k < 3; ++k)
      for (int w = 0; w < kThreads / 32; ++w) t[k] += smem[k][w];
    zshift[pair] = shift_from_sums(t[0], t[1], t[2]);
  }
}

template <int VEC>
__global__ void __launch_bounds__(kThreads, 3)
k_moments(const float* __restrict__ depth, const float* __restrict__ k4,
          const float* __restrict__ bflow, const float* __restrict__ weights,
          const int64_t* __restrict__ indices, int num_indices, double* __restrict__ moments,
          const float* __restrict__ zshift, float wsens, PairLayout lay, int H, int W) {
  __shared__ double smem[kNumMoments * (kThreads / 32)];
  const int pair = blockIdx.y;
  const int N = H * W;
  const PairAddr pa = pair_addr(lay, pair, N);
  const PairGeom g = pair_geom(k4, pa, H, W, __ldg(zshift + pair));
  const float* da = opaque_ptr(depth + pa.depth_a);
  const float* db = da + N;
  const float* fl = bflow + pa.flow;
  const float* wt = weights ? weights + pa.weight : nullptr;
  auto load_a = [da](int o) { return __ldg(da + o); };
  // float32 per-thread partials: a thread sees at most a few dozen (shifted, O(1)) terms, the
  // cross-thread / cross-block sums run in float64.
  float acc[kNumMoments];
#pragma unroll
  for (int i = 0; i < kNumMoments; ++i) acc[i] = 0.f;

  {  // index mode only (subsampled Procrustes, the focal sweep); all pixels: k_moments_dense
    for (int t = blockIdx.x * kThreads + threadIdx.x; t < num_indices; t += gridDim.x * kThreads) {
      const int j = (int)indices[t];
      const int r = j / W, c = j - r * W;
      float p[3], q[3];
      Taps taps;
      point_pq(g, pix_coord(c, g.grid.Wf, g.grid.invW), pix_coord(r, g.grid.Hf, g.grid.invH),
               __ldg(db + j), __ldg(fl + 2 * j), __ldg(fl + 2 * j + 1), load_a, p, q, taps);
      moments_add(acc, wt ? weight_of(__ldg(wt + j), wsens) : 1.f, p, q);
    }
  }
  block_accumulate<kNumMoments>(acc, moments + (size_t)pair * kNumMoments, smem);
}

template <int VEC, int LX>
__global__ void __launch_bounds__(kThreads, 3)
k_moments_dense(const float* __restrict__ depth, const float* __restrict__ k4,
                const float* __restrict__ bflow, const float* __restrict__ weights,
                double* __restrict__ moments, const float* __restrict__ zshift, float wsens, PairLayout lay,
                int H, int W, int BP, int rounds) {
  __shared__ double smem[kNumMoments * (kThreads / 32)];
  const int N = H * W;
  constexpr int kChunk = kThreads * VEC;
  const int chunks = (N + kChunk - 1) / kChunk;
  const int dr = kChunk / W, dc = kChunk - dr * W;
  const int tiles_x = LX > 0 ? W / (4 * LX) : 1, tiles = N / 128;
#pragma unroll 1
  for (int round = 0; round < rounds; ++round) {
  const ItemRange range = block_item_range((long long)BP * chunks, rounds, round);
#pragma unroll 1
  for (int i = range.i0; i < range.i1;) {
    const int pair = i / chunks, cb = i - pair * chunks;
    const int ce = (cb + (range.i1 - i) < chunks) ? cb + (range.i1 - i) : chunks;
    const PairAddr pa = pair_addr(lay, pair, N);
    const PairGeom g = pair_geom(k4, pa, H, W, __ldg(zshift + pair));
    const float* da = opaque_ptr(depth + pa.depth_a);
    const float* db = da + N;
    const float* fl = bflow + pa.flow;
    const float* wt = weights ? weights + pa.weight : nullptr;
    auto load_a = [da](int o) { return __ldg(da + o); };
    float acc[kNumMoments];
#pragma unroll
    for (int k = 0; k < kNumMoments; ++k) acc[k] = 0.f;
    int base = (cb * kThreads + (int)threadIdx.x) * VEC;
    int r = base / W, c0 = base - r * W;
#pragma unroll 1
    for (int c = cb; c < ce; ++c, base += kChunk) {
      bool inside = base < N;
      if constexpr (LX > 0) {
        const PatchSite<LX> ps = patch_site<LX>(c, W, tiles_x, tiles);
        base = ps.base; r = ps.r; c0 = ps.c0; inside = ps.inside;
      }
      if (inside) {
        float dv[VEC], wv[VEC], fv[2 * VEC];
        load_vec<VEC>(db + base, dv);
        load_vec2<VEC>(fl + 2 * base, fv);
        if (wt) {
          load_vec<VEC>(wt + base, wv);
#pragma unroll
          for (int v = 0; v < VEC; ++v) wv[v] = weight_of(wv[v], wsens);
        } else {
#pragma unroll
          for (int v = 0; v < VEC; ++v) wv[v] = 1.f;
        }
        const float y = pix_coord(r, g.grid.Hf, g.grid.invH);
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          float p[3], q[3];
          Taps taps;
          point_pq(g, pix_coord(c0 + v, g.grid.Wf, g.grid.invW), y, dv[v], fv[2 * v], fv[2 * v + 1],
                   load_a, p, q, taps);
          moments_add(acc, wv[v], p, q);
        }
      }
      r += dr; c0 += dc;
      if (c0 >= W) { c0 -= W; ++r; }
    }
    block_accumulate<kNumMoments>(acc, moments + (size_t)pair * kNumMoments, smem);
    i += ce - cb;
  }
  }
}

// ================================================================== phase B: solve
// moments_k4 != NULL: the sums were accumulated with the intrinsics moments_k4 (same principal points,
// other focal lengths) before the step's own K was known.  Points scale per axis with the focal
// ratio (p = S_b p', q = S_a q', S = diag(fx'/fx, fy'/fy, 1); the conditioning shift is along z), so
// the 16 sums are rescaled exactly here -- and written back for later readers of the workspace.
__global__ void k_solve(double* __restrict__ moments, const float* __restrict__ zshift,
                        float* __restrict__ rt, PairState* __restrict__ state, int BP, PairLayout lay,
                        int H, int W, const float* __restrict__ moments_k4 = nullptr,
                        const float* __restrict__ k4 = nullptr) {
  const int pair = blockIdx.x * blockDim.x + threadIdx.x;
  if (pair >= BP) return;
  const PairAddr pa = pair_addr(lay, pair, H * W);
  const double z0 = (double)zshift[pair];  // the shift the moment pass used
  double m[kNumMoments];
  for (int k = 0; k < kNumMoments; ++k) m[k] = moments[(size_t)pair * kNumMoments + k];
  if (moments_k4) {
    const int fa = pa.k4_frame_a, fb = fa + 1;
    const double sa[3] = {(double)moments_k4[fa * 4 + 0] / (double)k4[fa * 4 + 0],
                          (double)moments_k4[fa * 4 + 1] / (double)k4[fa * 4 + 1], 1.0};
    const double sb[3] = {(double)moments_k4[fb * 4 + 0] / (double)k4[fb * 4 + 0],
                          (double)moments_k4[fb * 4 + 1] / (double)k4[fb * 4 + 1], 1.0};
    for (int i = 0; i < 3; ++i) { m[1 + i] *= sb[i]; m[4 + i] *= sa[i]; }
    for (int a = 0; a < 3; ++a)
      for (int c = 0; c < 3; ++c) m[7 + a * 3 + c] *= sa[a] * sb[c];
    for (int k = 0; k < kNumMoments; ++k) moments[(size_t)pair * kNumMoments + k] = m[k];
  }
  const double shift[3] = {0.0, 0.0, z0};
  PairState st;
  float out[12];
  procrustes_solve(m, shift, out, st);
  for (int k = 0; k < 12; ++k) rt[(size_t)pair * 12 + k] = out[k];
  state[pair] = st;
}

// ================================================================== phase C: flow loss
// Accumulator slots per frame k (kFlowAcc doubles):
//  0        loss numerator (already scaled by weight / mask_sum)
//  1..9     forward term of pair (k, k+1): A[l][m] = sum (s - t)_l dY_m      (dR)
//  10..12   forward term: b = sum dY                                        (dt = -R b)
//  13..21   backward term of pair (k-1, k): sum dX_l s_m                    (dR)
//  22..24   backward term: sum dX                                           (dt)
//  25..28   dK_k through the unprojection ray (fx fy cx cy)
//  29..32   dK_{k+1} through the forward-term projection
//  33..36   dK_{k-1} through the backward-term projection
// Body for one frame with compile-time knowledge of which of its two pairs exist.
template <int VEC, bool HASF, bool HASB>
__device__ __forceinline__ void flow_frame_body(const FlowFrame& f, const float* __restrict__ D,
                                                const float* __restrict__ ff, const float* __restrict__ mf,
                                                const float* __restrict__ fb, const float* __restrict__ mb,
                                                float* __restrict__ gd, float g, const RobustCfg& rc,
                                                const GridDims& grid, int N, float* acc) {
  const int W = grid.W;
  const int stride = gridDim.x * kThreads * VEC;
  int base = (blockIdx.x * kThreads + threadIdx.x) * VEC;
  int r = base / W, c0 = base - r * W;          // one division, then incremental updates
  const int dr = stride / W, dc = stride - dr * W;
#pragma unroll 1
  for (; base < N; base += stride) {
    float dv[VEC], ffv[2 * VEC], fbv[2 * VEC], mfv[VEC], mbv[VEC], out[VEC];
    load_vec<VEC>(D + base, dv);
    if (HASF) { load_vec2<VEC>(ff + 2 * base, ffv); load_vec<VEC>(mf + base, mfv); }
    if (HASB) { load_vec2<VEC>(fb + 2 * base, fbv); load_vec<VEC>(mb + base, mbv); }
    const float y = pix_coord(r, grid.Hf, grid.invH);
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
      out[v] = flow_pixel<HASF, HASB>(f, pix_coord(c0 + v, grid.Wf, grid.invW), y, dv[v],
                                      HASF ? ffv[2 * v] : 0.f, HASF ? ffv[2 * v + 1] : 0.f,
                                      HASF ? mfv[v] : 0.f, HASB ? fbv[2 * v] : 0.f,
                                      HASB ? fbv[2 * v + 1] : 0.f, HASB ? mbv[v] : 0.f, g, rc, acc);
    }
    if (VEC == 4) *reinterpret_cast<float4*>(gd + base) = make_float4(out[0], out[1], out[2], out[3]);
    else gd[base] = out[0];
    r += dr; c0 += dc;
    if (c0 >= W) { c0 -= W; ++r; }
  }
}

template <int VEC>
__global__ void __launch_bounds__(kThreads, 2)
k_flow(const float* __restrict__ depth, const float* __restrict__ k4, const float* __restrict__ rt,
       const float* __restrict__ fflow, const float* __restrict__ bflow,
       const float* __restrict__ fmask, const float* __restrict__ bmask,
       const double* __restrict__ mask_sum, const float* __restrict__ grad_scale, int mapping,
       float delta, float loss_weight, float* __restrict__ g_depth, double* __restrict__ flowacc, int F,
       int H, int W) {
  __shared__ double smem[kFlowVals * (kThreads / 32)];
  const int frame = blockIdx.y;
  const int bi = frame / F, i = frame - bi * F;
  const int N = H * W;
  FlowFrame f;
  f.hasF = i < F - 1;
  f.hasB = i > 0;
  f.kk = make_cam(load_k4(k4, frame));
  f.kn = make_cam(load_k4(k4, f.hasF ? frame + 1 : frame));
  f.kp = make_cam(load_k4(k4, f.hasB ? frame - 1 : frame));
  const int pairF = bi * (F - 1) + i, pairB = pairF - 1;
  if (f.hasF) f.tf = load_rt(rt, pairF);
  if (f.hasB) f.tb = load_rt(rt, pairB);
  double den = mask_sum ? *mask_sum : 1.0;
  if (den == 0.0) den = 1.0;  // loss_flow.py:70 "valid_sum or 1"
  const float g = (float)((double)loss_weight * (grad_scale ? (double)*grad_scale : 1.0) / den);
  const RobustCfg rc = make_robust(mapping, delta, H, W);
  const GridDims grid = make_grid(H, W);

  const float* D = depth + (size_t)frame * N;
  const float* ff = fflow + (size_t)(f.hasF ? pairF : 0) * N * 2;
  const float* mf = fmask + (size_t)(f.hasF ? pairF : 0) * N;
  const float* fb = bflow + (size_t)(f.hasB ? pairB : 0) * N * 2;
  const float* mb = bmask + (size_t)(f.hasB ? pairB : 0) * N;
  float* gd = g_depth + (size_t)frame * N;

  float acc[kFlowVals];
#pragma unroll
  for (int k = 0; k < kFlowVals; ++k) acc[k] = 0.f;
  if (f.hasF && f.hasB) flow_frame_body<VEC, true, true>(f, D, ff, mf, fb, mb, gd, g, rc, grid, N, acc);
  else if (f.hasF) flow_frame_body<VEC, true, false>(f, D, ff, mf, fb, mb, gd, g, rc, grid, N, acc);
  else flow_frame_body<VEC, false, true>(f, D, ff, mf, fb, mb, gd, g, rc, grid, N, acc);
  block_accumulate<kFlowVals>(acc, flowacc + (size_t)frame * kFlowAcc, smem);
}

// Chunks ahead whose streaming operands k_flow_lean requests into L2.
constexpr int kFlowPrefetchChunks = 2;
// Lean phase C (constant intrinsics or one shared focal length): see fm_pixel.cuh.  The vector
// instantiation processes its 4 pixels as two pairs (F2, fm_math.cuh).
template <int VEC, bool HASF, bool HASB, bool FOCAL>
__device__ __forceinline__ void flow_frame_body_lean(const FlowFrameLean& f, const float* __restrict__ D,
                                                     const float* __restrict__ ff, const float* __restrict__ mf,
                                                     const float* __restrict__ fb, const float* __restrict__ mb,
                                                     float* __restrict__ gd, float g, const RobustCfg& rc,
                                                     const GridDims& grid, int N, float* acc, int chunk_begin,
                                                     int chunk_end) {
  const int W = grid.W;
  constexpr int stride = kThreads * VEC;  // one chunk per iteration (see block_item_range)
  int base = (chunk_begin * kThreads + (int)threadIdx.x) * VEC;
  int r = base / W, c0 = base - r * W;
  const int dr = stride / W, dc = stride - dr * W;
  F2 acc2[kFlowLeanVals];
  if (VEC == 4) {
#pragma unroll
    for (int k = 0; k < kFlowLeanVals; ++k) acc2[k] = f2s(0.f);
  }
  const int end = chunk_end * stride < N ? chunk_end * stride : N;
#pragma unroll 1
  for (; base < end; base += stride) {
    float dv[VEC], ffv[2 * VEC], fbv[2 * VEC], mfv[VEC], mbv[VEC], out[VEC];
    load_vec<VEC>(D + base, dv);
    if (HASF) { load_vec2<VEC>(ff + 2 * base, ffv); load_vec<VEC>(mf + base, mfv); }
    if (HASB) { load_vec2<VEC>(fb + 2 * base, fbv); load_vec<VEC>(mb + base, mbv); }
    {
      const int pb = base + kFlowPrefetchChunks * stride;
      if (pb < N) {
        prefetch_l2(D + pb);
        if (HASF) { prefetch_l2(ff + 2 * pb); prefetch_l2(mf + pb); }
        if (HASB) { prefetch_l2(fb + 2 * pb); prefetch_l2(mb + pb); }
      }
    }
    const float y = pix_coord(r, grid.Hf, grid.invH);
    if (VEC == 4) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int v = 2 * h;
        const F2 x = f2(pix_coord(c0 + v, grid.Wf, grid.invW), pix_coord(c0 + v + 1, grid.Wf, grid.invW));
        const F2 z = f2s(0.f);
        const F2 o = flow_pixel_lean2<HASF, HASB, FOCAL>(
            f, x, y, f2(dv[v], dv[v + 1]), HASF ? f2(ffv[2 * v], ffv[2 * v + 2]) : z,
            HASF ? f2(ffv[2 * v + 1], ffv[2 * v + 3]) : z, HASF ? f2(mfv[v], mfv[v + 1]) : z,
            HASB ? f2(fbv[2 * v], fbv[2 * v + 2]) : z, HASB ? f2(fbv[2 * v + 1], fbv[2 * v + 3]) : z,
            HASB ? f2(mbv[v], mbv[v + 1]) : z, g, rc, acc2);
        out[v] = o.x; out[v + 1] = o.y;
      }
      *reinterpret_cast<float4*>(gd + base) = make_float4(out[0], out[1], out[2], out[3]);
    } else {
      out[0] = flow_pixel_lean<HASF, HASB, FOCAL>(
          f, pix_coord(c0, grid.Wf, grid.invW), y, dv[0], HASF ? ffv[0] : 0.f, HASF ? ffv[1] : 0.f,
          HASF ? mfv[0] : 0.f, HASB ? fbv[0] : 0.f, HASB ? fbv[1] : 0.f, HASB ? mbv[0] : 0.f, g, rc, acc);
      gd[base] = out[0];
    }
    r += dr; c0 += dc;
    if (c0 >= W) { c0 -= W; ++r; }
  }
  if (VEC == 4) {
#pragma unroll
    for (int k = 0; k < kFlowLeanVals; ++k) acc[k] += acc2[k].x + acc2[k].y;
  }
}

template <int VEC, bool FOCAL, int MINB>
__global__ void __launch_bounds__(kThreads, MINB)
k_flow_lean(const float* __restrict__ depth, const float* __restrict__ k4, const float* __restrict__ rt,
            const float* __restrict__ fflow, const float* __restrict__ bflow,
            const float* __restrict__ fmask, const float* __restrict__ bmask,
            const double* __restrict__ mask_sum, int mapping, float delta, float loss_weight,
            float* __restrict__ g_depth, double* __restrict__ leanacc, int F, int H, int W, int BF) {
  __shared__ double smem[kFlowLeanVals * (kThreads / 32)];
  const int N = H * W;
  constexpr int kChunk = kThreads * VEC;
  const int chunks = (N + kChunk - 1) / kChunk;
  const ItemRange range = block_item_range((long long)BF * chunks);
  double den = mask_sum ? *mask_sum : 1.0;
  if (den == 0.0) den = 1.0;  // loss_flow.py:70 "valid_sum or 1"
  const float g = (float)((double)loss_weight / den);
  const RobustCfg rc = make_robust(mapping, delta, H, W);
  const GridDims grid = make_grid(H, W);
#pragma unroll 1
  for (int it = range.i0; it < range.i1;) {
    const int frame = it / chunks, cb = it - frame * chunks;
    const int ce = (cb + (range.i1 - it) < chunks) ? cb + (range.i1 - it) : chunks;
    const int bi = frame / F, i = frame - bi * F;
    const bool hasF = i < F - 1, hasB = i > 0;
    FlowFrameLean f;
    f.kk = make_cam(load_k4(k4, frame));
    f.kn = make_cam(load_k4(k4, hasF ? frame + 1 : frame));
    f.kp = make_cam(load_k4(k4, hasB ? frame - 1 : frame));
    const int pairF = bi * (F - 1) + i, pairB = pairF - 1;
    Rt tf, tb;
    if (hasF) tf = load_rt(rt, pairF);
    if (hasB) tb = load_rt(rt, pairB);
    fill_lean(f, hasF ? &tf : nullptr, hasB ? &tb : nullptr);
    const float* D = depth + (size_t)frame * N;
    const float* ff = fflow + (size_t)(hasF ? pairF : 0) * N * 2;
    const float* mf = fmask + (size_t)(hasF ? pairF : 0) * N;
    const float* fb = bflow + (size_t)(hasB ? pairB : 0) * N * 2;
    const float* mb = bmask + (size_t)(hasB ? pairB : 0) * N;
    float* gd = g_depth + (size_t)frame * N;
    float acc[kFlowLeanVals];
#pragma unroll
    for (int k = 0; k < kFlowLeanVals; ++k) acc[k] = 0.f;
    if (hasF && hasB) flow_frame_body_lean<VEC, true, true, FOCAL>(f, D, ff, mf, fb, mb, gd, g, rc, grid, N, acc, cb, ce);
    else if (hasF) flow_frame_body_lean<VEC, true, false, FOCAL>(f, D, ff, mf, fb, mb, gd, g, rc, grid, N, acc, cb, ce);
    else flow_frame_body_lean<VEC, false, true, FOCAL>(f, D, ff, mf, fb, mb, gd, g, rc, grid, N, acc, cb, ce);
    // lean slots live in the upper half of the frame's accumulator row until k_flow_lean_convert
    block_accumulate<kFlowLeanVals>(acc, leanacc + (size_t)frame * kFlowAcc, smem);
    it += ce - cb;
  }
}

// Rewrites each frame's lean accumulators (slots 0-13) into the standard layout in place.
__global__ void k_flow_lean_convert(double* __restrict__ flowacc, const float* __restrict__ rt,
                                    const float* __restrict__ k4, int focal_mode, int B, int F, int H, int W) {
  const int frame = blockIdx.x * blockDim.x + threadIdx.x;
  if (frame >= B * F) return;
  const int bi = frame / F, i = frame - bi * F;
  double lean[kFlowLeanVals], out[kFlowVals];
  double* row = flowacc + (size_t)frame * kFlowAcc;
  for (int k = 0; k < kFlowLeanVals; ++k) lean[k] = row[k];
  const int pairF = bi * (F - 1) + i;
  const float* rtF = i < F - 1 ? rt + (size_t)pairF * 12 : nullptr;
  const float* rtB = i > 0 ? rt + (size_t)(pairF - 1) * 12 : nullptr;
  const double s = sqrt((double)H * (double)W);
  const double focal = (double)k4[(size_t)frame * 4] * (double)W / s;
  lean_to_standard<double>(lean, rtF, rtB, focal, (double)W / s, focal_mode != 0, out);
  for (int k = 0; k < kFlowVals; ++k) row[k] = out[k];
}

// Assemble dL/d[R|t] of pair p (float64, 12 values) from the per-frame accumulators.
__device__ inline void flow_pose_grad(const double* flowacc, const PairState* st, const float* rt,
                                      int pair, int F, double* g) {
  const int bi = pair / (F - 1), i = pair - bi * (F - 1);
  const int a = bi * F + i;
  const double* fa = flowacc + (size_t)a * kFlowAcc;        // forward term lives on frame a
  const double* fb = flowacc + (size_t)(a + 1) * kFlowAcc;  // backward term on frame b
  double R[9];
  if (st) { for (int k = 0; k < 9; ++k) R[k] = st[pair].R[k]; }
  else { for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) R[r * 3 + c] = rt[(size_t)pair * 12 + r * 4 + c]; }
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) g[r * 4 + c] = fa[1 + r * 3 + c] + fb[13 + r * 3 + c];
    g[r * 4 + 3] = fb[22 + r] - (R[r * 3 + 0] * fa[10] + R[r * 3 + 1] * fa[11] + R[r * 3 + 2] * fa[12]);
  }
}

// Per-frame dK from the flow loss: own ray term + projection terms of the neighbours.
__device__ inline void flow_k4_grad(const double* flowacc, int frame, int F, double* g) {
  const int i = frame % F;
  const double* f = flowacc + (size_t)frame * kFlowAcc;
  for (int k = 0; k < 4; ++k) g[k] = f[25 + k];
  if (i > 0) { const double* p = f - kFlowAcc; for (int k = 0; k < 4; ++k) g[k] += p[29 + k]; }
  if (i < F - 1) { const double* n = f + kFlowAcc; for (int k = 0; k < 4; ++k) g[k] += n[33 + k]; }
}

__global__ void k_flow_finalize(const double* __restrict__ flowacc, const float* __restrict__ rt,
                                float* __restrict__ loss, float* __restrict__ g_rt,
                                float* __restrict__ g_k4, int B, int F) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int BP = B * (F - 1), BF = B * F;
  if (t < BP && g_rt) {
    double g[12];
    flow_pose_grad(flowacc, nullptr, rt, t, F, g);
    for (int k = 0; k < 12; ++k) g_rt[(size_t)t * 12 + k] = (float)g[k];
  }
  if (t < BF && g_k4) {
    double g[4];
    flow_k4_grad(flowacc, t, F, g);
    for (int k = 0; k < 4; ++k) g_k4[(size_t)t * 4 + k] = (float)g[k];
  }
  if (blockIdx.x == 0 && loss) {  // block 0: the per-frame loss terms, summed in parallel
    __shared__ double part[32];
    double s = 0.0;
    for (int k = threadIdx.x; k < BF; k += blockDim.x) s += flowacc[(size_t)k * kFlowAcc];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      double tot = 0.0;
      for (int w = 0; w < (int)((blockDim.x + 31) >> 5); ++w) tot += part[w];
      *loss = (float)tot;
    }
  }
}

// ================================================================== phase D1: adjoint solve
// focal_moments != NULL (tiled path, all frames share one focal length): the pair's Procrustes part
// of d loss / d focal is taken from the moment sums (fm_procrustes.cuh) and booked as the
// equivalent d/dfx of the pair's earlier frame in k4acc -- the per-pixel kernels carry no
// intrinsics accumulators at all.
__global__ void k_adjoint(const double* __restrict__ flowacc, const PairState* __restrict__ state,
                          const float* __restrict__ g_rt, int include_flow,
                          const float* __restrict__ flow_scale, PairAdjoint* __restrict__ adj, int BP,
                          int F, const double* __restrict__ focal_moments = nullptr,
                          const float* __restrict__ k4 = nullptr, double* __restrict__ k4acc = nullptr) {
  const int pair = blockIdx.x * blockDim.x + threadIdx.x;
  if (pair >= BP) return;
  double g[12];
  for (int k = 0; k < 12; ++k) g[k] = 0.0;
  if (include_flow) {
    flow_pose_grad(flowacc, state, nullptr, pair, F, g);
    const double s = flow_scale ? (double)*flow_scale : 1.0;
    for (int k = 0; k < 12; ++k) g[k] *= s;
  }
  if (g_rt) for (int k = 0; k < 12; ++k) g[k] += (double)g_rt[(size_t)pair * 12 + k];
  PairAdjoint out;
  if (focal_moments) {
    double dbl[15];
    procrustes_adjoint(state[pair], g, out, dbl);
    const int bi = pair / (F - 1), a = bi * F + (pair - bi * (F - 1));
    const double fdf = procrustes_focal_log_grad(state[pair], focal_moments + (size_t)pair * kNumMoments, dbl);
    k4acc[(size_t)a * 4] = fdf / (double)k4[(size_t)a * 4];  // f dL/df = fx dL/dfx
  } else {
    procrustes_adjoint(state[pair], g, out);
  }
  adj[pair] = out;
}

// ================================================================== phase D2: distribute
// Optional Adam update of the weight logits inside phase D2 (dense path): their gradient is
// final there and the kernel is bound by its scatter, not HBM, so the 28 B/parameter of a separate
// Adam pass over the weights disappear into it.
struct AdamFuse {
  float* m; float* v;
  float beta1, beta2, omb1, omb2, eps, step_size, bc2_sqrt;
  int on;
  int first_pair;  // pairs below this index are left to a later, separate Adam call
  const float* consts;  // device {step_size, bc2_sqrt} of a step clock (CUDA-graph replays), or NULL
};

template <int VEC>
__global__ void __launch_bounds__(kThreads, 3)
k_distribute(const float* __restrict__ depth, const float* __restrict__ k4,
             const float* __restrict__ bflow, float* weights,
             const int64_t* __restrict__ indices, int num_indices,
             const PairAdjoint* __restrict__ adj, float* __restrict__ g_depth,
             float* __restrict__ g_weights, double* __restrict__ k4acc, float wsens, PairLayout lay,
             AdamFuse adam, int H, int W) {
  __shared__ double smem[8 * (kThreads / 32)];
  __shared__ PairAdjoint s_adj;
  const int pair = blockIdx.y;
  const int N = H * W;
  if (threadIdx.x < sizeof(PairAdjoint) / 4)
    reinterpret_cast<float*>(&s_adj)[threadIdx.x] = reinterpret_cast<const float*>(adj + pair)[threadIdx.x];
  __syncthreads();
  const PairAdjoint ad = s_adj;
  const PairAddr pa = pair_addr(lay, pair, N);
  const PairGeom g = pair_geom(k4, pa, H, W, ad.shift[2]);
  const int a = pa.k4_frame_a;
  if (adam.on && adam.consts) { adam.step_size = __ldg(adam.consts); adam.bc2_sqrt = __ldg(adam.consts + 1); }
  const float* da = opaque_ptr(depth + pa.depth_a);
  const float* db = da + N;
  const float* fl = bflow + pa.flow;
  float* wt = weights ? weights + pa.weight : nullptr;
  float* gda = g_depth + pa.depth_a;
  auto load_a = [da](int o) { return __ldg(da + o); };
  auto scatter = [gda, W](int y0, int x0, float v0, float v1) { red_pair<VEC == 4>(gda + y0 * W, x0, W, v0, v1); };
  float* gdb = gda + N;
  float* gw = g_weights ? g_weights + pa.weight : nullptr;
  float kacc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) kacc[k] = 0.f;

  {  // index mode only; all pixels: k_distribute_window / k_distribute_dense
    for (int t = blockIdx.x * kThreads + threadIdx.x; t < num_indices; t += gridDim.x * kThreads) {
      const int j = (int)indices[t];
      const int r = j / W, c = j - r * W;
      float gdj, gwj;
      const float wj = wt ? weight_of(__ldg(wt + j), wsens) : 1.f;
      distribute_point(g, ad, pix_coord(c, g.grid.Wf, g.grid.invW),
                       pix_coord(r, g.grid.Hf, g.grid.invH), __ldg(db + j),
                       wj, __ldg(fl + 2 * j), __ldg(fl + 2 * j + 1), load_a,
                       scatter, gdj, gwj, kacc);
      red_add(gdb + j, gdj);
      if (gw) red_add(gw + j, wsens != 0.f ? gwj * wsens * wj * (1.0f - wj) : gwj);
    }
  }
  // kacc[0..3] -> frame a, kacc[4..7] -> frame b = a + 1: contiguous in k4acc
  block_accumulate<8>(kacc, k4acc + (size_t)a * 4, smem);
}

// Per-pixel work of the dense phase D2 for the VEC consecutive pixels of row r from column c0
// (linear index base in the frame, wi = base + the pair's offset in the weight-shaped arrays): the
// earlier frame's taps go to `scatter`, the later frame's depth gradient is one aligned RED, then the
// weight gradient and (fuse_adam) the Adam update of the logits.  The weight-shaped arrays are passed
// without the pair's offset.
template <int VEC, typename Scatter>
__device__ __forceinline__ void distribute_pixels(const PairGeom& g, const PairAdjoint& ad, const float* da,
                                                  const float* db, const float* fl, float* weights, float* gdb,
                                                  float* g_weights, float wsens, const AdamFuse& adam,
                                                  bool fuse_adam, long long wi, int base, int r, int c0,
                                                  Scatter scatter, float* kacc) {
  auto load_a = [da](int o) { return __ldg(da + o); };
  float dv[VEC], wv[VEC], wraw[VEC], fv[2 * VEC], gwv[VEC], gdv[VEC];
  load_vec<VEC>(db + base, dv);
  load_vec2<VEC>(fl + 2 * base, fv);
  float* wt = weights ? weights + wi : nullptr;
  if (wt) {
    if (VEC == 4) {  // plain (coherent) load: the logits may be updated in place below
      const float4 w4 = *reinterpret_cast<const float4*>(wt);
      wraw[0] = w4.x; wraw[1] = w4.y; wraw[2] = w4.z; wraw[3] = w4.w;
    } else {
      wraw[0] = *wt;
    }
#pragma unroll
    for (int v = 0; v < VEC; ++v) wv[v] = weight_of(wraw[v], wsens);
  } else {
#pragma unroll
    for (int v = 0; v < VEC; ++v) wv[v] = 1.f;
  }
  const float y = pix_coord(r, g.grid.Hf, g.grid.invH);
#pragma unroll
  for (int v = 0; v < VEC; ++v)
    distribute_point(g, ad, pix_coord(c0 + v, g.grid.Wf, g.grid.invW), y, dv[v], wv[v],
                     fv[2 * v], fv[2 * v + 1], load_a, scatter, gdv[v], gwv[v], kacc);
  if (VEC == 4) red_add4(gdb + base, gdv[0], gdv[1], gdv[2], gdv[3]);
  else red_add(gdb + base, gdv[0]);
  if (wt) {
    if (wsens != 0.f) {  // chain rule of the sigmoid: d/d logit = sens * w (1 - w) * d/dw
#pragma unroll
      for (int v = 0; v < VEC; ++v) gwv[v] *= wsens * wv[v] * (1.0f - wv[v]);
    }
    if (g_weights) {
      if (VEC == 4) *reinterpret_cast<float4*>(g_weights + wi) = make_float4(gwv[0], gwv[1], gwv[2], gwv[3]);
      else g_weights[wi] = gwv[0];
    }
    if (VEC == 4 && fuse_adam) {  // torch.optim.Adam on the logits (k_adam's order)
      // the step clock's constants are re-read here (L1 hits) rather than held across the pixel loop
      const float step_size = adam.consts ? __ldg(adam.consts) : adam.step_size;
      const float bc2_sqrt = adam.consts ? __ldg(adam.consts + 1) : adam.bc2_sqrt;
      float4 mm = *reinterpret_cast<float4*>(adam.m + wi);
      float4 vv = *reinterpret_cast<float4*>(adam.v + wi);
      float* mp = &mm.x; float* vp = &vv.x;
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        mp[v] = mp[v] + adam.omb1 * (gwv[v] - mp[v]);
        vp[v] = vp[v] * adam.beta2 + adam.omb2 * gwv[v] * gwv[v];
        wraw[v] = wraw[v] - step_size * (mp[v] / (sqrtf(vp[v]) / bc2_sqrt + adam.eps));
      }
      *reinterpret_cast<float4*>(adam.m + wi) = mm;
      *reinterpret_cast<float4*>(adam.v + wi) = vv;
      *reinterpret_cast<float4*>(wt) = make_float4(wraw[0], wraw[1], wraw[2], wraw[3]);
    }
  }
}

// Dense (all-pixel) phase D2 for widths that are not a multiple of 4: one pixel per thread on the
// item decomposition of block_item_range (chunks of kThreads pixels), taps as REDs, per-pair constants
// re-staged when a block moves on to its next pair.  The weight Adam runs as a separate pass.
__global__ void __launch_bounds__(kThreads, 3)
k_distribute_dense(const float* __restrict__ depth, const float* __restrict__ k4,
                   const float* __restrict__ bflow, float* weights, const PairAdjoint* __restrict__ adj,
                   float* __restrict__ g_depth, float* __restrict__ g_weights, double* __restrict__ k4acc,
                   float wsens, PairLayout lay, AdamFuse adam, int H, int W, int BP, int rounds) {
  __shared__ double smem[8 * (kThreads / 32)];
  __shared__ PairAdjoint s_adj;
  const int N = H * W;
  const int chunks = (N + kThreads - 1) / kThreads;
  const int dr = kThreads / W, dc = kThreads - dr * W;
#pragma unroll 1
  for (int round = 0; round < rounds; ++round) {
  const ItemRange range = block_item_range((long long)BP * chunks, rounds, round);
#pragma unroll 1
  for (int i = range.i0; i < range.i1;) {
    const int pair = i / chunks, cb = i - pair * chunks;
    const int ce = (cb + (range.i1 - i) < chunks) ? cb + (range.i1 - i) : chunks;
    __syncthreads();  // the previous pair's s_adj is no longer read
    if (threadIdx.x < sizeof(PairAdjoint) / 4)
      reinterpret_cast<float*>(&s_adj)[threadIdx.x] = reinterpret_cast<const float*>(adj + pair)[threadIdx.x];
    __syncthreads();
    const PairAdjoint ad = s_adj;
    const PairAddr pa = pair_addr(lay, pair, N);
    const PairGeom g = pair_geom(k4, pa, H, W, ad.shift[2]);
    const float* da = opaque_ptr(depth + pa.depth_a);
    float* gda = g_depth + pa.depth_a;
    auto scatter = [gda, W](int y0, int x0, float v0, float v1) { red_pair<false>(gda + y0 * W, x0, W, v0, v1); };
    float kacc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) kacc[k] = 0.f;
    int base = cb * kThreads + (int)threadIdx.x;
    int r = base / W, c0 = base - r * W;
#pragma unroll 1
    for (int c = cb; c < ce; ++c, base += kThreads) {
      if (base < N)
        distribute_pixels<1>(g, ad, da, da + N, bflow + pa.flow, weights, gda + N, g_weights, wsens, adam, false,
                             pa.weight + base, base, r, c0, scatter, kacc);
      r += dr; c0 += dc;
      if (c0 >= W) { c0 -= W; ++r; }
    }
    // kacc[0..3] -> frame a, kacc[4..7] -> frame b = a + 1: contiguous in k4acc
    block_accumulate<8>(kacc, k4acc + (size_t)pa.k4_frame_a * 4, smem);
    i += ce - cb;
  }
  }
}

// Tile and halo of k_distribute_window (build-time knobs for tools/ab_libs.py).  With the defaults
// 0.04 % of the tap rows of N(0, 0.01^2) flows (6.4 x 3.6 px at 640 x 360) miss the window
// (tools/window_fallback.py).
#ifndef FM_WIN_TW
#define FM_WIN_TW 64
#endif
#ifndef FM_WIN_TH
#define FM_WIN_TH 32
#endif
#ifndef FM_WIN_HX
#define FM_WIN_HX 16
#endif
#ifndef FM_WIN_HY
#define FM_WIN_HY 12
#endif
#ifndef FM_WIN_CTAS  // resident blocks per SM (register cap: 80 at 3, 128 at 2)
#define FM_WIN_CTAS 3
#endif
constexpr int kWinTW = FM_WIN_TW, kWinTH = FM_WIN_TH;      // tile of the later frame
constexpr int kWinW = kWinTW + 2 * FM_WIN_HX, kWinH = kWinTH + 2 * FM_WIN_HY;  // window of the earlier frame
// A tap pair (x0, x0 + 1) goes to the window when x0 is inside it, so x0 + 1 may be one column past
// it: each row has one more aligned group, flushed like the others where it lies inside the image.
constexpr int kWinPitch = kWinW + 4;
constexpr int kWinRowThreads = kWinTW / 4, kWinRowsPerPass = kThreads / kWinRowThreads;
static_assert(kWinTW % 4 == 0 && FM_WIN_HX % 2 == 0 && kThreads % kWinRowThreads == 0 &&
              kWinTH % kWinRowsPerPass == 0 && kWinTW % 16 == 0 && kWinTH % 8 == 0, "window geometry");
// The window holds fixed-point sums (fix_encode in fm_math.cuh) in two int32 planes, hi and lo.
// They cannot overflow: a pixel adds to a given cell at most once (its four taps are distinct
// cells; a bottom tap row clamped onto the top one carries weight 0, and zero values are not added), so a cell
// receives at most kWinTW * kWinTH = 2048 nonzero adds per tile, each with |hi| <= 2^19 and
// lo in [0, 2^16]: |sum hi| <= 2^30 and sum lo <= 2^27.
static_assert(kWinTW * kWinTH <= 2048, "fixed-point window sums would overflow int32");
static_assert(2 * kWinH * kWinPitch * 4 + 8 * (kThreads / 32) * 8 + (int)sizeof(PairAdjoint) +
                  (int)sizeof(PairGeom) + 8 <= 48 * 1024,
              "static shared memory");

#ifdef FM_WIN_COUNT  // counting build: tap rows {in the window, out of fixed-point range, outside the window}
__device__ unsigned long long fm_win_counts[3];
#define FM_WIN_TALLY(i) atomicAdd(&fm_win_counts[i], 1ull)
}  // namespace
// copies the counts to out[3] and resets them (tools/window_counts.py); exported, so outside the
// anonymous namespace
extern "C" int fm_window_counts(unsigned long long* out) {
  static const unsigned long long zero[3] = {0, 0, 0};
  if (cudaMemcpyFromSymbol(out, fm_win_counts, sizeof(zero)) != cudaSuccess) return 1;
  return cudaMemcpyToSymbol(fm_win_counts, zero, sizeof(zero)) == cudaSuccess ? 0 : 1;
}
namespace {
#else
#define FM_WIN_TALLY(i)
#endif

// Dense phase D2 for W % 4 == 0.  Work unit: a kWinTW x kWinTH tile of the later frame (a thread owns
// 4 consecutive pixels of a row), walked with the rounds of block_item_range.  The taps into the earlier
// frame's depth gradient are added into a window of that frame in shared memory: the tile plus a halo,
// shifted by the mean backward flow of the tile and clamped onto the image, with a 16-byte aligned x
// origin.  The window sums in fixed point with native 32-bit integer shared-memory atomics (float
// atomics on shared memory are compare-and-swap loops on sm_90a), at a power-of-two scale chosen per
// pair from its constants (tap_magnitude).  Taps outside the window, and values outside the
// fixed-point range (including non-finite ones), are float REDs as in k_distribute_dense.  After the
// tile the window is converted back to float and flushed with aligned vector REDs (not stores:
// neighbouring windows overlap, and k_track_apply adds into the same gradient concurrently in
// fm_overfit_step) and zeroed.  This replaces ~2.6 scattered 32-byte RED requests per pixel (bound by
// the L2 atomic units) with ~0.7 coalesced ones.
__global__ void __launch_bounds__(kThreads, FM_WIN_CTAS)
k_distribute_window(const float* __restrict__ depth, const float* __restrict__ k4,
                    const float* __restrict__ bflow, float* weights, const PairAdjoint* __restrict__ adj,
                    float* __restrict__ g_depth, float* __restrict__ g_weights, double* __restrict__ k4acc,
                    float wsens, PairLayout lay, AdamFuse adam, int H, int W, int BP, int rounds) {
  __shared__ double smem[8 * (kThreads / 32)];
  __shared__ PairAdjoint s_adj;
  __shared__ PairGeom s_geom;
  __shared__ float s_fix[2];  // the pair's fixed-point scale 2^e and its inverse
  __shared__ __align__(16) int win_hi[kWinH * kWinPitch];
  __shared__ __align__(16) int win_lo[kWinH * kWinPitch];
  const int N = H * W;
  const int tiles_x = (W + kWinTW - 1) / kWinTW, tiles = tiles_x * ((H + kWinTH - 1) / kWinTH);
  const int lane = threadIdx.x & 31;
  for (int k = threadIdx.x; k < kWinH * kWinPitch / 4; k += kThreads) {  // barrier: the s_adj staging
    reinterpret_cast<int4*>(win_hi)[k] = make_int4(0, 0, 0, 0);
    reinterpret_cast<int4*>(win_lo)[k] = make_int4(0, 0, 0, 0);
  }
#pragma unroll 1
  for (int round = 0; round < rounds; ++round) {
  const ItemRange range = block_item_range((long long)BP * tiles, rounds, round);
#pragma unroll 1
  for (int i = range.i0; i < range.i1;) {
    const int pair = i / tiles, tb = i - pair * tiles;
    const int te = (tb + (range.i1 - i) < tiles) ? tb + (range.i1 - i) : tiles;
    __syncthreads();  // the previous pair's s_adj is no longer read
    const PairAddr pa = pair_addr(lay, pair, N);
    if (threadIdx.x < sizeof(PairAdjoint) / 4)
      reinterpret_cast<float*>(&s_adj)[threadIdx.x] = reinterpret_cast<const float*>(adj + pair)[threadIdx.x];
    if (threadIdx.x == 32) {
      const PairGeom pg = pair_geom(k4, pa, H, W, adj[pair].shift[2]);
      s_geom = pg;
      const int e = fix_exponent(tap_magnitude(adj[pair], pg));
      s_fix[0] = fix_pow2(e);
      s_fix[1] = fix_pow2(-e);
    }
    __syncthreads();
    // the pair's constants are read from shared memory: as register copies they more than double the
    // spills of the pixel loop at the 80 registers of 3 blocks per SM
    const PairAdjoint& ad = s_adj;
    const PairGeom& g = s_geom;
    const float* da = opaque_ptr(depth + pa.depth_a);
    const float* fl = bflow + pa.flow;
    float* gda = g_depth + pa.depth_a;
    const bool fuse_adam = adam.on && pair >= adam.first_pair;
    float kacc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) kacc[k] = 0.f;
#pragma unroll 1
    for (int t = tb; t < te; ++t) {
      const int ty = t / tiles_x, X0 = (t - ty * tiles_x) * kWinTW, Y0 = ty * kWinTH;
      // Window shift: the mean backward flow of 8 x 4 samples spread over the tile (every warp sums the
      // same samples in the same order, so all warps place the window identically).  A single sample
      // would move the window by the flow's own noise.
      float sx, sy;
      {
        const int sr = min(Y0 + (lane >> 3) * (kWinTH / 4) + kWinTH / 8, H - 1);
        const int sc = min(X0 + (lane & 7) * (kWinTW / 8) + kWinTW / 16, W - 1);
        const float2 f = __ldg(reinterpret_cast<const float2*>(fl) + sr * W + sc);
        sx = warp_sum_f(f.x);
        sy = warp_sum_f(f.y);
      }
      // the taps of column c lie around c + W flx - .5 (bilinear_taps); clamped first so that a
      // non-finite flow cannot overflow the integer
      const int shx = __float2int_rn(fminf(fmaxf(sx * (g.grid.Wf / 32.f) - 0.5f, -g.grid.Wf), g.grid.Wf));
      const int shy = __float2int_rn(fminf(fmaxf(sy * (g.grid.Hf / 32.f) - 0.5f, -g.grid.Hf), g.grid.Hf));
      const int wx0 = max(0, min((X0 - FM_WIN_HX + shx + 2) & ~3, W - kWinW));
      const int wy0 = max(0, min(Y0 - FM_WIN_HY + shy, H - kWinH));
      auto scatter = [=](int y0, int x0, float v0, float v1) {
        const unsigned ly = (unsigned)(y0 - wy0), lx = (unsigned)(x0 - wx0);
        const bool inside = (ly < (unsigned)kWinH) & (lx < (unsigned)kWinW);
        int h0, l0, h1, l1;
        const float fix_s = s_fix[0];  // an LDS per call: one register fewer across the pixel loop
        if (inside & fix_encode(v0, fix_s, h0, l0) & fix_encode(v1, fix_s, h1, l1)) {
          FM_WIN_TALLY(0);
          const int o = ly * kWinPitch + lx;
          if (h0 != 0) atomicAdd(win_hi + o, h0);
          if (l0 != 0) atomicAdd(win_lo + o, l0);
          if (h1 != 0) atomicAdd(win_hi + o + 1, h1);
          if (l1 != 0) atomicAdd(win_lo + o + 1, l1);
        } else {
          FM_WIN_TALLY(inside ? 1 : 2);
          red_pair<true>(gda + y0 * W, x0, W, v0, v1);
        }
      };
      const int c0 = X0 + 4 * ((int)threadIdx.x % kWinRowThreads);
#pragma unroll 1
      for (int r = Y0 + (int)threadIdx.x / kWinRowThreads; r < Y0 + kWinTH; r += kWinRowsPerPass)
        if (r < H && c0 < W)
          distribute_pixels<4>(g, ad, da, da + N, fl, weights, gda + N, g_weights, wsens, adam, fuse_adam,
                               pa.weight + r * W + c0, r * W + c0, r, c0, scatter, kacc);
      __syncthreads();
      const float inv_s = s_fix[1];
      for (int k = threadIdx.x; k < kWinH * (kWinPitch / 4); k += kThreads) {
        const int ly = k / (kWinPitch / 4), lx = (k - ly * (kWinPitch / 4)) * 4;
        int4* sh = reinterpret_cast<int4*>(win_hi) + k;
        int4* sl = reinterpret_cast<int4*>(win_lo) + k;
        const int4 h = *sh, l = *sl;
        *sh = make_int4(0, 0, 0, 0);
        *sl = make_int4(0, 0, 0, 0);
        if (wy0 + ly < H && wx0 + lx < W && ((h.x | h.y | h.z | h.w | l.x | l.y | l.z | l.w) != 0))
          red_add4(gda + (wy0 + ly) * W + wx0 + lx, fix_decode(h.x, l.x, inv_s), fix_decode(h.y, l.y, inv_s),
                   fix_decode(h.z, l.z, inv_s), fix_decode(h.w, l.w, inv_s));
      }
      __syncthreads();  // the window is zero again before the next tile's taps
    }
    // kacc[0..3] -> frame a, kacc[4..7] -> frame b = a + 1: contiguous in k4acc
    block_accumulate<8>(kacc, k4acc + (size_t)pa.k4_frame_a * 4, smem);
    i += te - tb;
  }
  }
}

#include "fm_tiled.cuh"

__global__ void k_k4_finalize(const double* __restrict__ k4acc, const double* __restrict__ flowacc,
                              int include_flow, const float* __restrict__ flow_scale,
                              float* __restrict__ g_k4, int B, int F) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * F) return;
  double g[4] = {0, 0, 0, 0};
  if (include_flow) {
    flow_k4_grad(flowacc, t, F, g);
    const double s = flow_scale ? (double)*flow_scale : 1.0;
    for (int k = 0; k < 4; ++k) g[k] *= s;
  }
  for (int k = 0; k < 4; ++k) g_k4[(size_t)t * 4 + k] = (float)(g[k] + k4acc[(size_t)t * 4 + k]);
}

__global__ void k_scale_inplace(float* __restrict__ buf, const float* __restrict__ scale, size_t n) {
  const float s = *scale;
  if (s == 1.0f) return;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    buf[i] *= s;
}

// ================================================================== mask sum
__global__ void __launch_bounds__(kThreads)
k_mask_sum(const float* __restrict__ a, const float* __restrict__ b, double* __restrict__ out, size_t n) {
  __shared__ double smem[kThreads / 32];
  double acc = 0.0;
  const size_t n4 = n / 4;
  for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n4; i += (size_t)gridDim.x * kThreads) {
    const float4 x = __ldg(reinterpret_cast<const float4*>(a) + i);
    const float4 y = __ldg(reinterpret_cast<const float4*>(b) + i);
    acc += (double)((x.x + x.y) + (x.z + x.w)) + (double)((y.x + y.y) + (y.z + y.w));
  }
  for (size_t i = n4 * 4 + (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads)
    acc += (double)a[i] + (double)b[i];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) s += smem[w];
    atomicAdd(out, s);
  }
}

// ================================================================== utilities
__global__ void k_unproject(const float* __restrict__ depth, const float* __restrict__ k4,
                            float* __restrict__ surf, int H, int W) {
  const int frame = blockIdx.y, N = H * W;
  const Cam k = make_cam(load_k4(k4, frame));
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < N; j += gridDim.x * blockDim.x) {
    const int r = j / W, c = j - r * W;
    float rx, ry;
    ray_of(pix_x(c, W), pix_y(r, H), k, rx, ry);
    const float d = __ldg(depth + (size_t)frame * N + j);
    float* o = surf + ((size_t)frame * N + j) * 3;
    o[0] = d * rx; o[1] = d * ry; o[2] = d;
  }
}

__global__ void __launch_bounds__(kThreads)
k_unproject_bwd(const float* __restrict__ depth, const float* __restrict__ k4,
                const float* __restrict__ gs, float* __restrict__ gd, double* __restrict__ gk, int H, int W) {
  __shared__ double smem[4 * (kThreads / 32)];
  const int frame = blockIdx.y, N = H * W;
  const Cam k = make_cam(load_k4(k4, frame));
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < N; j += gridDim.x * blockDim.x) {
    const int r = j / W, c = j - r * W;
    float rx, ry;
    ray_of(pix_x(c, W), pix_y(r, H), k, rx, ry);
    const float d = __ldg(depth + (size_t)frame * N + j);
    const float* g = gs + ((size_t)frame * N + j) * 3;
    const float g0 = g[0], g1 = g[1], g2 = g[2];
    gd[(size_t)frame * N + j] = g0 * rx + g1 * ry + g2;
    acc[0] -= g0 * d * rx * k.ifx;
    acc[1] -= g1 * d * ry * k.ify;
    acc[2] -= g0 * d * k.ifx;
    acc[3] -= g1 * d * k.ify;
  }
  block_accumulate<4>(acc, gk + (size_t)frame * 4, smem);
}

__global__ void k_d2f(const double* __restrict__ src, float* __restrict__ dst, int n) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) dst[t] = (float)src[t];
}

__global__ void k_reproject(const float* __restrict__ xyz, const float* __restrict__ rt,
                            const float* __restrict__ k4, float* __restrict__ xy,
                            unsigned char* __restrict__ in_front, int n) {
  const int item = blockIdx.y;
  const Rt t = load_rt(rt, item);
  const Cam k = make_cam(load_k4(k4, item));
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const float* p = xyz + ((size_t)item * n + j) * 3;
    const float s0 = p[0], s1 = p[1], s2 = p[2];
    const float X0 = t.r[0] * s0 + t.r[1] * s1 + t.r[2] * s2 + t.t[0];
    const float X1 = t.r[3] * s0 + t.r[4] * s1 + t.r[5] * s2 + t.t[1];
    const float X2 = t.r[6] * s0 + t.r[7] * s1 + t.r[8] * s2 + t.t[2];
    const Proj pr = project_point(X0, X1, X2, k);
    float* o = xy + ((size_t)item * n + j) * 2;
    o[0] = pr.uvx; o[1] = pr.uvy;
    if (in_front) in_front[(size_t)item * n + j] = X2 >= 0.f ? 1 : 0;  // projection.py:72
  }
}

// ---- pose chain as a parallel scan
// P_0 = I, P_{k+1} = P_k @ T_k (projection.py:207-209) is a prefix product of rigid [R|t]
// transforms, an associative operation: one block per batch item, every thread owns a contiguous
// chunk of pairs, a Hillis-Steele scan over the 256 chunk aggregates in shared memory (8 steps),
// then each thread walks its chunk from its exclusive prefix.  O(log F) dependent steps instead of
// F - 1, no limit on F.  (Rounding differs from the sequential product at the 1e-7 level.)
constexpr int kChainThreads = 256;

struct Rigid { float m[12]; };  // [R | t] row-major 3x4

__device__ __forceinline__ Rigid rigid_identity() {
  Rigid r;
#pragma unroll
  for (int i = 0; i < 12; ++i) r.m[i] = (i == 0 || i == 5 || i == 10) ? 1.f : 0.f;
  return r;
}
__device__ __forceinline__ Rigid rigid_load(const float* p) {  // 48 bytes, 16-byte aligned
  Rigid r;
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1),
               c = __ldg(reinterpret_cast<const float4*>(p) + 2);
  r.m[0] = a.x; r.m[1] = a.y; r.m[2] = a.z; r.m[3] = a.w; r.m[4] = b.x; r.m[5] = b.y; r.m[6] = b.z; r.m[7] = b.w;
  r.m[8] = c.x; r.m[9] = c.y; r.m[10] = c.z; r.m[11] = c.w;
  return r;
}
// A o B = [A_R B_R | A_R B_t + A_t]
__device__ __forceinline__ Rigid rigid_mul(const Rigid& A, const Rigid& B) {
  Rigid C;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float v = A.m[r * 4 + 0] * B.m[0 * 4 + c] + A.m[r * 4 + 1] * B.m[1 * 4 + c] + A.m[r * 4 + 2] * B.m[2 * 4 + c];
      if (c == 3) v += A.m[r * 4 + 3];
      C.m[r * 4 + c] = v;
    }
  }
  return C;
}
// X (3x4, general) times T4^T:  out[r][m] = sum_c X[r][c] T4[m][c], T4 row 3 = (0, 0, 0, 1)
__device__ __forceinline__ Rigid mul_transposed(const Rigid& X, const Rigid& T) {
  Rigid o;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int m = 0; m < 3; ++m)
      o.m[r * 4 + m] = X.m[r * 4 + 0] * T.m[m * 4 + 0] + X.m[r * 4 + 1] * T.m[m * 4 + 1] +
                       X.m[r * 4 + 2] * T.m[m * 4 + 2] + X.m[r * 4 + 3] * T.m[m * 4 + 3];
    o.m[r * 4 + 3] = X.m[r * 4 + 3];
  }
  return o;
}
__device__ __forceinline__ void rigid_to_smem(float* dst, const Rigid& r) {
#pragma unroll
  for (int i = 0; i < 12; ++i) dst[i * kChainThreads] = r.m[i];  // element-major: conflict-free
}
__device__ __forceinline__ Rigid rigid_from_smem(const float* src) {
  Rigid r;
#pragma unroll
  for (int i = 0; i < 12; ++i) r.m[i] = src[i * kChainThreads];
  return r;
}

__global__ void __launch_bounds__(kChainThreads)
k_pose_chain(const float* __restrict__ rt, float* __restrict__ ext, int B, int F) {
  __shared__ float s_agg[12 * kChainThreads];
  const int b = blockIdx.x, t = threadIdx.x;
  const int P = F - 1;
  const int chunk = (P + kChainThreads - 1) / kChainThreads;
  const int lo = min(t * chunk, P), hi = min(lo + chunk, P);
  const float* T = rt + (size_t)b * P * 12;
  Rigid agg = rigid_identity();
  for (int k = lo; k < hi; ++k) agg = rigid_mul(agg, rigid_load(T + (size_t)k * 12));
  rigid_to_smem(s_agg + t, agg);
  __syncthreads();
  for (int off = 1; off < kChainThreads; off <<= 1) {
    Rigid left;
    if (t >= off) left = rigid_from_smem(s_agg + t - off);
    __syncthreads();
    if (t >= off) { agg = rigid_mul(left, agg); rigid_to_smem(s_agg + t, agg); }
    __syncthreads();
  }
  Rigid run = t > 0 ? rigid_from_smem(s_agg + t - 1) : rigid_identity();  // exclusive prefix = P_lo
  float* o = ext + (size_t)b * F * 16;
  auto store = [o](int k, const Rigid& r) {
    float4* d = reinterpret_cast<float4*>(o + (size_t)k * 16);
    d[0] = make_float4(r.m[0], r.m[1], r.m[2], r.m[3]);
    d[1] = make_float4(r.m[4], r.m[5], r.m[6], r.m[7]);
    d[2] = make_float4(r.m[8], r.m[9], r.m[10], r.m[11]);
    d[3] = make_float4(0.f, 0.f, 0.f, 1.f);
  };
  if (t == 0) store(0, run);  // P_0 = I
  for (int k = lo; k < hi; ++k) {
    run = rigid_mul(run, rigid_load(T + (size_t)k * 12));
    store(k + 1, run);
  }
}

// Adjoint of the chain.  With G_a = dL/dP_a (top 3 rows; the bottom row is constant):
//   S_{F-1} = G_{F-1},  S_a = G_a + S_{a+1} T4_a^T,  dT_k = P_k^T S_{k+1} (3x4 part).
// S_a = f_a(S_{a+1}) with the affine maps f_a(X) = G_a + X T4_a^T, whose composition
// f_a o f_b (a < b) is the pair (T_a o T_b, G_a + G_b T4_a^T): a reverse (suffix) scan over the
// elements a = 1 .. F-1, same block layout as the forward chain.
__global__ void __launch_bounds__(kChainThreads)
k_pose_chain_bwd(const float* __restrict__ rt, const float* __restrict__ ext,
                 const float* __restrict__ g_ext, float* __restrict__ g_rt, int B, int F) {
  __shared__ float s_t[12 * kChainThreads];
  __shared__ float s_b[12 * kChainThreads];
  const int b = blockIdx.x, t = threadIdx.x;
  const int n = F - 1;                       // elements j = a - 1 for a = 1 .. F-1
  const int chunk = (n + kChainThreads - 1) / kChainThreads;
  const int lo = min(t * chunk, n), hi = min(lo + chunk, n);
  const float* T = rt + (size_t)b * n * 12;
  const float* G = g_ext + (size_t)b * F * 16;
  const float* Pm = ext + (size_t)b * F * 16;
  // element j: (T_a, G_a) with a = j + 1; the last one (a = F-1) has no T: identity
  auto elem_t = [T, n](int j) { return j + 1 < n + 0 ? rigid_load(T + (size_t)(j + 1) * 12) : rigid_identity(); };
  Rigid aggT = rigid_identity(), aggB;
#pragma unroll
  for (int i = 0; i < 12; ++i) aggB.m[i] = 0.f;
  // chunk aggregate: f_lo o ... o f_{hi-1}, built right to left
  for (int j = hi - 1; j >= lo; --j) {
    const Rigid tj = elem_t(j), gj = rigid_load(G + (size_t)(j + 1) * 16);
    const Rigid moved = mul_transposed(aggB, tj);
#pragma unroll
    for (int i = 0; i < 12; ++i) aggB.m[i] = gj.m[i] + moved.m[i];
    aggT = rigid_mul(tj, aggT);
  }
  rigid_to_smem(s_t + t, aggT);
  rigid_to_smem(s_b + t, aggB);
  __syncthreads();
  for (int off = 1; off < kChainThreads; off <<= 1) {
    Rigid rT, rB;
    const bool has = t + off < kChainThreads;
    if (has) { rT = rigid_from_smem(s_t + t + off); rB = rigid_from_smem(s_b + t + off); }
    __syncthreads();
    if (has) {  // (aggT, aggB) o (rT, rB) = (aggT o rT, aggB + rB aggT4^T)
      const Rigid moved = mul_transposed(rB, aggT);
#pragma unroll
      for (int i = 0; i < 12; ++i) aggB.m[i] += moved.m[i];
      aggT = rigid_mul(aggT, rT);
      rigid_to_smem(s_t + t, aggT);
      rigid_to_smem(s_b + t, aggB);
    }
    __syncthreads();
  }
  // exclusive suffix: S of the first element of the next chunk (0 past the end)
  Rigid S;
  if (t + 1 < kChainThreads) S = rigid_from_smem(s_b + t + 1);
  else {
#pragma unroll
    for (int i = 0; i < 12; ++i) S.m[i] = 0.f;
  }
  float* out = g_rt + (size_t)b * n * 12;
  for (int j = hi - 1; j >= lo; --j) {
    const Rigid tj = elem_t(j), gj = rigid_load(G + (size_t)(j + 1) * 16);
    const Rigid moved = mul_transposed(S, tj);
#pragma unroll
    for (int i = 0; i < 12; ++i) S.m[i] = gj.m[i] + moved.m[i];       // S_{j+1}
    const Rigid Pk = rigid_load(Pm + (size_t)j * 16);                  // P_j, dT_j = P_j^T S_{j+1}
    float4* d = reinterpret_cast<float4*>(out + (size_t)j * 12);
    float v[12];
#pragma unroll
    for (int m = 0; m < 3; ++m)
#pragma unroll
      for (int c = 0; c < 4; ++c)
        v[m * 4 + c] = Pk.m[0 * 4 + m] * S.m[0 * 4 + c] + Pk.m[1 * 4 + m] * S.m[1 * 4 + c] + Pk.m[2 * 4 + m] * S.m[2 * 4 + c];
    d[0] = make_float4(v[0], v[1], v[2], v[3]);
    d[1] = make_float4(v[4], v[5], v[6], v[7]);
    d[2] = make_float4(v[8], v[9], v[10], v[11]);
  }
}

// torch.optim.Adam (single-tensor, no amsgrad / weight decay), same operation order.
__global__ void __launch_bounds__(kThreads)
k_adam(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
       size_t n, float beta1, float beta2, float omb1, float omb2, float eps, float step_size,
       float bc2_sqrt, const float* __restrict__ consts = nullptr) {
  if (consts) { step_size = __ldg(consts); bc2_sqrt = __ldg(consts + 1); }  // device step clock
  const size_t n4 = n / 4;
  for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n4; i += (size_t)gridDim.x * kThreads) {
    float4 pp = reinterpret_cast<float4*>(p)[i];
    const float4 gg = __ldg(reinterpret_cast<const float4*>(g) + i);
    float4 mm = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
#define FM_ADAM1(P, G, M, V)                                   \
    M = M + omb1 * (G - M);                                    \
    V = V * beta2 + omb2 * G * G;                              \
    P = P - step_size * (M / (sqrtf(V) / bc2_sqrt + eps));
    FM_ADAM1(pp.x, gg.x, mm.x, vv.x)
    FM_ADAM1(pp.y, gg.y, mm.y, vv.y)
    FM_ADAM1(pp.z, gg.z, mm.z, vv.z)
    FM_ADAM1(pp.w, gg.w, mm.w, vv.w)
    reinterpret_cast<float4*>(p)[i] = pp;
    reinterpret_cast<float4*>(m)[i] = mm;
    reinterpret_cast<float4*>(v)[i] = vv;
  }
  for (size_t i = n4 * 4 + (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads) {
    float pp = p[i], gg = g[i], mm = m[i], vv = v[i];
    FM_ADAM1(pp, gg, mm, vv)
    p[i] = pp; m[i] = mm; v[i] = vv;
  }
#undef FM_ADAM1
}

// ================================================================== tracking loss
// projection.py:255-298 (compute_track_flow) + loss_tracking.py:28-61, all segments in one
// launch.  Samples are packed per segment: sample(s, row, p) = seg.sample_start + row * n + p.
// seg table (int32 x 4 per segment): sample_start, rows f_s, points n_s, start_frame.
//
// The loss is sum / count with a count that depends on the PREDICTED positions, so the
// gradient scale is only known after a full pass.  Everything is therefore accumulated
// unscaled in ONE sweep over the (source, target, point) triples and scaled at the end:
//   k_track_src     work item = (segment, source row, half of its points): bilinear-sample xyz at the track
//                   location, lift to world space, loop over the segment's target rows:
//                   loss sum + valid count, the unscaled camera-space adjoint of the sampled
//                   point (stored per sample), source-frame K / pose-twist sums in registers,
//                   target-frame K / pose-twist sums by a recursive-halving warp reduction per
//                   row (10 values / 12 shuffles; 6 / 8 when all frames share their intrinsics).
//   k_track_apply   (backward) per sample: scale * adjoint -> bilinear scatter into the depth
//                   gradient (4 REDs).
//   k_track_finalize  scale the per-frame sums, expand twists to ambient 3x4 gradients.
// Pose gradients are left-perturbation twists (a = d/d omega, b = d/d v with delta R = [omega]x R,
// delta t = v); only the tangent part survives the rigid chain / Procrustes adjoint (SURVEY A.10).
constexpr int kTrackAcc = 10;   // per frame: dK (4), a (3), b (3)
constexpr int kTrackRec = 24;   // per-frame record in shared memory, see load_segment_frames

struct SegInfo { int sample_start, rows, n, start_frame; };

// Source-frame sharding (multi-GPU, SURVEY 8(e)): this call samples depth only at source frames
// [src_lo, src_hi); depth / g_depth point at frame depth_frame0.  Targets are never restricted.
struct TrackShard {
  int depth_frame0, src_lo, src_hi;
  __device__ __forceinline__ bool owns(int frame) const { return frame >= src_lo && frame < src_hi; }
};

__device__ __forceinline__ SegInfo load_seg(const int* seg, int s) {
  const int4 v = __ldg(reinterpret_cast<const int4*>(seg) + s);
  SegInfo i; i.sample_start = v.x; i.rows = v.y; i.n = v.z; i.start_frame = v.w;
  return i;
}

// Per-frame record: R (9, row-major, camera-to-world), t (3), c = -R^T t (3), fx fy cx cy ifx ify,
// 3 pad -- kTrackRec floats, 16-byte aligned, so that a warp reads a record with six broadcast
// 16-byte shared-memory loads (TrackRec).
__device__ __forceinline__ void load_segment_frames(float* sm, const float* ext, const float* k4,
                                                    const SegInfo& si) {
  for (int row = threadIdx.x; row < si.rows; row += blockDim.x) {
    const float* P = ext + (size_t)(si.start_frame + row) * 16;
    float* o = sm + row * kTrackRec;
    float v[kTrackRec];
    float* R = v;
    float* t = v + 9;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      R[i * 3 + 0] = __ldg(P + i * 4 + 0); R[i * 3 + 1] = __ldg(P + i * 4 + 1); R[i * 3 + 2] = __ldg(P + i * 4 + 2);
      t[i] = __ldg(P + i * 4 + 3);
    }
#pragma unroll
    for (int i = 0; i < 3; ++i)
      v[12 + i] = -(R[0 * 3 + i] * t[0] + R[1 * 3 + i] * t[1] + R[2 * 3 + i] * t[2]);
    const float4 k = __ldg(reinterpret_cast<const float4*>(k4) + si.start_frame + row);
    v[15] = k.x; v[16] = k.y; v[17] = k.z; v[18] = k.w; v[19] = 1.0f / k.x; v[20] = 1.0f / k.y;
    v[21] = v[22] = v[23] = 0.f;
#pragma unroll
    for (int i = 0; i < kTrackRec / 4; ++i)
      reinterpret_cast<float4*>(o)[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
  }
  __syncthreads();
}
static_assert(kTrackRec % 4 == 0, "frame records are read as float4");
struct TrackRec {
  float R[9], t[3], c[3];
  Cam k;
};
__device__ __forceinline__ TrackRec load_rec(const float* rec) {
  const float4* r4 = reinterpret_cast<const float4*>(rec);
  const float4 a = r4[0], b = r4[1], c = r4[2], d = r4[3], e = r4[4], f = r4[5];
  TrackRec r;
  r.R[0] = a.x; r.R[1] = a.y; r.R[2] = a.z; r.R[3] = a.w; r.R[4] = b.x; r.R[5] = b.y; r.R[6] = b.z; r.R[7] = b.w;
  r.R[8] = c.x; r.t[0] = c.y; r.t[1] = c.z; r.t[2] = c.w;
  r.c[0] = d.x; r.c[1] = d.y; r.c[2] = d.z;
  r.k.fx = d.w; r.k.fy = e.x; r.k.cx = e.y; r.k.cy = e.z; r.k.ifx = e.w; r.k.ify = f.x;
  return r;
}

// Warp sum of N per-lane values by recursive halving (N = 10: 12 shuffles instead of 50; N = 6:
// 8 instead of 30).  Afterwards lane l holds the total of value track_slot<N>(l).slot in v[0];
// `owner` marks one lane per value.
struct TrackSlot { int slot; bool owner; };
template <int N, int OFF>
struct SlotWalk {
  __device__ __forceinline__ static void run(int lane, int& pos, bool& ok) {
    if (N == 1) {
      SlotWalk<1, OFF / 2>::run(lane, pos, ok);
      ok = ok && (lane & OFF) == 0;
    } else {
      constexpr int HALF = (N + 1) / 2;
      SlotWalk<HALF, OFF / 2>::run(lane, pos, ok);  // position among the HALF survivors
      if (lane & OFF) pos += HALF;
      ok = ok && pos < N;
    }
  }
};
template <int N>
struct SlotWalk<N, 0> {
  __device__ __forceinline__ static void run(int, int& pos, bool& ok) { pos = 0; ok = true; }
};
template <int N>
__device__ __forceinline__ TrackSlot track_slot(int lane) {
  TrackSlot t;
  SlotWalk<N, 16>::run(lane, t.slot, t.owner);
  return t;
}
template <int N, int OFF>
__device__ __forceinline__ void halve_exchange(float* v, bool upper) {
  constexpr int HALF = (N + 1) / 2;
#pragma unroll
  for (int j = 0; j < HALF; ++j) {
    const float hi = (j + HALF < N) ? v[j + HALF] : 0.f;
    const float send = upper ? v[j] : hi;
    const float keep = upper ? hi : v[j];
    v[j] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
  }
}
template <int N, int OFF>
struct WarpSumN {
  __device__ __forceinline__ static void run(float* v, int lane) {
    if (N == 1) {
      v[0] += __shfl_xor_sync(0xffffffffu, v[0], OFF);
      WarpSumN<1, OFF / 2>::run(v, lane);
    } else {
      halve_exchange<N, OFF>(v, lane & OFF);
      WarpSumN<(N + 1) / 2, OFF / 2>::run(v, lane);
    }
  }
};
template <int N>
struct WarpSumN<N, 0> {
  __device__ __forceinline__ static void run(float*, int) {}
};
template <int N>
__device__ __forceinline__ float warp_sum_n(float* v, int lane) {
  WarpSumN<N, 16>::run(v, lane);
  return v[0];
}

// One sweep over the (source row, target row, point) triples.  Work item = one of kTrackParts
// contiguous point ranges of a (segment, source row): a persistent grid of kTrackThreads-thread blocks
// takes the items in order from a counter in the workspace, so the per-item costs -- staging the
// segment's frame records, the source-side block sums and the float64 atomics of the target-side
// sums -- are paid kTrackParts times per row.  Items cost about the same (rows x usable points); at the
// benchmark shape whole rows are 1146 items for 660 resident blocks, and halves of rows measured
// faster on H100 (a shorter last wave) than whole rows or thirds.
//
// Per item the range's usable source points (visible and inside [0,1)^2, recorded in `flag`) are compacted
// in point order into a shared list, at most kTrackListCap points per round.  The list is cut into warp
// passes of kTrackPass points, and warp w takes passes w, w + NW, ...: every warp of the block stays busy
// until the last kTrackPass points.  In a pass every lane keeps kTrackPPT source points in registers and
// evaluates their terms (lean_term of fm_pixel.cuh, the flow kernel's term) against each target row of
// the segment.  The source-side sums stay in registers for the whole item; the target-side sums of one
// target row (pose twist and K of the TARGET frame) belong to one frame for the whole warp, so the
// lane's points are added and the warp reduces them with warp_sum_n into its own [target row][10]
// slice of shared memory, which accumulates over the warp's passes and is folded into the per-frame
// accumulators once per item.
// SHARED_K: every frame has the same intrinsics (one focal length, or constants), so only the SUM
// over frames of the intrinsics gradient matters: the target-frame terms are then added to the
// thread's own (source-frame) accumulators and only the 6 pose values go through the reduction.
constexpr int kTrackThreads = 128;
#ifndef FM_TRACK_PPT
#define FM_TRACK_PPT 2  // source points per lane (1 or 2); 2 measured faster on H100
#endif
#ifndef FM_TRACK_BPS
#define FM_TRACK_BPS 5  // blocks per SM the register budget is sized for
#endif
#ifndef FM_TRACK_PARTS
#define FM_TRACK_PARTS 2  // work items per source row (halves of its points: a shorter last wave)
#endif
constexpr int kTrackParts = FM_TRACK_PARTS;
constexpr int kTrackPPT = FM_TRACK_PPT;
constexpr int kTrackPass = 32 * kTrackPPT;
constexpr int kTrackListCap = 2048;
static_assert(kTrackPPT == 1 || kTrackPPT == 2, "FM_TRACK_PPT must be 1 or 2");

// Dynamic shared memory of k_track_src: frame records, the warps' target-side slices, the point list.
__host__ __device__ constexpr size_t track_smem_bytes(int max_rows, int list_cap) {
  return ((size_t)max_rows * (kTrackRec + (kTrackThreads / 32) * kTrackAcc) + (size_t)list_cap) * sizeof(float);
}

template <bool SHARED_K>
__global__ void __launch_bounds__(kTrackThreads, FM_TRACK_BPS)
k_track_src(const float* __restrict__ depth, const float* __restrict__ k4, const float* __restrict__ ext,
            const int* __restrict__ seg, const float* __restrict__ txy,
            const unsigned char* __restrict__ tvis, int mapping, float delta, double* __restrict__ sums,
            unsigned char* __restrict__ flag, float* __restrict__ dq_out,
            double* __restrict__ trackacc, int* __restrict__ next_item, int num_items, int max_rows,
            int list_cap, int H, int W, TrackShard sh) {
  extern __shared__ float4 sm4[];
  float* sm = reinterpret_cast<float*>(sm4);
  constexpr int NW = kTrackThreads / 32;
  constexpr int NRED = SHARED_K ? 6 : kTrackAcc;
  constexpr int SLOT0 = kTrackAcc - NRED;  // twist values live in slots 4..9 either way
  __shared__ double red[kTrackAcc * NW];
  __shared__ int s_wbase[NW];
  __shared__ int s_item[2];
  float* s_tgt = sm + (size_t)max_rows * kTrackRec;  // [warp][target row][kTrackAcc]
  int* s_list = reinterpret_cast<int*>(s_tgt + (size_t)NW * max_rows * kTrackAcc);
  const GridDims grid = make_grid(H, W);
  const RobustCfg rc = make_robust(mapping, delta, H, W);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const TrackSlot slot = track_slot<NRED>(lane);
  const float2* xy2 = reinterpret_cast<const float2*>(txy);
  for (int it = 0;; ++it) {
    // s_item alternates, so the next item can be fetched while slow threads still read this one
    if (threadIdx.x == 0) s_item[it & 1] = atomicAdd(next_item, 1);
    __syncthreads();
    const int item = s_item[it & 1];
    if (item >= num_items) break;
    const int part = item % kTrackParts, srow = item / kTrackParts;
    const SegInfo si = load_seg(seg, srow / max_rows);
    const int row = srow % max_rows;
    if (row >= si.rows || !sh.owns(si.start_frame + row)) continue;
    load_segment_frames(sm, ext, k4, si);
    float* tgt = s_tgt + (size_t)warp * si.rows * kTrackAcc;
    for (int i = lane; i < si.rows * kTrackAcc; i += 32) tgt[i] = 0.f;
    __syncwarp();
    const int frame = si.start_frame + row;
    const float* D = depth + (size_t)(frame - sh.depth_frame0) * H * W;
    const float* rsrec = sm + row * kTrackRec;
    const size_t row0 = (size_t)si.sample_start + (size_t)row * si.n;
    const float2* seg_xy = xy2 + si.sample_start;
    const unsigned char* seg_vis = tvis + si.sample_start;
    float acc[kTrackAcc], lc[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < kTrackAcc; ++i) acc[i] = 0.f;
    const int p_end = (int)((long long)si.n * (part + 1) / kTrackParts);
    for (int base = (int)((long long)si.n * part / kTrackParts); base < p_end; base += list_cap) {
      // compaction in point order: warp w scans [lo, hi), counts, then writes at its offset
      const int len = min(list_cap, p_end - base);
      const int per = (len + NW * 32 - 1) / (NW * 32) * 32;
      const int lo = base + warp * per, hi = min(base + len, lo + per);
      int cnt = 0;
      for (int p0 = lo; p0 < hi; p0 += 32) {
        const int p = p0 + lane;
        bool ok = false;
        if (p < hi) {
          const size_t sidx = row0 + p;
          const float2 sxy = __ldg(xy2 + sidx);
          ok = tvis[sidx] && in_unit_square(sxy.x, sxy.y);
          flag[sidx] = ok ? 1 : 0;
        }
        cnt += __popc(__ballot_sync(0xffffffffu, ok));
      }
      if (lane == 0) s_wbase[warp] = cnt;
      __syncthreads();
      int wb = 0, total = 0;
#pragma unroll
      for (int w = 0; w < NW; ++w) {
        const int c = s_wbase[w];
        if (w < warp) wb += c;
        total += c;
      }
      for (int p0 = lo; p0 < hi; p0 += 32) {
        const int p = p0 + lane;
        const bool ok = p < hi && flag[row0 + p];  // this lane's own store above
        const unsigned m = __ballot_sync(0xffffffffu, ok);
        if (ok) s_list[wb + __popc(m & ((1u << lane) - 1u))] = p;
        wb += __popc(m);
      }
      __syncthreads();
      const int npass = (total + kTrackPass - 1) / kTrackPass;
      for (int ps = warp; ps < npass; ps += NW) {  // warp-uniform: the shuffles below need all 32 lanes
        const int pb = ps * kTrackPass + lane;
        // lift the pass's source points to world space
        float Xw[kTrackPPT][3];
        int ix[kTrackPPT];  // sample offset within the segment: row ft of point p is p + ft * n
        {
          const TrackRec rs = load_rec(rsrec);
#pragma unroll
          for (int j = 0; j < kTrackPPT; ++j) {
            Xw[j][0] = Xw[j][1] = Xw[j][2] = 0.f;
            ix[j] = -1;
            if (pb + 32 * j < total) {
              const int p = s_list[pb + 32 * j];
              ix[j] = p;
              const float2 sxy = __ldg(xy2 + row0 + p);
              const Taps t = bilinear_taps(sxy.x, sxy.y, grid);
              float q[3];
              sample_surface(t, grid, rs.k, [D](int o) { return __ldg(D + o); }, q[0], q[1], q[2]);
#pragma unroll
              for (int i = 0; i < 3; ++i)
                Xw[j][i] = fm_fma(rs.R[i * 3 + 0], q[0], fm_fma(rs.R[i * 3 + 1], q[1], fm_fma(rs.R[i * 3 + 2], q[2], rs.t[i])));
            }
          }
        }
        float G[kTrackPPT][3];
#pragma unroll
        for (int j = 0; j < kTrackPPT; ++j) G[j][0] = G[j][1] = G[j][2] = 0.f;
        // the next target row's visibility / position is fetched while the current one is processed
        unsigned char vn[kTrackPPT];
        float2 gn[kTrackPPT];
#pragma unroll
        for (int j = 0; j < kTrackPPT; ++j) {
          vn[j] = ix[j] >= 0 ? seg_vis[ix[j]] : 0;
          gn[j] = ix[j] >= 0 ? __ldg(seg_xy + ix[j]) : make_float2(0.f, 0.f);
        }
        for (int ft = 0; ft < si.rows; ++ft) {
          unsigned char v[kTrackPPT];
          float2 g[kTrackPPT];
          bool any = false;
#pragma unroll
          for (int j = 0; j < kTrackPPT; ++j) {
            v[j] = vn[j]; g[j] = gn[j];
            any |= v[j] != 0;
            if (ft + 1 < si.rows && ix[j] >= 0) {
              ix[j] += si.n;
              vn[j] = seg_vis[ix[j]];
              gn[j] = __ldg(seg_xy + ix[j]);
            }
          }
          float c[NRED];
#pragma unroll
          for (int i = 0; i < NRED; ++i) c[i] = 0.f;
          bool ok = false;
          if (any) {
            const TrackRec r = load_rec(sm + ft * kTrackRec);
#pragma unroll
            for (int j = 0; j < kTrackPPT; ++j) {
              // Y = R_t^T Xw + c_t
              const float dir0 = fm_fma(r.R[0], Xw[j][0], fm_fma(r.R[3], Xw[j][1], __fmul_rn(r.R[6], Xw[j][2])));
              const float dir1 = fm_fma(r.R[1], Xw[j][0], fm_fma(r.R[4], Xw[j][1], __fmul_rn(r.R[7], Xw[j][2])));
              const float dir2 = fm_fma(r.R[2], Xw[j][0], fm_fma(r.R[5], Xw[j][1], __fmul_rn(r.R[8], Xw[j][2])));
              const LeanTerm lt = lean_term(1.0f, dir0, dir1, dir2, r.c[0], r.c[1], r.c[2], r.k, g[j].x, g[j].y, 0.f,
                                            0.f, 1.0f, rc);
              // projection.py:294-296: the PREDICTED target position decides
              const bool o = v[j] && in_unit_square(lt.uvx, lt.uvy);
              ok |= o;
              // an invalid point contributes nothing (selects, not products: its adjoint may hold inf / nan;
              // the camera-space point P itself is always finite)
              const float d0 = o ? lt.d0 : 0.f, d1 = o ? lt.d1 : 0.f, d2 = o ? lt.d2 : 0.f;
              lc[0] = __fadd_rn(lc[0], o ? lt.loss : 0.f);
              lc[1] = __fadd_rn(lc[1], o ? 1.f : 0.f);
              // world-space gradient g = R_t dY
              const float g0 = fm_fma(r.R[0], d0, fm_fma(r.R[1], d1, __fmul_rn(r.R[2], d2)));
              const float g1 = fm_fma(r.R[3], d0, fm_fma(r.R[4], d1, __fmul_rn(r.R[5], d2)));
              const float g2 = fm_fma(r.R[6], d0, fm_fma(r.R[7], d1, __fmul_rn(r.R[8], d2)));
              G[j][0] = __fadd_rn(G[j][0], g0); G[j][1] = __fadd_rn(G[j][1], g1); G[j][2] = __fadd_rn(G[j][2], g2);
              // target-frame K gradient: duv = d (P_z + eps) / f and uv - c = f P / (P_z + eps)
              const float ex = __fmul_rn(d0, r.k.ifx), ey = __fmul_rn(d1, r.k.ify);
              if (SHARED_K) {  // straight into the thread's own intrinsics sums
                acc[0] = fm_fma(ex, lt.P0, acc[0]); acc[1] = fm_fma(ey, lt.P1, acc[1]);
                acc[2] = fm_fma(ex, lt.P2, acc[2]); acc[3] = fm_fma(ey, lt.P2, acc[3]);
              } else {
                c[0] = __fadd_rn(c[0], __fmul_rn(ex, lt.P0)); c[1] = __fadd_rn(c[1], __fmul_rn(ey, lt.P1));
                c[2] = __fadd_rn(c[2], __fmul_rn(ex, lt.P2)); c[3] = __fadd_rn(c[3], __fmul_rn(ey, lt.P2));
              }
              // twist of the target pose: (Xw - t) x g, -g (an invalid point has g = 0)
              const float e0 = __fsub_rn(Xw[j][0], r.t[0]), e1 = __fsub_rn(Xw[j][1], r.t[1]);
              const float e2 = __fsub_rn(Xw[j][2], r.t[2]);
              float* tw = c + (SHARED_K ? 0 : 4);
              tw[0] = __fadd_rn(tw[0], fm_fma(e2, g1, -__fmul_rn(e1, g2)));
              tw[1] = __fadd_rn(tw[1], fm_fma(e0, g2, -__fmul_rn(e2, g0)));
              tw[2] = __fadd_rn(tw[2], fm_fma(e1, g0, -__fmul_rn(e0, g1)));
              tw[3] = __fsub_rn(tw[3], g0); tw[4] = __fsub_rn(tw[4], g1); tw[5] = __fsub_rn(tw[5], g2);
            }
          }
          if (__ballot_sync(0xffffffffu, ok)) {
            const float total_c = warp_sum_n<NRED>(c, lane);
            if (slot.owner) tgt[ft * kTrackAcc + SLOT0 + slot.slot] += total_c;
          }
        }
        // camera-space adjoint of the sampled points (unscaled), source K / twist sums; the sampled
        // point is evaluated again instead of being kept in registers through the target loop
        const TrackRec rs = load_rec(rsrec);
#pragma unroll
        for (int j = 0; j < kTrackPPT; ++j) {
          if (pb + 32 * j >= total) continue;
          const size_t sidx = row0 + s_list[pb + 32 * j];
          const float2 sxy = __ldg(xy2 + sidx);
          const Taps t = bilinear_taps(sxy.x, sxy.y, grid);
          float q[3];
          sample_surface(t, grid, rs.k, [D](int o) { return __ldg(D + o); }, q[0], q[1], q[2]);
          const float G0 = G[j][0], G1 = G[j][1], G2 = G[j][2];
          const float dq0 = fm_fma(rs.R[0], G0, fm_fma(rs.R[3], G1, rs.R[6] * G2));
          const float dq1 = fm_fma(rs.R[1], G0, fm_fma(rs.R[4], G1, rs.R[7] * G2));
          const float dq2 = fm_fma(rs.R[2], G0, fm_fma(rs.R[5], G1, rs.R[8] * G2));
          dq_out[sidx * 3 + 0] = dq0; dq_out[sidx * 3 + 1] = dq1; dq_out[sidx * 3 + 2] = dq2;
          const float e0 = dq0 * rs.k.ifx, e1 = dq1 * rs.k.ify;
          acc[0] -= e0 * q[0]; acc[1] -= e1 * q[1]; acc[2] -= e0 * q[2]; acc[3] -= e1 * q[2];
          const float c0 = Xw[j][0] - rs.t[0], c1 = Xw[j][1] - rs.t[1], c2 = Xw[j][2] - rs.t[2];
          acc[4] += c1 * G2 - c2 * G1;
          acc[5] += c2 * G0 - c0 * G2;
          acc[6] += c0 * G1 - c1 * G0;
          acc[7] += G0; acc[8] += G1; acc[9] += G2;
        }
      }
      __syncthreads();  // s_list / s_wbase are rewritten by the next round
    }
    block_accumulate<2, kTrackThreads>(lc, sums, red);
    block_accumulate<kTrackAcc, kTrackThreads>(acc, trackacc + (size_t)frame * kTrackAcc, red);
    // fold the warps' target-side slices into the per-frame accumulators (block_accumulate ended
    // with a barrier, so every slice is complete)
    for (int i = threadIdx.x; i < si.rows * kTrackAcc; i += kTrackThreads) {
      if (SHARED_K && i % kTrackAcc < 4) continue;  // those slots are not written in this mode
      double t = 0.0;
#pragma unroll
      for (int w = 0; w < NW; ++w) t += (double)s_tgt[(size_t)w * si.rows * kTrackAcc + i];
      if (t != 0.0) atomicAdd(trackacc + (size_t)si.start_frame * kTrackAcc + i, t);
    }
  }
}

__device__ __forceinline__ double track_scale(const double* sums, float loss_weight, const float* go) {
  double cnt = sums[1];
  if (cnt == 0.0) cnt = 1.0;  // loss_tracking.py:61 "valid_sum or 1"
  return (double)loss_weight * (go ? (double)*go : 1.0) / cnt;
}

__global__ void k_track_loss(const double* __restrict__ sums, float loss_weight, float* __restrict__ loss) {
  *loss = (float)(track_scale(sums, loss_weight, nullptr) * sums[0]);
}

// scale * (stored camera-space adjoint) -> the four depth taps of every source sample.
__global__ void __launch_bounds__(kThreads)
k_track_apply(const float* __restrict__ k4, const int* __restrict__ seg, const float* __restrict__ txy,
              const unsigned char* __restrict__ flag, const float* __restrict__ dq,
              const double* __restrict__ sums, float loss_weight, const float* __restrict__ go,
              float* __restrict__ g_depth, int H, int W, TrackShard sh) {
  const SegInfo si = load_seg(seg, blockIdx.z);
  const int row = blockIdx.y;
  const int p = blockIdx.x * kThreads + threadIdx.x;
  if (row >= si.rows || p >= si.n || !sh.owns(si.start_frame + row)) return;
  const size_t sidx = (size_t)si.sample_start + (size_t)row * si.n + p;
  if (!flag[sidx]) return;
  const float scale = (float)track_scale(sums, loss_weight, go);
  const int frame = si.start_frame + row;
  const GridDims grid = make_grid(H, W);
  const Cam ks = make_cam(load_k4(k4, frame));
  const float2 sxy = __ldg(reinterpret_cast<const float2*>(txy) + sidx);
  const Taps t = bilinear_taps(sxy.x, sxy.y, grid);
  const float dq0 = scale * dq[sidx * 3 + 0], dq1 = scale * dq[sidx * 3 + 1], dq2 = scale * dq[sidx * 3 + 2];
  float rx0, ry0, rx1, ry1;
  tap_rays(t, grid, ks, rx0, ry0, rx1, ry1);
  float* gd = g_depth + (size_t)(frame - sh.depth_frame0) * H * W;
  red_add(gd + t.y0 * W + t.x0, t.w00 * (dq0 * rx0 + dq1 * ry0 + dq2));
  red_add(gd + t.y0 * W + t.x1, t.w01 * (dq0 * rx1 + dq1 * ry0 + dq2));
  red_add(gd + t.y1 * W + t.x0, t.w10 * (dq0 * rx0 + dq1 * ry1 + dq2));
  red_add(gd + t.y1 * W + t.x1, t.w11 * (dq0 * rx1 + dq1 * ry1 + dq2));
}

__global__ void k_track_finalize(const double* __restrict__ trackacc, const double* __restrict__ sums,
                                 float loss_weight, const float* __restrict__ go,
                                 const float* __restrict__ ext, float* __restrict__ g_ext,
                                 float* __restrict__ g_k4, int F) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const double sc = track_scale(sums, loss_weight, go);
  const double* a = trackacc + (size_t)f * kTrackAcc;
  for (int k = 0; k < 4; ++k) g_k4[(size_t)f * 4 + k] = (float)(sc * a[k]);
  const float* P = ext + (size_t)f * 16;
  const double w0 = 0.5 * sc * a[4], w1 = 0.5 * sc * a[5], w2 = 0.5 * sc * a[6];
  float* o = g_ext + (size_t)f * 16;
  for (int c = 0; c < 3; ++c) {  // G_R = 1/2 [a]x R
    const double r0 = P[0 * 4 + c], r1 = P[1 * 4 + c], r2 = P[2 * 4 + c];
    o[0 * 4 + c] = (float)(-w2 * r1 + w1 * r2);
    o[1 * 4 + c] = (float)(w2 * r0 - w0 * r2);
    o[2 * 4 + c] = (float)(-w1 * r0 + w0 * r1);
  }
  o[3] = (float)(sc * a[7]); o[7] = (float)(sc * a[8]); o[11] = (float)(sc * a[9]);
  o[12] = o[13] = o[14] = o[15] = 0.f;
}

// ================================================================== focal-length sweep
// intrinsics_softmin.py:84-131: for every candidate focal length, Procrustes on the first
// frame pair at the selected points (k_moments / k_solve with a broadcast PairLayout), then
// the backward-flow error  err_n = sum_points sum_xy | (uv - xy - flow) * w |.
// k_sweep<false>: err per candidate.  k_sweep<true>: given d loss / d err_n, the direct
// depth / weight gradients (REDs) and the pose-gradient sums per candidate.
constexpr int kSweepAcc = 80;  // doubles reserved per virtual item inside Workspace::flowacc

// The candidates of the sweep differ only by S_n = diag(fx_0/fx_n, fy_0/fy_n, 1) applied to the
// points: p_n = S_n p_0, q_n = S_n q_0 (same principal point, bilinear sampling is linear in the
// rays).  So the 16 moment sums are accumulated ONCE (candidate 0) and scaled per candidate, and
// the per-point adjoints of all candidates collapse into ONE PairAdjoint in candidate-0
// coordinates:  A = sum S C_n S,  pb = sum S (pb_n - C_n^T qbar_n),  qb = sum S (qb_n - C_n pbar_n),
// wconst = sum (qbar_n^T C_n pbar_n - pb_n . pbar_n - qb_n . qbar_n),  centroids 0.
__global__ void k_sweep_base_k4(const float* __restrict__ cand_k4, float* __restrict__ base_k4, int B, int n) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * 8) return;
  const int b = t >> 3, e = t & 7;
  base_k4[t] = cand_k4[(size_t)b * n * 8 + e];  // frames 0/1 of candidate 0
}

__global__ void k_sweep_scale_solve(const double* __restrict__ base_moments, const float* __restrict__ base_zshift,
                                    const float* __restrict__ cand_k4, float* __restrict__ rt,
                                    PairState* __restrict__ state, int B, int n) {
  const int item = blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= B * n) return;
  const int b = item / n;
  const double z0 = (double)base_zshift[b];  // the shift of the real pair's moment pass (along z: S_n keeps it)
  const double sx = (double)cand_k4[(size_t)b * n * 8 + 0] / (double)cand_k4[(size_t)item * 8 + 0];
  const double sy = (double)cand_k4[(size_t)b * n * 8 + 1] / (double)cand_k4[(size_t)item * 8 + 1];
  const double sc[3] = {sx, sy, 1.0};
  double m[kNumMoments];
  const double* bm = base_moments + (size_t)b * kNumMoments;
  m[0] = bm[0];
  for (int i = 0; i < 3; ++i) { m[1 + i] = bm[1 + i] * sc[i]; m[4 + i] = bm[4 + i] * sc[i]; }
  for (int a = 0; a < 3; ++a)
    for (int c = 0; c < 3; ++c) m[7 + a * 3 + c] = bm[7 + a * 3 + c] * sc[a] * sc[c];
  const double shift[3] = {0.0, 0.0, z0};
  PairState st;
  float out[12];
  procrustes_solve(m, shift, out, st);
  for (int k = 0; k < 12; ++k) rt[(size_t)item * 12 + k] = out[k];
  state[item] = st;
}

__global__ void k_sweep_aggregate(const PairAdjoint* __restrict__ adj, const float* __restrict__ cand_k4,
                                  PairAdjoint* __restrict__ out, int B, int n) {
  const int b = blockIdx.x, lane = threadIdx.x;  // one warp per batch element, lanes stride the candidates
  double acc[16];  // A (9), pb (3), qb (3), wconst
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = 0.0;
  for (int c = lane; c < n; c += 32) {
    const int item = b * n + c;
    const PairAdjoint a = adj[item];
    const double s[3] = {(double)cand_k4[(size_t)b * n * 8 + 0] / (double)cand_k4[(size_t)item * 8 + 0],
                         (double)cand_k4[(size_t)b * n * 8 + 1] / (double)cand_k4[(size_t)item * 8 + 1], 1.0};
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      double cq = 0.0, cp = 0.0;  // (C^T qbar)_r, (C pbar)_r
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        acc[r * 3 + k] += s[r] * (double)a.cbar[r * 3 + k] * s[k];
        cq += (double)a.cbar[k * 3 + r] * (double)a.qbar[k];
        cp += (double)a.cbar[r * 3 + k] * (double)a.pbar[k];
      }
      acc[9 + r] += s[r] * ((double)a.pb[r] - cq);
      acc[12 + r] += s[r] * ((double)a.qb[r] - cp);
      acc[15] += (double)a.qbar[r] * cp - (double)a.pb[r] * (double)a.pbar[r] - (double)a.qb[r] * (double)a.qbar[r];
    }
  }
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = warp_sum(acc[i]);
  if (lane == 0) {
    PairAdjoint o;
    for (int i = 0; i < 9; ++i) o.cbar[i] = (float)acc[i];
    for (int i = 0; i < 3; ++i) {
      o.pb[i] = (float)acc[9 + i]; o.qb[i] = (float)acc[12 + i]; o.pbar[i] = 0.f; o.qbar[i] = 0.f;
      o.shift[i] = adj[b * n].shift[i];
    }
    o.wconst = (float)acc[15];
    out[b] = o;
  }
}

template <bool BWD>
__global__ void __launch_bounds__(kThreads)
k_sweep(const float* __restrict__ depth, const float* __restrict__ k4, const float* __restrict__ rt,
        const float* __restrict__ bflow, const float* __restrict__ weights, float wsens,
        const int64_t* __restrict__ indices, int num_indices, const float* __restrict__ g_err,
        double* __restrict__ acc_out, float* __restrict__ g_depth, float* __restrict__ g_weights,
        PairLayout lay, int H, int W) {
  __shared__ double smem[12 * (kThreads / 32)];
  const int item = blockIdx.y;
  const int N = H * W;
  const PairAddr pa = pair_addr(lay, item, N);  // F == 2: one pair per item
  const Cam ka = make_cam(load_k4(k4, pa.k4_frame_a));
  const Cam kb = make_cam(load_k4(k4, pa.k4_frame_a + 1));
  const Rt T = load_rt(rt, item);
  const GridDims grid = make_grid(H, W);
  const float* d1 = depth + pa.depth_a + N;
  const float* fl = bflow + pa.flow;
  const float* wt = weights ? weights + pa.weight : nullptr;
  float* gd1 = BWD ? g_depth + pa.depth_a + N : nullptr;
  float* gw = (BWD && g_weights) ? g_weights + pa.weight : nullptr;
  const float ge = BWD ? __ldg(g_err + item) : 0.f;
  float acc[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) acc[i] = 0.f;
  for (int t = blockIdx.x * kThreads + threadIdx.x; t < num_indices; t += gridDim.x * kThreads) {
    const int j = (int)indices[t];
    const int r = j / W, c = j - r * W;
    const float x = pix_coord(c, grid.Wf, grid.invW), y = pix_coord(r, grid.Hf, grid.invH);
    const float D = __ldg(d1 + j);
    float rx, ry;
    ray_of(x, y, kb, rx, ry);
    const float p0 = D * rx, p1 = D * ry, p2 = D;
    // The softmin over the candidates' errors amplifies their rounding: the transform and the
    // projection are rounded per operation, as the reference's float32 ops are (no FMA contraction).
    const float X0 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T.r[0], p0), __fmul_rn(T.r[1], p1)), __fmul_rn(T.r[2], p2)), T.t[0]);
    const float X1 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T.r[3], p0), __fmul_rn(T.r[4], p1)), __fmul_rn(T.r[5], p2)), T.t[1]);
    const float X2 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T.r[6], p0), __fmul_rn(T.r[7], p1)), __fmul_rn(T.r[8], p2)), T.t[2]);
    Proj pr = project_point(X0, X1, X2, ka);
    pr.uvx = __fadd_rn(__fmul_rn(ka.fx, pr.u[0]), __fmul_rn(ka.cx, pr.u[2]));
    pr.uvy = __fadd_rn(__fmul_rn(ka.fy, pr.u[1]), __fmul_rn(ka.cy, pr.u[2]));
    const float ex = (pr.uvx - x) - __ldg(fl + 2 * j), ey = (pr.uvy - y) - __ldg(fl + 2 * j + 1);
    const float w = wt ? weight_of(__ldg(wt + j), wsens) : 1.f;
    const float a = ex * w, b = ey * w;
    if (!BWD) {
      acc[0] += fabsf(a) + fabsf(b);
    } else {
      const float da = (a > 0.f ? ge : (a < 0.f ? -ge : 0.f)), db = (b > 0.f ? ge : (b < 0.f ? -ge : 0.f));
      float dX0, dX1, dX2, u0 = 0, u1 = 0, u2 = 0, u3 = 0;
      project_point_adj(pr, X0, X1, X2, ka, da * w, db * w, dX0, dX1, dX2, u0, u1, u2, u3);
      acc[0] += dX0 * p0; acc[1] += dX0 * p1; acc[2] += dX0 * p2; acc[3] += dX0;
      acc[4] += dX1 * p0; acc[5] += dX1 * p1; acc[6] += dX1 * p2; acc[7] += dX1;
      acc[8] += dX2 * p0; acc[9] += dX2 * p1; acc[10] += dX2 * p2; acc[11] += dX2;
      const float dp0 = T.r[0] * dX0 + T.r[3] * dX1 + T.r[6] * dX2;
      const float dp1 = T.r[1] * dX0 + T.r[4] * dX1 + T.r[7] * dX2;
      const float dp2 = T.r[2] * dX0 + T.r[5] * dX1 + T.r[8] * dX2;
      red_add(gd1 + j, dp0 * rx + dp1 * ry + dp2);
      if (gw) {
        float dw = da * ex + db * ey;
        if (wsens != 0.f) dw *= wsens * w * (1.0f - w);
        red_add(gw + j, dw);
      }
    }
  }
  if (!BWD) block_accumulate<1>(acc, acc_out + (size_t)item * kSweepAcc, smem);
  else block_accumulate<12>(acc, acc_out + (size_t)item * kSweepAcc + 1, smem);
}

__global__ void k_sweep_out(const double* __restrict__ acc, float* __restrict__ out, int items, int off,
                            int count) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= items * count) return;
  const int item = t / count, k = t - item * count;
  out[t] = (float)acc[(size_t)item * kSweepAcc + off + k];
}

// softmin((err - min) * 10) over the candidates -> focal estimate (intrinsics_softmin.py:126-139),
// one block per batch element.  Writes the weights and f_hat = sum_n softmin_n f_n.
__global__ void k_softmin_focal(const float* __restrict__ err, const float* __restrict__ cand_f, int n,
                                float* __restrict__ sm_out, float* __restrict__ f_hat) {
  const int b = blockIdx.x, lane = threadIdx.x;  // one warp per batch element
  float mn = 3.0e38f;
  for (int i = lane; i < n; i += 32) mn = fminf(mn, err[b * n + i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  double z = 0.0;
  for (int i = lane; i < n; i += 32) z += exp(-(double)((err[b * n + i] - mn) * 10.0f));
  z = warp_sum(z);
  double f = 0.0;
  for (int i = lane; i < n; i += 32) {
    const double sm = exp(-(double)((err[b * n + i] - mn) * 10.0f)) / z;
    sm_out[b * n + i] = (float)sm;
    f += sm * (double)cand_f[i];
  }
  f = warp_sum(f);
  if (lane == 0) f_hat[b] = (float)f;
}

// d f_hat / d err_m = -10 sm_m (f_m - f_hat)   (softmin is shift invariant: the min drops out)
__global__ void k_softmin_focal_bwd(const float* __restrict__ sm, const float* __restrict__ cand_f,
                                    const float* __restrict__ f_hat, const float* __restrict__ g_f_hat, int n,
                                    int B, float* __restrict__ g_err) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * n) return;
  const int b = t / n, i = t - b * n;
  g_err[t] = -10.0f * sm[t] * (cand_f[i] - f_hat[b]) * g_f_hat[b];
}

// ================================================================== standalone API kernels
// flowmap/model/procrustes.py:7-51 on explicit point sets (*batch, n, 3): moments -> solve ->
// [R|t]; backward: closed-form per-point adjoints.  One item per blockIdx.y.
//
// Conditioning shift of an item: the weighted mean of (p + q) / 2 over up to kShiftSamples evenly
// spaced points (unweighted if their weights sum to zero), subtracted from p and q before the
// moments, as the image path subtracts its z0.  One block per item.
__global__ void __launch_bounds__(kThreads)
k_points_shift(const float* __restrict__ p, const float* __restrict__ q, const float* __restrict__ w,
               float* __restrict__ shift, int n) {
  __shared__ double smem[7][kThreads / 32];
  const int item = blockIdx.x;
  const int cnt = n < kShiftSamples ? n : kShiftSamples;
  double s[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};  // w c (3), w, c (3)
  for (int i = threadIdx.x; i < cnt; i += kThreads) {
    const long long j = (long long)i * n / cnt;
    const size_t o = ((size_t)item * n + j) * 3;
    const double wj = (double)__ldg(w + (size_t)item * n + j);
    for (int c = 0; c < 3; ++c) {
      const double m = 0.5 * ((double)__ldg(p + o + c) + (double)__ldg(q + o + c));
      s[c] += wj * m; s[4 + c] += m;
    }
    s[3] += wj;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    const double v = warp_sum(s[k]);
    if (lane == 0) smem[k][warp] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int k = 0; k < 7; ++k)
      for (int v = 0; v < kThreads / 32; ++v) t[k] += smem[k][v];
    for (int c = 0; c < 3; ++c) shift[item * 3 + c] = shift_from_sums(t[c], t[3], t[4 + c], cnt);
  }
}

__global__ void __launch_bounds__(kThreads)
k_points_moments(const float* __restrict__ p, const float* __restrict__ q, const float* __restrict__ w,
                 const float* __restrict__ shift, double* __restrict__ moments, int n) {
  __shared__ double smem[kNumMoments * (kThreads / 32)];
  const int item = blockIdx.y;
  const float c0 = __ldg(shift + item * 3), c1 = __ldg(shift + item * 3 + 1), c2 = __ldg(shift + item * 3 + 2);
  float acc[kNumMoments];
#pragma unroll
  for (int i = 0; i < kNumMoments; ++i) acc[i] = 0.f;
  for (int j = blockIdx.x * kThreads + threadIdx.x; j < n; j += gridDim.x * kThreads) {
    const size_t o = ((size_t)item * n + j) * 3;
    const float pp[3] = {__ldg(p + o) - c0, __ldg(p + o + 1) - c1, __ldg(p + o + 2) - c2};
    const float qq[3] = {__ldg(q + o) - c0, __ldg(q + o + 1) - c1, __ldg(q + o + 2) - c2};
    moments_add(acc, __ldg(w + (size_t)item * n + j), pp, qq);
  }
  block_accumulate<kNumMoments>(acc, moments + (size_t)item * kNumMoments, smem);
}

__global__ void k_points_solve(const double* __restrict__ moments, const float* __restrict__ pshift,
                               float* __restrict__ rt, PairState* __restrict__ state, int items) {
  const int item = blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= items) return;
  double m[kNumMoments];
  for (int k = 0; k < kNumMoments; ++k) m[k] = moments[(size_t)item * kNumMoments + k];
  const double shift[3] = {(double)pshift[item * 3], (double)pshift[item * 3 + 1], (double)pshift[item * 3 + 2]};
  PairState st;
  float out[12];
  procrustes_solve(m, shift, out, st);
  for (int k = 0; k < 12; ++k) rt[(size_t)item * 12 + k] = out[k];
  state[item] = st;
}

__global__ void __launch_bounds__(kThreads)
k_points_distribute(const float* __restrict__ p, const float* __restrict__ q, const float* __restrict__ w,
                    const PairAdjoint* __restrict__ adj, float* __restrict__ gp, float* __restrict__ gq,
                    float* __restrict__ gw, int n) {
  const int item = blockIdx.y;
  const PairAdjoint ad = adj[item];
  for (int j = blockIdx.x * kThreads + threadIdx.x; j < n; j += gridDim.x * kThreads) {
    const size_t o = ((size_t)item * n + j) * 3;
    // the shifted points of the moment pass minus their (shifted) centroids
    const float dp[3] = {(__ldg(p + o) - ad.shift[0]) - ad.pbar[0], (__ldg(p + o + 1) - ad.shift[1]) - ad.pbar[1],
                         (__ldg(p + o + 2) - ad.shift[2]) - ad.pbar[2]};
    const float dq[3] = {(__ldg(q + o) - ad.shift[0]) - ad.qbar[0], (__ldg(q + o + 1) - ad.shift[1]) - ad.qbar[1],
                         (__ldg(q + o + 2) - ad.shift[2]) - ad.qbar[2]};
    float wb, pb[3], qb[3];
    point_adjoint(ad, __ldg(w + (size_t)item * n + j), dp, dq, wb, pb, qb);
    gp[o] = pb[0]; gp[o + 1] = pb[1]; gp[o + 2] = pb[2];
    gq[o] = qb[0]; gq[o + 1] = qb[1]; gq[o + 2] = qb[2];
    gw[(size_t)item * n + j] = wb;
  }
}

// flowmap/model/projection.py:76-90 on explicit coordinates: out = z * K^-1 [x y 1]^T.
// xy: (xy_items, n, 2) with xy_items == items or 1 (shared grid).
__global__ void k_unproject_points(const float* __restrict__ xy, const float* __restrict__ z,
                                   const float* __restrict__ k4, float* __restrict__ out, int n, int xy_shared) {
  const int item = blockIdx.y;
  const Cam k = make_cam(load_k4(k4, item));
  const float* c = xy + (xy_shared ? 0 : (size_t)item * n * 2);
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    float rx, ry;
    ray_of(__ldg(c + 2 * j), __ldg(c + 2 * j + 1), k, rx, ry);
    const float d = __ldg(z + (size_t)item * n + j);
    float* o = out + ((size_t)item * n + j) * 3;
    o[0] = d * rx; o[1] = d * ry; o[2] = d;
  }
}

__global__ void __launch_bounds__(kThreads)
k_unproject_points_bwd(const float* __restrict__ xy, const float* __restrict__ z, const float* __restrict__ k4,
                       const float* __restrict__ g_out, float* __restrict__ g_z, double* __restrict__ g_k,
                       int n, int xy_shared) {
  __shared__ double smem[4 * (kThreads / 32)];
  const int item = blockIdx.y;
  const Cam k = make_cam(load_k4(k4, item));
  const float* c = xy + (xy_shared ? 0 : (size_t)item * n * 2);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    float rx, ry;
    ray_of(__ldg(c + 2 * j), __ldg(c + 2 * j + 1), k, rx, ry);
    const float d = __ldg(z + (size_t)item * n + j);
    const float* g = g_out + ((size_t)item * n + j) * 3;
    const float g0 = g[0], g1 = g[1], g2 = g[2];
    g_z[(size_t)item * n + j] = g0 * rx + g1 * ry + g2;
    acc[0] -= g0 * d * rx * k.ifx;
    acc[1] -= g1 * d * ry * k.ify;
    acc[2] -= g0 * d * k.ifx;
    acc[3] -= g1 * d * k.ify;
  }
  block_accumulate<4>(acc, g_k + (size_t)item * 4, smem);
}

// n distinct pseudo-random indices in [0, N): the first n outputs of a keyed random PERMUTATION
// of [0, N) (4-round Feistel network on the next even power of two, cycle-walking back into
// range).  Stands in for `torch.randperm(N)[:n]` (intrinsics_softmin.py:90) without sorting N
// keys every step; like randperm it yields a uniform sample without replacement in random order.
__device__ __forceinline__ unsigned feistel_hash(unsigned v, unsigned key) {
  v ^= key; v *= 0x9E3779B1u; v ^= v >> 15; v *= 0x85EBCA77u; v ^= v >> 13; v *= 0xC2B2AE3Du; v ^= v >> 16;
  return v;
}
__global__ void k_random_subset(unsigned long long seed, long long N, int n, int64_t* __restrict__ out,
                                const unsigned long long* __restrict__ seed_dev = nullptr) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  if (seed_dev) seed = *seed_dev;  // the step clock's per-step seed (CUDA-graph replays)
  int bits = 2;
  while ((1ll << bits) < N) bits += 2;  // even number of bits: two equal halves
  const int half = bits / 2;
  const unsigned mask = (1u << half) - 1u;
  unsigned long long x = (unsigned long long)t;
  do {
    unsigned l = (unsigned)(x >> half) & mask, r = (unsigned)x & mask;
#pragma unroll
    for (int round = 0; round < 4; ++round) {
      const unsigned f = feistel_hash(r, (unsigned)(seed >> (16 * round)) ^ (0xA511E9B3u * (round + 1))) & mask;
      const unsigned nl = r, nr = l ^ f;
      l = nl; r = nr;
    }
    x = ((unsigned long long)l << half) | r;
  } while ((long long)x >= N);
  out[t] = (int64_t)x;
}

// ================================================================== step clock
// Everything that changes from one optimisation step to the next OUTSIDE the parameters -- Adam's
// bias corrections (model_wrapper_overfit.py:104-105, torch.optim.Adam's per-parameter step count)
// and the seed of the softmin point sample (intrinsics_softmin.py:90) -- kept in device memory and
// advanced by a one-thread kernel, so that a whole step is a fixed sequence of launches with fixed
// arguments: capturable in a CUDA graph and replayable.
struct StepClock {
  unsigned step, focal_step;
  float step_size, bc2_sqrt;              // lr / (1 - beta1^step), sqrt(1 - beta2^step)
  float focal_step_size, focal_bc2_sqrt;  // the same on the focal length's own count
  unsigned long long seed;
};
static_assert(sizeof(StepClock) == 32, "StepClock layout (FM_STEP_CLOCK_BYTES)");

__global__ void k_clock_tick(StepClock* c, double lr, double b1, double b2, unsigned long long base_seed,
                             int tick_focal) {
  const unsigned t = c->step + 1u;
  c->step = t;
  c->step_size = (float)(lr / (1.0 - pow(b1, (double)t)));
  c->bc2_sqrt = (float)sqrt(1.0 - pow(b2, (double)t));
  const unsigned tf = c->focal_step + (tick_focal ? 1u : 0u);
  c->focal_step = tf;
  if (tf > 0u) {
    c->focal_step_size = (float)(lr / (1.0 - pow(b1, (double)tf)));
    c->focal_bc2_sqrt = (float)sqrt(1.0 - pow(b2, (double)tf));
  }
  unsigned long long z = base_seed + 0x9E3779B97F4A7C15ull * (unsigned long long)t;  // splitmix64
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  c->seed = z ^ (z >> 31);
}

// ================================================================== trajectory metrics
// scipy.spatial.procrustes ATE (fm_ate.cuh), one block per trajectory.  The block size fixes the
// order of the float64 sums, so a trajectory's result does not depend on how it was batched, nor on
// whether the fused step or fm_trajectory_ate evaluated it.
constexpr int kAteThreads = 128;

// Sums up to 9 doubles over the block; every thread receives the totals (in the same order).
struct BlockSum {
  double* sh;  // [kAteThreads / 32][9] shared
  __device__ void operator()(double* v, int n) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int k = 0; k < n; ++k) {
      v[k] = warp_sum(v[k]);
      if (lane == 0) sh[warp * 9 + k] = v[k];
    }
    __syncthreads();
    for (int k = 0; k < n; ++k) {
      double t = 0.0;
      for (int w = 0; w < kAteThreads / 32; ++w) t += sh[w * 9 + k];
      v[k] = t;
    }
    __syncthreads();
  }
};

// The row of the fused step's metrics ring (fm_overfit_step_args.metrics_log) that the block also
// writes; log == NULL for plain fm_trajectory_ate.
struct MetricsRow {
  float* log;
  int capacity;
  const StepClock* clock;
  const float *loss, *track_loss, *k4;  // track_loss NULL: no tracking loss in this step
  float gt_fx, gt_fy;
};

__global__ void __launch_bounds__(kAteThreads)
k_trajectory_ate(const float* __restrict__ gt, const float* __restrict__ pred, int pred_stride, int pred_cstride, int F,
                 float* __restrict__ ate, float* __restrict__ aligned_gt, float* __restrict__ aligned_pred,
                 int* __restrict__ status, MetricsRow row) {
  __shared__ double s_red[kAteThreads / 32 * 9];
  const size_t t = blockIdx.x;
  float* ate_out = ate ? ate + t : nullptr;
  if (row.log) {  // the fused step: columns flow loss, tracking loss, |fx error|, |fy error|, ATE
    float* r = row.log + (size_t)((row.clock->step - 1u) % (unsigned)row.capacity) * 5;
    if (threadIdx.x == 0) {
      double fx = 0.0, fy = 0.0;
      for (int f = 0; f < F; ++f) { fx += (double)row.k4[f * 4 + 0]; fy += (double)row.k4[f * 4 + 1]; }
      r[0] = *row.loss;
      r[1] = row.track_loss ? *row.track_loss : 0.f;
      r[2] = (float)fabs((double)row.gt_fx - fx / F);
      r[3] = (float)fabs((double)row.gt_fy - fy / F);
      if (!gt) r[4] = NAN;
    }
    if (!gt) return;
    ate_out = r + 4;
  }
  AtePoints x;
  x.gt = gt + t * F * 3;
  x.pred = pred + t * F * pred_stride;
  x.gt_stride = 3;
  x.pred_stride = pred_stride;
  x.pred_cstride = pred_cstride;
  x.F = F;
  BlockSum red{s_red};
  double v;
  const int st = trajectory_ate(x, threadIdx.x, kAteThreads, red, v, aligned_gt ? aligned_gt + t * F * 3 : nullptr,
                                aligned_pred ? aligned_pred + t * F * 3 : nullptr);
  if (threadIdx.x == 0) {
    *ate_out = (float)v;
    if (status) status[t] = st;
  }
}

// ================================================================== fused overfit step helpers
// focal_lengths_to_intrinsics (intrinsics/common.py:6-20) for a shared focal length, as k4 rows.
__global__ void k_k4_from_focal(const float* __restrict__ focal, float* __restrict__ k4, int BF, int H, int W) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= BF) return;
  const float scaled = *focal * sqrtf((float)H * (float)W);  // float32 like the reference
  k4[t * 4 + 0] = scaled / (float)W;
  k4[t * 4 + 1] = scaled / (float)H;
  k4[t * 4 + 2] = 0.5f;
  k4[t * 4 + 3] = 0.5f;
}

// d loss / d focal from the per-frame k4 gradients (flow-loss part + Procrustes part).
__global__ void k_focal_grad(const double* __restrict__ k4acc, const double* __restrict__ flowacc,
                             const float* __restrict__ extra_g_k4, float* __restrict__ g_focal, int B,
                             int F, int H, int W, const float* __restrict__ flow_scale = nullptr) {
  double sx = 0.0, sy = 0.0;
  const double fs = flow_scale ? (double)*flow_scale : 1.0;  // d total / d flow loss (the Procrustes part in k4acc carries it already)
  for (int t = threadIdx.x; t < B * F; t += blockDim.x) {
    double g[4];
    flow_k4_grad(flowacc, t, F, g);
    sx += fs * g[0] + k4acc[(size_t)t * 4 + 0] + (extra_g_k4 ? (double)extra_g_k4[t * 4 + 0] : 0.0);
    sy += fs * g[1] + k4acc[(size_t)t * 4 + 1] + (extra_g_k4 ? (double)extra_g_k4[t * 4 + 1] : 0.0);
  }
  __shared__ double sm[2][32];
  sx = warp_sum(sx); sy = warp_sum(sy);
  if ((threadIdx.x & 31) == 0) { sm[0][threadIdx.x >> 5] = sx; sm[1][threadIdx.x >> 5] = sy; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double ax = 0.0, ay = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { ax += sm[0][w]; ay += sm[1][w]; }
    const double sc = sqrt((double)H * (double)W);
    *g_focal = (float)(ax * sc / W + ay * sc / H);
  }
}

// ---------------------------------------------------------------- launch geometry
int blocks_for(int n_items_per_row, int vec) {
  // ~4096 items per block keeps thousands of blocks in flight at the BASELINE sizes and
  // still gives every thread a few independent loads.
  const int per_block = kThreads * vec * 16;
  int nb = (n_items_per_row + per_block - 1) / per_block;
  return nb < 1 ? 1 : nb;
}

// Lanes per row of the warp patch of the dense Procrustes kernels (PatchSite); tools/ab_libs.py
// compares builds with other values.
#ifndef FM_PATCH_LANES  // build-time knob for tools/ab_libs.py (0 = strips only)
#define FM_PATCH_LANES 8
#endif
constexpr int kPatchLanes = FM_PATCH_LANES;
static bool patch_shape_ok(int H, int W) {
  constexpr int lx = kPatchLanes > 0 ? kPatchLanes : 1;
  return kPatchLanes > 0 && W % (4 * lx) == 0 && H % (32 / lx) == 0;
}

// 1-D grid of the dense kernels (block_item_range): every SM holds `ctas_per_sm` blocks for the whole
// launch.
int sm_count_cached() {
  static const int n = [] {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v < 1)
      v = 132;
    return v;
  }();
  return n;
}
int persistent_grid(int ctas_per_sm, long long items) {
  const long long g = (long long)sm_count_cached() * ctas_per_sm;
  return (int)(items < g ? (items < 1 ? 1 : items) : g);
}

// Rounds of the dense Procrustes kernels (block_item_range): runs of about kRunChunks chunks per block
// and round.  The dense phase-D2 kernels (REDs + the fused Adam streams) use rounds at every shape;
// k_moments_dense (read-only gathers) only once the resident blocks' row bands (sized for flows of a few
// percent of the image) stop fitting in a third of L2, and keeps one round below that.
constexpr int kRunChunks = 8;
int procrustes_rounds(int H, int W, long long items, int grid, bool gathers_only) {
  if (gathers_only) {
    static const double l2_bytes = [] {
      int dev = 0, v = 0;
      if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrL2CacheSize, dev) != cudaSuccess || v < 1)
        v = 50 << 20;
      return (double)v;
    }();
    const double band_rows = 0.07 * H + 6.0;
    if ((double)grid * band_rows * W * 4.0 <= 0.35 * l2_bytes) return 1;
  }
  const long long per_block = (items + grid - 1) / grid;
  const long long rounds = per_block / kRunChunks;
  return (int)(rounds < 1 ? 1 : rounds);
}

// Index-mode launches (subsampled Procrustes, the focal sweep): few points, dependent gathers ->
// one point per thread so that the latency is covered by parallelism, not by a per-thread loop.
int blocks_for_points(int n) {
  int nb = (n + kThreads - 1) / kThreads;
  return nb < 1 ? 1 : nb;
}

bool bad_dims(int B, int F, int H, int W) { return B < 1 || F < 2 || H < 1 || W < 1 || (long long)H * W > (1ll << 30); }

}  // namespace

namespace {
// intrinsics_mode: 0 = per-frame k4 with full gradients, 1 = one shared focal length (gradient
// booked as d/dfx of each frame), 2 = constant intrinsics (no gradient).
int launch_flow(const float* depth, const float* k4, const float* rt, const float* ff, const float* fb,
                const float* mf, const float* mb, const double* mask_sum, int mapping, float delta,
                float loss_weight, int intrinsics_mode, float* g_depth, double* flowacc, int B, int F,
                int H, int W, cudaStream_t s) {
  const int BF = B * F;
  const int vec = (W % 4 == 0) ? 4 : 1;
  dim3 grid(blocks_for(H * W, vec), BF);
  if (intrinsics_mode == 0) {
    if (vec == 4) k_flow<4><<<grid, kThreads, 0, s>>>(depth, k4, rt, ff, fb, mf, mb, mask_sum, nullptr, mapping, delta, loss_weight, g_depth, flowacc, F, H, W);
    else k_flow<1><<<grid, kThreads, 0, s>>>(depth, k4, rt, ff, fb, mf, mb, mask_sum, nullptr, mapping, delta, loss_weight, g_depth, flowacc, F, H, W);
    FM_CHECK_LAUNCH("k_flow");
    return 0;
  }
  const bool focal = intrinsics_mode == 1;
  const int pg = persistent_grid(2, (long long)BF * ((H * W + kThreads * vec - 1) / (kThreads * vec)));
  if (vec == 4) {
    if (focal) k_flow_lean<4, true, 2><<<pg, kThreads, 0, s>>>(depth, k4, rt, ff, fb, mf, mb, mask_sum, mapping, delta, loss_weight, g_depth, flowacc, F, H, W, BF);
    else k_flow_lean<4, false, 2><<<pg, kThreads, 0, s>>>(depth, k4, rt, ff, fb, mf, mb, mask_sum, mapping, delta, loss_weight, g_depth, flowacc, F, H, W, BF);
  } else {
    if (focal) k_flow_lean<1, true, 2><<<pg, kThreads, 0, s>>>(depth, k4, rt, ff, fb, mf, mb, mask_sum, mapping, delta, loss_weight, g_depth, flowacc, F, H, W, BF);
    else k_flow_lean<1, false, 2><<<pg, kThreads, 0, s>>>(depth, k4, rt, ff, fb, mf, mb, mask_sum, mapping, delta, loss_weight, g_depth, flowacc, F, H, W, BF);
  }
  FM_CHECK_LAUNCH("k_flow_lean");
  k_flow_lean_convert<<<(BF + 63) / 64, 64, 0, s>>>(flowacc, rt, k4, focal ? 1 : 0, B, F, H, W);
  FM_CHECK_LAUNCH("k_flow_lean_convert");
  return 0;
}
}  // namespace

// ---------------------------------------------------------------- tiled path: host side
namespace {
typedef CUresult (*TensorMapEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                      const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                      CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                      CUtensorMapFloatOOBfill);
TensorMapEncodeFn tensor_map_encoder() {
  static const TensorMapEncodeFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return (TensorMapEncodeFn)p;
  }();
  return fn;
}

// (W, H, frames) float32 tensor, box = one (kWX x kWY x 1) window; out-of-range parts read as 0.
int make_window_map(CUtensorMap* m, const float* base, int W, int H, int frames) {
  const TensorMapEncodeFn enc = tensor_map_encoder();
  if (!enc) return fail_msg("tiled path: cuTensorMapEncodeTiled is not available from this driver");
  const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)frames};
  const cuuint64_t strides[2] = {(cuuint64_t)W * 4ull, (cuuint64_t)W * (cuuint64_t)H * 4ull};
  const cuuint32_t box[3] = {(cuuint32_t)tiled::kWX, (cuuint32_t)tiled::kWY, 1u};
  const cuuint32_t estr[3] = {1u, 1u, 1u};
  const CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[128];
    snprintf(msg, sizeof(msg), "tiled path: cuTensorMapEncodeTiled failed (CUresult %d) for %d x %d x %d", (int)r, W, H, frames);
    return fail_msg(msg);
  }
  return 0;
}

int sm_count() {
  static const int n = [] {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v < 1)
      v = 132;
    return v;
  }();
  return n;
}

bool tiled_shape_ok(int F, int H, int W) { return F >= 2 && W % 4 == 0 && H >= 1 && W < 32768 && H < 32768; }

// Phase A through the plan: moments of all pairs (+ the step's correspondence weights into the
// plan's scratch for phase D), then the solve.
int launch_moments_tiled(const float* depth, const float* k4, const float* bflow, const float* weights, float wsens,
                         const tiled::Plan& pl, double* moments, const float* zshift, int F, int H, int W,
                         cudaStream_t s) {
  CUtensorMap tm;
  int rc = make_window_map(&tm, depth, W, H, F);
  if (rc) return rc;
  tiled::MomArgs b;
  b.depth = depth; b.k4 = k4; b.bflow = bflow; b.weights = weights; b.wscratch = pl.wscratch; b.moments = moments;
  b.zshift = zshift;
  b.tinfo = pl.tiles; b.wsens = wsens; b.F = F; b.H = H; b.W = W; b.tiles_x = pl.tiles_x;
  b.tiles = pl.tiles_x * pl.tiles_y; b.n_items = (F - 1) * b.tiles;
  int grid = sm_count() * 3;
  if (grid > b.n_items) grid = b.n_items;
  static const cudaError_t at1 = cudaFuncSetAttribute(tiled::k_moments_tiled<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tiled::kMomSmem);
  static const cudaError_t at0 = cudaFuncSetAttribute(tiled::k_moments_tiled<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, tiled::kMomSmem);
  if (at1 != cudaSuccess || at0 != cudaSuccess) return fail("k_moments_tiled: shared memory attribute", at1 != cudaSuccess ? at1 : at0);
  if (weights) tiled::k_moments_tiled<true><<<grid, tiled::kT, tiled::kMomSmem, s>>>(tm, b);
  else tiled::k_moments_tiled<false><<<grid, tiled::kT, tiled::kMomSmem, s>>>(tm, b);
  FM_CHECK_LAUNCH("k_moments_tiled");
  return 0;
}

// Phase D2 through the plan: transposed (gather-form) bilinear splat + per-pixel adjoints + final depth
// gradient in one pass; flow outliers afterwards as REDs.
int launch_backward_tiled(const float* depth, const float* k4, const float* bflow, float* weights, float wsens,
                          const tiled::Plan& pl, unsigned ovf_max, const PairAdjoint* adj, float* g_depth,
                          float* g_weights, const AdamFuse& af, int F, int H, int W, cudaStream_t s) {
  CUtensorMap tm_d, tm_w;
  int rc = make_window_map(&tm_d, depth, W, H, F);
  if (rc) return rc;
  if ((rc = make_window_map(&tm_w, pl.wscratch, W, H, F - 1))) return rc;
  tiled::BwdArgs b;
  b.depth = depth; b.k4 = k4; b.bflow = bflow; b.weights = weights; b.adj = adj; b.tinfo = pl.tiles;
  b.perm = pl.perm; b.entries = pl.entries; b.g_depth = g_depth; b.g_weights = g_weights; b.adam = af;
  b.wsens = wsens; b.F = F; b.H = H; b.W = W; b.tiles_x = pl.tiles_x; b.tiles = pl.tiles_x * pl.tiles_y;
  b.n_items = F * b.tiles;
  int grid = sm_count() * 2;
  if (grid > b.n_items) grid = b.n_items;
  static const cudaError_t at1 = cudaFuncSetAttribute(tiled::k_backward_tiled<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tiled::kBwdSmem);
  static const cudaError_t at0 = cudaFuncSetAttribute(tiled::k_backward_tiled<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, tiled::kBwdSmem);
  if (at1 != cudaSuccess || at0 != cudaSuccess) return fail("k_backward_tiled: shared memory attribute", at1 != cudaSuccess ? at1 : at0);
  if (weights) tiled::k_backward_tiled<true><<<grid, tiled::kT, tiled::kBwdSmem, s>>>(tm_d, tm_w, b);
  else tiled::k_backward_tiled<false><<<grid, tiled::kT, tiled::kBwdSmem, s>>>(tm_d, tm_w, b);
  FM_CHECK_LAUNCH("k_backward_tiled");
  if (ovf_max > 0u) {
    const unsigned n = ovf_max < (unsigned)pl.ovf_cap ? ovf_max : (unsigned)pl.ovf_cap;
    dim3 g2((n + 255u) / 256u, F - 1);
    tiled::k_backward_overflow<<<g2, 256, 0, s>>>(depth, k4, weights ? pl.wscratch : nullptr, adj, pl.ovf_count, pl.ovf,
                                                  pl.ovf_cap, g_depth, H, W);
    FM_CHECK_LAUNCH("k_backward_overflow");
  }
  return 0;
}
}  // namespace

// =================================================================== C ABI
extern "C" {

int fm_version(void) { return 102; }
unsigned long long fm_launch_count(void) { return fm_host::launches(); }
const char* fm_last_error(void) { return fm_host::last_error(); }

size_t fm_workspace_bytes(int B, int F, int H, int W) {
  (void)H; (void)W;
  if (B < 1 || F < 2) return 0;
  return carve(nullptr, B, F).bytes;
}

int fm_workspace_reset(void* ws, int B, int F, int H, int W, void* stream) {
  if (!ws || bad_dims(B, F, H, W)) return fail_msg("fm_workspace_reset: bad arguments");
  Workspace w = carve(ws, B, F);
  cudaError_t e = cudaMemsetAsync(ws, 0, (char*)w.state - (char*)ws, (cudaStream_t)stream);
  if (e != cudaSuccess) return fail("fm_workspace_reset", e);
  return 0;
}

int fm_unproject(const float* depth, const float* k4, float* surfaces, int BF, int H, int W, void* stream) {
  if (!depth || !k4 || !surfaces || BF < 1) return fail_msg("fm_unproject: bad arguments");
  dim3 grid(blocks_for(H * W, 4), BF);
  k_unproject<<<grid, kThreads, 0, (cudaStream_t)stream>>>(depth, k4, surfaces, H, W);
  FM_CHECK_LAUNCH("fm_unproject");
  return 0;
}

int fm_unproject_bwd(const float* depth, const float* k4, const float* g_surfaces, float* g_depth,
                     float* g_k4, void* ws, int B, int F, int H, int W, void* stream) {
  if (!depth || !k4 || !g_surfaces || !g_depth || !g_k4 || !ws || bad_dims(B, F, H, W))
    return fail_msg("fm_unproject_bwd: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  Workspace w = carve(ws, B, F);
  const int BF = B * F;
  cudaError_t e = cudaMemsetAsync(w.k4acc, 0, (size_t)BF * 4 * sizeof(double), s);
  if (e != cudaSuccess) return fail("fm_unproject_bwd: memset", e);
  dim3 grid(blocks_for(H * W, 4), BF);
  k_unproject_bwd<<<grid, kThreads, 0, s>>>(depth, k4, g_surfaces, g_depth, w.k4acc, H, W);
  FM_CHECK_LAUNCH("fm_unproject_bwd: k_unproject_bwd");
  k_d2f<<<(BF * 4 + 127) / 128, 128, 0, s>>>(w.k4acc, g_k4, BF * 4);
  FM_CHECK_LAUNCH("fm_unproject_bwd: k_d2f");
  return 0;
}

int fm_reproject(const float* xyz, const float* rt, const float* k4, float* xy, unsigned char* in_front,
                 int items, int n, void* stream) {
  if (!xyz || !rt || !k4 || !xy || items < 1 || n < 1) return fail_msg("fm_reproject: bad arguments");
  dim3 grid(blocks_for(n, 1), items);
  k_reproject<<<grid, kThreads, 0, (cudaStream_t)stream>>>(xyz, rt, k4, xy, in_front, n);
  FM_CHECK_LAUNCH("fm_reproject");
  return 0;
}

static int procrustes_fwd_impl(const float* depth, const float* k4, const float* backward_flow,
                               const float* weights, float wsens, const int64_t* indices,
                               int num_indices, float* rt, void* ws, int B, int F, int H, int W,
                               void* stream, const PairLayout* layout = nullptr, void* plan = nullptr,
                               const float* moments_k4 = nullptr, bool solve = true) {
  const PairLayout lay = layout ? *layout : dense_layout(F, H, W);
  if (!depth || !k4 || !backward_flow || (!rt && solve) || !ws || bad_dims(B, F, H, W))
    return fail_msg("fm_procrustes_fwd: bad arguments");
  if (plan && (B != 1 || indices || layout || !tiled_shape_ok(F, H, W)))
    return fail_msg("fm_procrustes_fwd: the splat plan serves the dense single-video path with W % 4 == 0");
  if (indices && num_indices < 1) return fail_msg("fm_procrustes_fwd: empty index set");
  cudaStream_t s = (cudaStream_t)stream;
  Workspace w = carve(ws, B, F);
  const int BP = B * (F - 1);
  if (moments_k4) {  // fm_procrustes_moments already ran with those intrinsics
    if (plan || indices || layout) return fail_msg("fm_procrustes_fwd: precomputed moments serve the dense path");
    if (!solve) return 0;
    k_solve<<<(BP + 63) / 64, 64, 0, s>>>(w.moments, w.zshift, rt, w.state, BP, lay, H, W, moments_k4, k4);
    FM_CHECK_LAUNCH("fm_procrustes_fwd: k_solve");
    return 0;
  }
  cudaError_t e = cudaMemsetAsync(w.moments, 0, (size_t)BP * kNumMoments * sizeof(double), s);
  if (e != cudaSuccess) return fail("fm_procrustes_fwd: memset", e);
  k_pair_shift<<<BP, kThreads, 0, s>>>(depth, weights, wsens, w.zshift, lay, H, W);
  FM_CHECK_LAUNCH("fm_procrustes_fwd: k_pair_shift");
  if (plan) {
    const tiled::Plan pl = tiled::plan_carve(plan, F, H, W);
    const int rc = launch_moments_tiled(depth, k4, backward_flow, weights, wsens, pl, w.moments, w.zshift, F, H, W, s);
    if (rc) return rc;
  } else if (indices) {
    dim3 grid(blocks_for_points(num_indices), BP);
    k_moments<1><<<grid, kThreads, 0, s>>>(depth, k4, backward_flow, weights, indices, num_indices, w.moments, w.zshift, wsens, lay, H, W);
  } else if (patch_shape_ok(H, W)) {
    const long long items = (long long)BP * ((H * W + kThreads * 4 - 1) / (kThreads * 4));
    const int pg = persistent_grid(3, items);
    k_moments_dense<4, kPatchLanes><<<pg, kThreads, 0, s>>>(depth, k4, backward_flow, weights, w.moments, w.zshift, wsens, lay, H, W, BP, procrustes_rounds(H, W, items, pg, true));
  } else if (W % 4 == 0) {
    const long long items = (long long)BP * ((H * W + kThreads * 4 - 1) / (kThreads * 4));
    const int pg = persistent_grid(3, items);
    k_moments_dense<4, 0><<<pg, kThreads, 0, s>>>(depth, k4, backward_flow, weights, w.moments, w.zshift, wsens, lay, H, W, BP, procrustes_rounds(H, W, items, pg, true));
  } else {
    const long long items = (long long)BP * ((H * W + kThreads - 1) / kThreads);
    const int pg = persistent_grid(3, items);
    k_moments_dense<1, 0><<<pg, kThreads, 0, s>>>(depth, k4, backward_flow, weights, w.moments, w.zshift, wsens, lay, H, W, BP, procrustes_rounds(H, W, items / 4, pg, true));
  }
  if (!plan) FM_CHECK_LAUNCH("fm_procrustes_fwd: k_moments");
  if (!solve) return 0;
  k_solve<<<(BP + 63) / 64, 64, 0, s>>>(w.moments, w.zshift, rt, w.state, BP, lay, H, W);
  FM_CHECK_LAUNCH("fm_procrustes_fwd: k_solve");
  return 0;
}

int fm_procrustes_fwd(const float* depth, const float* k4, const float* backward_flow,
                      const float* weights, const int64_t* indices, int num_indices, float* rt,
                      void* ws, int B, int F, int H, int W, void* stream) {
  return procrustes_fwd_impl(depth, k4, backward_flow, weights, 0.f, indices, num_indices, rt, ws, B, F,
                             H, W, stream);
}

int fm_procrustes_moments(const float* depth, const float* k4, const float* backward_flow,
                          const float* weights, float weight_sensitivity, void* ws, int F, int H, int W,
                          void* stream) {
  return procrustes_fwd_impl(depth, k4, backward_flow, weights, weight_sensitivity, nullptr, 0, nullptr, ws, 1, F,
                             H, W, stream, nullptr, nullptr, nullptr, /*solve=*/false);
}

static int procrustes_bwd_impl(const float* depth, const float* k4, const float* backward_flow,
                               const float* weights, float wsens, const int64_t* indices,
                               int num_indices, const float* g_rt, int include_flow_loss,
                               const float* flow_scale, float* g_depth, float* g_weights, float* g_k4,
                               void* ws, int B, int F, int H, int W, void* stream,
                               const PairLayout* layout = nullptr, const AdamFuse* adam = nullptr,
                               void* plan = nullptr, unsigned plan_ovf_max = 0u, bool depth_prescaled = false) {
  const PairLayout lay = layout ? *layout : dense_layout(F, H, W);
  if (plan && (B != 1 || indices || layout || !tiled_shape_ok(F, H, W)))
    return fail_msg("fm_procrustes_bwd: the splat plan serves the dense single-video path with W % 4 == 0");
  if (!depth || !k4 || !backward_flow || !g_depth || !g_k4 || !ws || bad_dims(B, F, H, W))
    return fail_msg("fm_procrustes_bwd: bad arguments");
  if (!g_rt && !include_flow_loss) return fail_msg("fm_procrustes_bwd: no pose gradient given");
  cudaStream_t s = (cudaStream_t)stream;
  Workspace w = carve(ws, B, F);
  const int BP = B * (F - 1), BF = B * F;
  cudaError_t e = cudaMemsetAsync(w.k4acc, 0, (size_t)BF * 4 * sizeof(double), s);
  if (e != cudaSuccess) return fail("fm_procrustes_bwd: memset", e);
  AdamFuse af;
  if (adam) af = *adam; else memset(&af, 0, sizeof(af));
  float* weights_rw = const_cast<float*>(weights);
  if (include_flow_loss && flow_scale && !depth_prescaled) {
    // the direct depth gradient already sitting in g_depth was computed for scale 1
    k_scale_inplace<<<sm_count_cached() * 4, kThreads, 0, s>>>(g_depth, flow_scale, (size_t)BF * H * W);
    FM_CHECK_LAUNCH("fm_procrustes_bwd: k_scale_inplace");
  }
  if (plan) {
    // one focal length shared by all frames (or constant intrinsics): the Procrustes part of the
    // intrinsics gradient comes from the moment sums, the pixel kernel carries no K accumulators
    k_adjoint<<<(BP + 63) / 64, 64, 0, s>>>(w.flowacc, w.state, g_rt, include_flow_loss, flow_scale, w.adj, BP, F,
                                            w.moments, k4, w.k4acc);
    FM_CHECK_LAUNCH("fm_procrustes_bwd: k_adjoint");
    const tiled::Plan pl = tiled::plan_carve(plan, F, H, W);
    const int rc = launch_backward_tiled(depth, k4, backward_flow, weights_rw, wsens, pl, plan_ovf_max, w.adj, g_depth,
                                         g_weights, af, F, H, W, s);
    if (rc) return rc;
    k_k4_finalize<<<(BF + 127) / 128, 128, 0, s>>>(w.k4acc, w.flowacc, include_flow_loss, flow_scale, g_k4, B, F);
    FM_CHECK_LAUNCH("fm_procrustes_bwd: k_k4_finalize");
    return 0;
  }
  k_adjoint<<<(BP + 63) / 64, 64, 0, s>>>(w.flowacc, w.state, g_rt, include_flow_loss, flow_scale, w.adj, BP, F);
  FM_CHECK_LAUNCH("fm_procrustes_bwd: k_adjoint");
  if (indices) {
    dim3 grid(blocks_for_points(num_indices), BP);
    k_distribute<1><<<grid, kThreads, 0, s>>>(depth, k4, backward_flow, weights_rw, indices, num_indices, w.adj, g_depth, g_weights, w.k4acc, wsens, lay, af, H, W);
  } else if (W % 4 == 0) {
    const long long items = (long long)BP * ((W + kWinTW - 1) / kWinTW) * ((H + kWinTH - 1) / kWinTH);
    const int pg = persistent_grid(FM_WIN_CTAS, items);
    const long long chunks = items * (kWinTW * kWinTH) / (kThreads * 4);  // rounds are sized in 1024-pixel chunks
    k_distribute_window<<<pg, kThreads, 0, s>>>(depth, k4, backward_flow, weights_rw, w.adj, g_depth, g_weights, w.k4acc, wsens, lay, af, H, W, BP, procrustes_rounds(H, W, chunks, pg, false));
  } else {
    const long long items = (long long)BP * ((H * W + kThreads - 1) / kThreads);
    const int pg = persistent_grid(3, items);
    k_distribute_dense<<<pg, kThreads, 0, s>>>(depth, k4, backward_flow, weights_rw, w.adj, g_depth, g_weights, w.k4acc, wsens, lay, af, H, W, BP, procrustes_rounds(H, W, items / 4, pg, false));
  }
  FM_CHECK_LAUNCH("fm_procrustes_bwd: k_distribute");
  k_k4_finalize<<<(BF + 127) / 128, 128, 0, s>>>(w.k4acc, w.flowacc, include_flow_loss, flow_scale, g_k4, B, F);
  FM_CHECK_LAUNCH("fm_procrustes_bwd: k_k4_finalize");
  return 0;
}

int fm_procrustes_bwd(const float* depth, const float* k4, const float* backward_flow,
                      const float* weights, const int64_t* indices, int num_indices,
                      const float* g_rt, int include_flow_loss, const float* flow_scale,
                      float* g_depth, float* g_weights, float* g_k4, void* ws, int B, int F, int H,
                      int W, void* stream) {
  return procrustes_bwd_impl(depth, k4, backward_flow, weights, 0.f, indices, num_indices, g_rt,
                             include_flow_loss, flow_scale, g_depth, g_weights, g_k4, ws, B, F, H, W,
                             stream);
}

size_t fm_splat_plan_bytes(int F, int H, int W) {
  if (!tiled_shape_ok(F, H, W) || (long long)H * W > (1ll << 30)) return 0;
  return tiled::plan_carve(nullptr, F, H, W).bytes;
}

int fm_splat_plan_build(const float* backward_flow, void* plan, int F, int H, int W, void* stream) {
  if (!backward_flow || !plan || !tiled_shape_ok(F, H, W) || bad_dims(1, F, H, W))
    return fail_msg("fm_splat_plan_build: bad arguments (needs F >= 2 and W % 4 == 0)");
  cudaStream_t s = (cudaStream_t)stream;
  const tiled::Plan pl = tiled::plan_carve(plan, F, H, W);
  const int P = F - 1, tiles = pl.tiles_x * pl.tiles_y;
  const size_t N = (size_t)H * W;
  cudaError_t e;
  if ((e = cudaMemsetAsync(pl.count, 0, (size_t)P * N * sizeof(unsigned), s)) != cudaSuccess ||
      (e = cudaMemsetAsync(pl.tile_sum, 0, (size_t)P * tiles * sizeof(int4), s)) != cudaSuccess ||
      (e = cudaMemsetAsync(pl.ovf_count, 0, (size_t)P * sizeof(unsigned), s)) != cudaSuccess)
    return fail("fm_splat_plan_build: memset", e);
  tiled::k_plan_init<<<1, 1, 0, s>>>(pl.hdr, F, H, W, pl.tiles_x, pl.tiles_y, pl.ovf_cap, (unsigned long long)pl.entry_capacity);
  FM_CHECK_LAUNCH("k_plan_init");
  int nb = (int)((N + 255) / 256);
  if (nb > 1024) nb = 1024;
  tiled::k_plan_count<<<dim3(nb, P), 256, 0, s>>>(backward_flow, pl.count, pl.tile_sum, H, W, pl.tiles_x, tiles);
  FM_CHECK_LAUNCH("k_plan_count");
  tiled::k_plan_sort<<<dim3(tiles, P), tiled::kT, 0, s>>>(backward_flow, pl.count, pl.tile_sum, pl.tiles, pl.perm, pl.slot_of,
                                                           pl.tile_total, pl.hdr, H, W, pl.tiles_x, tiles);
  FM_CHECK_LAUNCH("k_plan_sort");
  tiled::k_plan_scan<<<1, 1024, 0, s>>>(pl.tile_total, pl.tiles, pl.hdr, P * tiles, (unsigned long long)pl.entry_capacity);
  FM_CHECK_LAUNCH("k_plan_scan");
  if ((e = cudaMemsetAsync(pl.count, 0, (size_t)P * N * sizeof(unsigned), s)) != cudaSuccess)
    return fail("fm_splat_plan_build: memset", e);
  tiled::k_plan_fill<<<dim3(nb, P), 256, 0, s>>>(backward_flow, pl.tiles, pl.slot_of, pl.count, pl.entries, pl.ovf_count, pl.ovf,
                                                 pl.hdr, H, W, pl.tiles_x, tiles, (unsigned long long)pl.entry_capacity, pl.ovf_cap);
  FM_CHECK_LAUNCH("k_plan_fill");
  const size_t slots = (size_t)P * tiles * tiled::kCells;
  tiled::k_plan_canon<<<(unsigned)((slots + 255) / 256), 256, 0, s>>>(pl.tiles, pl.perm, pl.count, pl.entries, pl.ovf_count, pl.hdr,
                                                                     H, W, pl.tiles_x, tiles, P, (unsigned long long)pl.entry_capacity);
  FM_CHECK_LAUNCH("k_plan_canon");
  return 0;
}

int fm_splat_plan_info(const void* plan, int* status, unsigned* overflow_max, unsigned long long* total_entries,
                       void* stream) {
  if (!plan) return fail_msg("fm_splat_plan_info: bad arguments");
  tiled::PlanHeader h;
  cudaError_t e = cudaMemcpyAsync(&h, plan, sizeof(h), cudaMemcpyDeviceToHost, (cudaStream_t)stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t)stream);
  if (e != cudaSuccess) return fail("fm_splat_plan_info", e);
  if (h.magic != tiled::kPlanMagic) return fail_msg("fm_splat_plan_info: not a splat plan");
  if (status) *status = h.status;
  if (overflow_max) *overflow_max = h.ovf_max;
  if (total_entries) *total_entries = h.total_entries;
  return 0;
}

int fm_procrustes_fwd_planned(const float* depth, const float* k4, const float* backward_flow, const float* weights,
                              float weight_sensitivity, void* plan, float* rt, void* ws, int F, int H, int W,
                              void* stream) {
  if (!plan) return fail_msg("fm_procrustes_fwd_planned: plan missing");
  return procrustes_fwd_impl(depth, k4, backward_flow, weights, weight_sensitivity, nullptr, 0, rt, ws, 1, F, H, W,
                             stream, nullptr, plan);
}

int fm_procrustes_bwd_planned(const float* depth, const float* k4, const float* backward_flow, const float* weights,
                              float weight_sensitivity, void* plan, unsigned plan_overflow_max, const float* g_rt,
                              int include_flow_loss, float* g_depth, float* g_weights, float* g_k4, void* ws, int F,
                              int H, int W, void* stream) {
  if (!plan) return fail_msg("fm_procrustes_bwd_planned: plan missing");
  return procrustes_bwd_impl(depth, k4, backward_flow, weights, weight_sensitivity, nullptr, 0, g_rt, include_flow_loss,
                             nullptr, g_depth, g_weights, g_k4, ws, 1, F, H, W, stream, nullptr, nullptr, plan,
                             plan_overflow_max);
}

int fm_mask_sum(const float* forward_mask, const float* backward_mask, double* out, size_t count, void* stream) {
  if (!forward_mask || !backward_mask || !out) return fail_msg("fm_mask_sum: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(out, 0, sizeof(double), s);
  if (e != cudaSuccess) return fail("fm_mask_sum: memset", e);
  if (count == 0) return 0;
  size_t nb = (count / 4 + kThreads * 8 - 1) / (kThreads * 8);
  if (nb < 1) nb = 1;
  if (nb > (size_t)sm_count_cached() * 8) nb = (size_t)sm_count_cached() * 8;
  k_mask_sum<<<(unsigned)nb, kThreads, 0, s>>>(forward_mask, backward_mask, out, count);
  FM_CHECK_LAUNCH("fm_mask_sum");
  return 0;
}

int fm_flow_loss_fwd_bwd(const float* depth, const float* k4, const float* rt,
                         const float* forward_flow, const float* backward_flow,
                         const float* forward_mask, const float* backward_mask,
                         const double* mask_sum, int mapping, float delta, float loss_weight,
                         int intrinsics_mode, float* loss, float* g_depth, float* g_rt, float* g_k4,
                         void* ws, int B, int F, int H, int W, void* stream) {
  if (!depth || !k4 || !rt || !forward_flow || !backward_flow || !forward_mask || !backward_mask ||
      !mask_sum || !g_depth || !ws || bad_dims(B, F, H, W))
    return fail_msg("fm_flow_loss_fwd_bwd: bad arguments");
  if (mapping < 0 || mapping > 2) return fail_msg("fm_flow_loss_fwd_bwd: unknown mapping");
  if (intrinsics_mode < 0 || intrinsics_mode > 2) return fail_msg("fm_flow_loss_fwd_bwd: unknown intrinsics mode");
  cudaStream_t s = (cudaStream_t)stream;
  Workspace w = carve(ws, B, F);
  const int BP = B * (F - 1), BF = B * F;
  cudaError_t e = cudaMemsetAsync(w.flowacc, 0, (size_t)BF * kFlowAcc * sizeof(double), s);
  if (e != cudaSuccess) return fail("fm_flow_loss_fwd_bwd: memset", e);
  int rc = launch_flow(depth, k4, rt, forward_flow, backward_flow, forward_mask, backward_mask, mask_sum,
                       mapping, delta, loss_weight, intrinsics_mode, g_depth, w.flowacc, B, F, H, W, s);
  if (rc) return rc;
  const int n = BF > BP ? BF : BP;
  k_flow_finalize<<<(n + 127) / 128, 128, 0, s>>>(w.flowacc, rt, loss, g_rt, g_k4, B, F);
  FM_CHECK_LAUNCH("fm_flow_loss_fwd_bwd: k_flow_finalize");
  return 0;
}

int fm_pose_chain(const float* rt, float* extrinsics, int B, int F, void* stream) {
  if (!rt || !extrinsics || B < 1 || F < 2) return fail_msg("fm_pose_chain: bad arguments");
  k_pose_chain<<<B, kChainThreads, 0, (cudaStream_t)stream>>>(rt, extrinsics, B, F);
  FM_CHECK_LAUNCH("fm_pose_chain");
  return 0;
}

int fm_trajectory_ate(const float* gt, const float* pred, int T, int F, float* ate, float* aligned_gt,
                      float* aligned_pred, int* status, void* stream) {
  if (!gt || !pred || !ate || !status || T < 0 || F < 1) return fail_msg("fm_trajectory_ate: bad arguments");
  if (T == 0) return 0;
  MetricsRow none;
  memset(&none, 0, sizeof(none));
  k_trajectory_ate<<<T, kAteThreads, 0, (cudaStream_t)stream>>>(gt, pred, 3, 1, F, ate, aligned_gt, aligned_pred,
                                                                status, none);
  FM_CHECK_LAUNCH("fm_trajectory_ate");
  return 0;
}

int fm_pose_chain_bwd(const float* rt, const float* extrinsics, const float* g_extrinsics, float* g_rt,
                      int B, int F, void* stream) {
  if (!rt || !extrinsics || !g_extrinsics || !g_rt || B < 1 || F < 2) return fail_msg("fm_pose_chain_bwd: bad arguments");
  k_pose_chain_bwd<<<B, kChainThreads, 0, (cudaStream_t)stream>>>(rt, extrinsics, g_extrinsics, g_rt, B, F);
  FM_CHECK_LAUNCH("fm_pose_chain_bwd");
  return 0;
}

int fm_step_clock_tick(void* clock, double lr, double beta1, double beta2, unsigned long long base_seed,
                       int tick_focal, void* stream) {
  if (!clock) return fail_msg("fm_step_clock_tick: bad arguments");
  k_clock_tick<<<1, 1, 0, (cudaStream_t)stream>>>((StepClock*)clock, lr, beta1, beta2, base_seed, tick_focal);
  FM_CHECK_LAUNCH("fm_step_clock_tick");
  return 0;
}

int fm_adam_step_clock(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, size_t count,
                       const void* clock, int focal_clock, double beta1_d, double beta2_d, double eps_d,
                       void* stream) {
  if (!param || !grad || !exp_avg || !exp_avg_sq || !clock) return fail_msg("fm_adam_step_clock: bad arguments");
  if (count == 0) return 0;
  size_t nb = (count / 4 + kThreads * 2 - 1) / (kThreads * 2);
  if (nb < 1) nb = 1;
  if (nb > (size_t)sm_count_cached() * 16) nb = (size_t)sm_count_cached() * 16;
  const StepClock* c = (const StepClock*)clock;
  k_adam<<<(unsigned)nb, kThreads, 0, (cudaStream_t)stream>>>(
      param, grad, exp_avg, exp_avg_sq, count, (float)beta1_d, (float)beta2_d, (float)(1.0 - beta1_d),
      (float)(1.0 - beta2_d), (float)eps_d, 0.f, 1.f, focal_clock ? &c->focal_step_size : &c->step_size);
  FM_CHECK_LAUNCH("fm_adam_step_clock");
  return 0;
}

int fm_random_subset_clock(const void* clock, long long N, int n, int64_t* out, void* stream) {
  if (!clock || N < 1 || n < 1 || n > N || !out) return fail_msg("fm_random_subset_clock: bad arguments");
  k_random_subset<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(0ull, N, n, out, &((const StepClock*)clock)->seed);
  FM_CHECK_LAUNCH("fm_random_subset_clock");
  return 0;
}

int fm_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, size_t count,
                 double lr, double beta1_d, double beta2_d, double eps_d, int step, void* stream) {
  if (!param || !grad || !exp_avg || !exp_avg_sq || step < 1) return fail_msg("fm_adam_step: bad arguments");
  if (count == 0) return 0;
  const float beta1 = (float)beta1_d, beta2 = (float)beta2_d, eps = (float)eps_d;
  const double bc1 = 1.0 - pow(beta1_d, (double)step);
  const double bc2 = 1.0 - pow(beta2_d, (double)step);
  const float step_size = (float)(lr / bc1);
  const float bc2_sqrt = (float)sqrt(bc2);
  size_t nb = (count / 4 + kThreads * 2 - 1) / (kThreads * 2);
  if (nb < 1) nb = 1;
  if (nb > (size_t)sm_count_cached() * 16) nb = (size_t)sm_count_cached() * 16;
  k_adam<<<(unsigned)nb, kThreads, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, count, beta1, beta2, (float)(1.0 - (double)beta1_d), (float)(1.0 - (double)beta2_d), eps, step_size, bc2_sqrt);
  FM_CHECK_LAUNCH("fm_adam_step");
  return 0;
}

size_t fm_track_workspace_bytes(int F, long long total_samples) {
  if (F < 1 || total_samples < 0) return 0;
  size_t off = 0;
  off = align_up(off + 4 * sizeof(double), 256);                          // sums
  off = align_up(off + (size_t)F * kTrackAcc * sizeof(double), 256);      // per-frame accumulators
  off = align_up(off + (size_t)total_samples * 3 * sizeof(float), 256);   // unscaled point adjoints
  off = align_up(off + (size_t)total_samples, 256);                       // source-valid flags
  return off;
}

namespace {
// next_item: k_track_src's work counter, in the padding after the sums (zeroed with them)
struct TrackWs { double* sums; int* next_item; double* acc; float* dq; unsigned char* flag; };
TrackWs carve_track(void* base, int F, long long total) {
  char* p = (char*)base; size_t off = 0; TrackWs w;
  w.sums = (double*)(p + off); w.next_item = (int*)(p + off + 4 * sizeof(double));
  off = align_up(off + 4 * sizeof(double), 256);
  w.acc = (double*)(p + off); off = align_up(off + (size_t)F * kTrackAcc * sizeof(double), 256);
  w.dq = (float*)(p + off); off = align_up(off + (size_t)total * 3 * sizeof(float), 256);
  w.flag = (unsigned char*)(p + off);
  return w;
}
}  // namespace

size_t fm_track_reduce_bytes(int F) {
  if (F < 1) return 0;
  return align_up(4 * sizeof(double), 256) + align_up((size_t)F * kTrackAcc * sizeof(double), 256);
}

int fm_track_loss_fwd_sharded(const float* depth, const float* k4, const float* extrinsics, const int* segments,
                              int num_segments, int max_rows, int max_points, const float* track_xy,
                              const unsigned char* track_vis, long long total_samples, int mapping, float delta,
                              float loss_weight, float* loss, void* ws, int F, int H, int W, int depth_frame0,
                              int src_frame_lo, int src_frame_hi, int shared_intrinsics, void* stream) {
  if (!depth || !k4 || !extrinsics || !segments || !track_xy || !track_vis || !ws ||
      num_segments < 1 || max_rows < 1 || max_points < 1 || F < 1)
    return fail_msg("fm_track_loss_fwd: bad arguments");
  if (mapping < 0 || mapping > 2) return fail_msg("fm_track_loss_fwd: unknown mapping");
  if (depth_frame0 < 0 || src_frame_lo < depth_frame0 || src_frame_hi > F || src_frame_lo > src_frame_hi)
    return fail_msg("fm_track_loss_fwd: bad source-frame range");
  cudaStream_t s = (cudaStream_t)stream;
  TrackWs w = carve_track(ws, F, total_samples);
  // sums, work counter, accumulators
  cudaError_t e = cudaMemsetAsync(w.sums, 0, (char*)w.dq - (char*)w.sums, s);
  if (e != cudaSuccess) return fail("fm_track_loss_fwd: memset", e);
  const int list_cap = max_points < kTrackListCap ? max_points : kTrackListCap;
  const size_t smem = track_smem_bytes(max_rows, list_cap);
  if (smem > 200 * 1024) return fail_msg("fm_track_loss_fwd: segment too long for shared memory");
  // a persistent grid: as many blocks as fit on the GPU at once (registers or shared memory)
  const long long items = (long long)num_segments * max_rows * kTrackParts;
  if (items > INT_MAX) return fail_msg("fm_track_loss_fwd: too many segment rows");
  int per_sm = (int)((227 * 1024) / (smem + sizeof(double) * kTrackAcc * (kTrackThreads / 32) + 1024 + 64));
  if (per_sm > FM_TRACK_BPS) per_sm = FM_TRACK_BPS;
  if (per_sm < 1) per_sm = 1;
  const int grid = persistent_grid(per_sm, items);
  if (smem > 48 * 1024) {
    cudaError_t ea = shared_intrinsics
        ? cudaFuncSetAttribute(k_track_src<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
        : cudaFuncSetAttribute(k_track_src<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (ea != cudaSuccess) return fail("fm_track_loss_fwd: shared memory", ea);
  }
  const TrackShard sh = {depth_frame0, src_frame_lo, src_frame_hi};
  if (shared_intrinsics)
    k_track_src<true><<<grid, kTrackThreads, smem, s>>>(depth, k4, extrinsics, segments, track_xy, track_vis, mapping,
                                                        delta, w.sums, w.flag, w.dq, w.acc, w.next_item, (int)items,
                                                        max_rows, list_cap, H, W, sh);
  else
    k_track_src<false><<<grid, kTrackThreads, smem, s>>>(depth, k4, extrinsics, segments, track_xy, track_vis, mapping,
                                                         delta, w.sums, w.flag, w.dq, w.acc, w.next_item, (int)items,
                                                         max_rows, list_cap, H, W, sh);
  FM_CHECK_LAUNCH("fm_track_loss_fwd: k_track_src");
  if (loss) {
    k_track_loss<<<1, 1, 0, s>>>(w.sums, loss_weight, loss);
    FM_CHECK_LAUNCH("fm_track_loss_fwd: k_track_loss");
  }
  return 0;
}

int fm_track_loss_fwd(const float* depth, const float* k4, const float* extrinsics, const int* segments,
                      int num_segments, int max_rows, int max_points, const float* track_xy,
                      const unsigned char* track_vis, long long total_samples, int mapping, float delta,
                      float loss_weight, float* loss, void* ws, int F, int H, int W, void* stream) {
  if (!loss) return fail_msg("fm_track_loss_fwd: bad arguments");
  return fm_track_loss_fwd_sharded(depth, k4, extrinsics, segments, num_segments, max_rows, max_points, track_xy,
                                   track_vis, total_samples, mapping, delta, loss_weight, loss, ws, F, H, W, 0,
                                   0, F, 0, stream);
}

int fm_track_loss_value(const void* ws, float loss_weight, float* loss, void* stream) {
  if (!ws || !loss) return fail_msg("fm_track_loss_value: bad arguments");
  k_track_loss<<<1, 1, 0, (cudaStream_t)stream>>>((const double*)ws, loss_weight, loss);
  FM_CHECK_LAUNCH("fm_track_loss_value");
  return 0;
}

// The depth scatter of the tracking loss (k_track_apply, REDs into g_depth) and the pose / intrinsics
// gradients (k_track_finalize) are independent: `apply_stream` may differ from `s`.
static int track_bwd_impl(const float* k4, const float* extrinsics, const int* segments, int num_segments,
                          int max_rows, int max_points, const float* track_xy, long long total_samples,
                          float loss_weight, const float* grad_out, float* g_depth, float* g_extrinsics,
                          float* g_k4, void* ws, int F, int H, int W, int depth_frame0, int src_frame_lo,
                          int src_frame_hi, cudaStream_t s, cudaStream_t apply_stream) {
  if (!k4 || !extrinsics || !segments || !track_xy || !g_depth || !g_extrinsics || !g_k4 || !ws ||
      num_segments < 1 || max_rows < 1 || max_points < 1 || F < 1)
    return fail_msg("fm_track_loss_bwd: bad arguments");
  if (depth_frame0 < 0 || src_frame_lo < depth_frame0 || src_frame_hi > F || src_frame_lo > src_frame_hi)
    return fail_msg("fm_track_loss_bwd: bad source-frame range");
  TrackWs w = carve_track(ws, F, total_samples);
  dim3 grid((max_points + kThreads - 1) / kThreads, max_rows, num_segments);
  const TrackShard sh = {depth_frame0, src_frame_lo, src_frame_hi};
  k_track_apply<<<grid, kThreads, 0, apply_stream>>>(k4, segments, track_xy, w.flag, w.dq, w.sums, loss_weight,
                                                    grad_out, g_depth, H, W, sh);
  FM_CHECK_LAUNCH("fm_track_loss_bwd: k_track_apply");
  k_track_finalize<<<(F + 63) / 64, 64, 0, s>>>(w.acc, w.sums, loss_weight, grad_out, extrinsics, g_extrinsics,
                                               g_k4, F);
  FM_CHECK_LAUNCH("fm_track_loss_bwd: k_track_finalize");
  return 0;
}

int fm_track_loss_bwd_sharded(const float* depth, const float* k4, const float* extrinsics, const int* segments,
                              int num_segments, int max_rows, int max_points, const float* track_xy,
                              const unsigned char* track_vis, long long total_samples, int mapping, float delta,
                              float loss_weight, const float* grad_out, float* g_depth, float* g_extrinsics,
                              float* g_k4, void* ws, int F, int H, int W, int depth_frame0, int src_frame_lo,
                              int src_frame_hi, void* stream) {
  (void)depth; (void)track_vis; (void)mapping; (void)delta;
  return track_bwd_impl(k4, extrinsics, segments, num_segments, max_rows, max_points, track_xy, total_samples,
                        loss_weight, grad_out, g_depth, g_extrinsics, g_k4, ws, F, H, W, depth_frame0,
                        src_frame_lo, src_frame_hi, (cudaStream_t)stream, (cudaStream_t)stream);
}

int fm_track_loss_bwd(const float* depth, const float* k4, const float* extrinsics, const int* segments,
                      int num_segments, int max_rows, int max_points, const float* track_xy,
                      const unsigned char* track_vis, long long total_samples, int mapping, float delta,
                      float loss_weight, const float* grad_out, float* g_depth, float* g_extrinsics,
                      float* g_k4, void* ws, int F, int H, int W, void* stream) {
  return fm_track_loss_bwd_sharded(depth, k4, extrinsics, segments, num_segments, max_rows, max_points, track_xy,
                                   track_vis, total_samples, mapping, delta, loss_weight, grad_out, g_depth,
                                   g_extrinsics, g_k4, ws, F, H, W, 0, 0, F, stream);
}

size_t fm_points_workspace_bytes(int items) {
  if (items < 1) return 0;
  return carve(nullptr, items, 2).bytes;
}

int fm_align_rigid_fwd(const float* p, const float* q, const float* weights, float* rt, void* ws, int items,
                       int n, void* stream) {
  if (!p || !q || !weights || !rt || !ws || items < 1 || n < 1) return fail_msg("fm_align_rigid_fwd: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  Workspace w = carve(ws, items, 2);
  cudaError_t e = cudaMemsetAsync(w.moments, 0, (size_t)items * kNumMoments * sizeof(double), s);
  if (e != cudaSuccess) return fail("fm_align_rigid_fwd: memset", e);
  k_points_shift<<<items, kThreads, 0, s>>>(p, q, weights, w.pshift, n);
  FM_CHECK_LAUNCH("fm_align_rigid_fwd: k_points_shift");
  dim3 grid(blocks_for(n, 1), items);
  k_points_moments<<<grid, kThreads, 0, s>>>(p, q, weights, w.pshift, w.moments, n);
  FM_CHECK_LAUNCH("fm_align_rigid_fwd: k_points_moments");
  k_points_solve<<<(items + 63) / 64, 64, 0, s>>>(w.moments, w.pshift, rt, w.state, items);
  FM_CHECK_LAUNCH("fm_align_rigid_fwd: k_points_solve");
  return 0;
}

int fm_align_rigid_bwd(const float* p, const float* q, const float* weights, const float* g_rt, float* g_p,
                       float* g_q, float* g_w, void* ws, int items, int n, void* stream) {
  if (!p || !q || !weights || !g_rt || !g_p || !g_q || !g_w || !ws || items < 1 || n < 1)
    return fail_msg("fm_align_rigid_bwd: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  Workspace w = carve(ws, items, 2);
  // items "pairs" of a 2-frame layout: k_adjoint indexes state / adj by pair
  k_adjoint<<<(items + 63) / 64, 64, 0, s>>>(w.flowacc, w.state, g_rt, 0, nullptr, w.adj, items, 2);
  FM_CHECK_LAUNCH("fm_align_rigid_bwd: k_adjoint");
  dim3 grid(blocks_for(n, 1), items);
  k_points_distribute<<<grid, kThreads, 0, s>>>(p, q, weights, w.adj, g_p, g_q, g_w, n);
  FM_CHECK_LAUNCH("fm_align_rigid_bwd: k_points_distribute");
  return 0;
}

int fm_unproject_points(const float* xy, const float* z, const float* k4, float* out, int items, int n,
                        int xy_shared, void* stream) {
  if (!xy || !z || !k4 || !out || items < 1 || n < 1) return fail_msg("fm_unproject_points: bad arguments");
  dim3 grid(blocks_for(n, 1), items);
  k_unproject_points<<<grid, kThreads, 0, (cudaStream_t)stream>>>(xy, z, k4, out, n, xy_shared);
  FM_CHECK_LAUNCH("fm_unproject_points");
  return 0;
}

int fm_unproject_points_bwd(const float* xy, const float* z, const float* k4, const float* g_out, float* g_z,
                            float* g_k4, void* ws, int items, int n, int xy_shared, void* stream) {
  if (!xy || !z || !k4 || !g_out || !g_z || !g_k4 || !ws || items < 1 || n < 1)
    return fail_msg("fm_unproject_points_bwd: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  Workspace w = carve(ws, items, 2);  // k4acc has 2 * items rows; the first `items` are used
  cudaError_t e = cudaMemsetAsync(w.k4acc, 0, (size_t)items * 4 * sizeof(double), s);
  if (e != cudaSuccess) return fail("fm_unproject_points_bwd: memset", e);
  dim3 grid(blocks_for(n, 1), items);
  k_unproject_points_bwd<<<grid, kThreads, 0, s>>>(xy, z, k4, g_out, g_z, w.k4acc, n, xy_shared);
  FM_CHECK_LAUNCH("fm_unproject_points_bwd: k_unproject_points_bwd");
  k_d2f<<<(items * 4 + 127) / 128, 128, 0, s>>>(w.k4acc, g_k4, items * 4);
  FM_CHECK_LAUNCH("fm_unproject_points_bwd: k_d2f");
  return 0;
}

int fm_random_subset(unsigned long long seed, long long N, int n, int64_t* out, void* stream) {
  if (!out || N < 1 || n < 1 || n > N || N > (1ll << 40)) return fail_msg("fm_random_subset: bad arguments");
  k_random_subset<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(seed, N, n, out);
  FM_CHECK_LAUNCH("fm_random_subset");
  return 0;
}

size_t fm_softmin_workspace_bytes(int B, int num_candidates) {
  if (B < 1 || num_candidates < 1) return 0;
  const size_t items = (size_t)B * num_candidates;  // + B rows for the shared (candidate-0) quantities
  return align_up(carve(nullptr, (int)(items + B), 2).bytes, 256) +
         align_up((items * 12 + (items + B) * 8) * sizeof(float), 256);
}

namespace {
PairLayout sweep_layout(int F, int H, int W, int cand) {
  PairLayout l = dense_layout(F, H, W);  // strides of the REAL tensors
  l.F = 2;                               // the sweep only sees frames 0 and 1 (pair 0)
  l.cand = cand;
  return l;
}
}  // namespace

int fm_softmin_sweep_fwd(const float* depth, const float* weights, float weight_sensitivity,
                         const float* backward_flow, const int64_t* indices, int num_indices,
                         const float* cand_k4, int num_candidates, float* err, float* rt, void* ws, int B,
                         int F, int H, int W, void* stream) {
  if (!depth || !backward_flow || !indices || num_indices < 1 || !cand_k4 || num_candidates < 1 ||
      !err || !rt || !ws || bad_dims(B, F, H, W))
    return fail_msg("fm_softmin_sweep_fwd: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  const int items = B * num_candidates;
  const PairLayout lay = sweep_layout(F, H, W, num_candidates);
  const PairLayout lay1 = sweep_layout(F, H, W, 1);
  Workspace w = carve(ws, items + B, 2);
  float* scratch = (float*)((char*)ws + align_up(w.bytes, 256));
  float* base_k4 = scratch + (size_t)items * 12 + (size_t)items * 8;  // after g_rt and g_k4 of the bwd
  double* base_moments = w.moments + (size_t)items * kNumMoments;
  cudaError_t e = cudaMemsetAsync(base_moments, 0, (size_t)B * kNumMoments * sizeof(double), s);
  if (e != cudaSuccess) return fail("fm_softmin_sweep_fwd: memset", e);
  k_sweep_base_k4<<<(B * 8 + 127) / 128, 128, 0, s>>>(cand_k4, base_k4, B, num_candidates);
  FM_CHECK_LAUNCH("fm_softmin_sweep_fwd: k_sweep_base_k4");
  float* base_zshift = w.zshift + items;  // one conditioning shift per batch element, for all candidates
  k_pair_shift<<<B, kThreads, 0, s>>>(depth, weights, weight_sensitivity, base_zshift, lay1, H, W);
  FM_CHECK_LAUNCH("fm_softmin_sweep_fwd: k_pair_shift");
  {  // ONE moment pass (candidate 0); every candidate's moments are a rescaling of it
    dim3 grid(blocks_for_points(num_indices), B);
    k_moments<1><<<grid, kThreads, 0, s>>>(depth, base_k4, backward_flow, weights, indices, num_indices,
                                          base_moments, base_zshift, weight_sensitivity, lay1, H, W);
    FM_CHECK_LAUNCH("fm_softmin_sweep_fwd: k_moments");
  }
  k_sweep_scale_solve<<<(items + 63) / 64, 64, 0, s>>>(base_moments, base_zshift, cand_k4, rt, w.state, B,
                                                      num_candidates);
  FM_CHECK_LAUNCH("fm_softmin_sweep_fwd: k_sweep_scale_solve");
  e = cudaMemsetAsync(w.flowacc, 0, (size_t)items * kSweepAcc * sizeof(double), s);
  if (e != cudaSuccess) return fail("fm_softmin_sweep_fwd: memset", e);
  dim3 grid(blocks_for_points(num_indices), items);
  k_sweep<false><<<grid, kThreads, 0, s>>>(depth, cand_k4, rt, backward_flow, weights, weight_sensitivity,
                                          indices, num_indices, nullptr, w.flowacc, nullptr, nullptr, lay,
                                          H, W);
  FM_CHECK_LAUNCH("fm_softmin_sweep_fwd: k_sweep");
  k_sweep_out<<<(items + 127) / 128, 128, 0, s>>>(w.flowacc, err, items, 0, 1);
  FM_CHECK_LAUNCH("fm_softmin_sweep_fwd: k_sweep_out");
  return 0;
}

int fm_softmin_sweep_bwd(const float* depth, const float* weights, float weight_sensitivity,
                         const float* backward_flow, const int64_t* indices, int num_indices,
                         const float* cand_k4, int num_candidates, const float* rt, const float* g_err,
                         float* g_depth, float* g_weights, void* ws, int B, int F, int H, int W,
                         void* stream) {
  if (!depth || !backward_flow || !indices || num_indices < 1 || !cand_k4 || num_candidates < 1 || !rt ||
      !g_err || !g_depth || !ws || bad_dims(B, F, H, W))
    return fail_msg("fm_softmin_sweep_bwd: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  const int items = B * num_candidates;
  const PairLayout lay = sweep_layout(F, H, W, num_candidates);
  const PairLayout lay1 = sweep_layout(F, H, W, 1);
  Workspace w = carve(ws, items + B, 2);
  float* scratch = (float*)((char*)ws + align_up(w.bytes, 256));
  float* g_rt = scratch;
  float* base_k4 = scratch + (size_t)items * 12 + (size_t)items * 8;
  cudaError_t e = cudaMemsetAsync(w.flowacc, 0, (size_t)items * kSweepAcc * sizeof(double), s);
  if (e != cudaSuccess) return fail("fm_softmin_sweep_bwd: memset", e);
  e = cudaMemsetAsync(w.k4acc, 0, (size_t)(items + B) * 2 * 4 * sizeof(double), s);
  if (e != cudaSuccess) return fail("fm_softmin_sweep_bwd: memset", e);
  dim3 grid(blocks_for_points(num_indices), items);
  k_sweep<true><<<grid, kThreads, 0, s>>>(depth, cand_k4, rt, backward_flow, weights, weight_sensitivity,
                                         indices, num_indices, g_err, w.flowacc, g_depth, g_weights, lay, H,
                                         W);
  FM_CHECK_LAUNCH("fm_softmin_sweep_bwd: k_sweep");
  k_sweep_out<<<(items * 12 + 127) / 128, 128, 0, s>>>(w.flowacc, g_rt, items, 1, 12);
  FM_CHECK_LAUNCH("fm_softmin_sweep_bwd: k_sweep_out");
  // per-candidate adjoint constants, collapsed into one per batch element, then ONE distribution pass
  k_adjoint<<<(items + 63) / 64, 64, 0, s>>>(w.flowacc, w.state, g_rt, 0, nullptr, w.adj, items, 2);
  FM_CHECK_LAUNCH("fm_softmin_sweep_bwd: k_adjoint");
  k_sweep_aggregate<<<B, 32, 0, s>>>(w.adj, cand_k4, w.adj + items, B, num_candidates);
  FM_CHECK_LAUNCH("fm_softmin_sweep_bwd: k_sweep_aggregate");
  AdamFuse af;
  memset(&af, 0, sizeof(af));
  dim3 grid1(blocks_for_points(num_indices), B);
  k_distribute<1><<<grid1, kThreads, 0, s>>>(depth, base_k4, backward_flow, const_cast<float*>(weights), indices,
                                            num_indices, w.adj + items, g_depth, g_weights, w.k4acc,
                                            weight_sensitivity, lay1, af, H, W);
  FM_CHECK_LAUNCH("fm_softmin_sweep_bwd: k_distribute");
  return 0;
}

int fm_softmin_focal(const float* err, const float* cand_focal, int num_candidates, int B, float* softmin,
                     float* focal, void* stream) {
  if (!err || !cand_focal || !softmin || !focal || B < 1 || num_candidates < 1)
    return fail_msg("fm_softmin_focal: bad arguments");
  k_softmin_focal<<<B, 32, 0, (cudaStream_t)stream>>>(err, cand_focal, num_candidates, softmin, focal);
  FM_CHECK_LAUNCH("fm_softmin_focal");
  return 0;
}

int fm_softmin_focal_bwd(const float* softmin, const float* cand_focal, const float* focal,
                         const float* g_focal, int num_candidates, int B, float* g_err, void* stream) {
  if (!softmin || !cand_focal || !focal || !g_focal || !g_err || B < 1 || num_candidates < 1)
    return fail_msg("fm_softmin_focal_bwd: bad arguments");
  const int n = B * num_candidates;
  k_softmin_focal_bwd<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(softmin, cand_focal, focal, g_focal,
                                                                        num_candidates, B, g_err);
  FM_CHECK_LAUNCH("fm_softmin_focal_bwd");
  return 0;
}

// A second stream (per device) for work that only has to be finished when the step ends: forked
// from / joined to the caller's stream with events, so it is captured into the caller's CUDA graph as
// a parallel branch.
struct SideLane { cudaStream_t stream; cudaEvent_t fork, join; int state; };  // state 0 new, 1 ready, -1 unavailable
// One lane per (host thread, device): a thread's calls are sequential, so its events are never
// re-recorded while a wait on them is still to be issued; other threads have their own.  The lane is
// created on the first call that uses it (an eager warm-up step, not inside a capture).  Lane 0
// carries the tracking work, lane 1 the metrics log, which overlaps all of it.
static SideLane* side_lane(int which = 0) {
  static thread_local SideLane lanes[2][64];
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  SideLane& l = lanes[which][dev];
  if (l.state == 0) {
    const bool ok = cudaStreamCreateWithFlags(&l.stream, cudaStreamNonBlocking) == cudaSuccess &&
                    cudaEventCreateWithFlags(&l.fork, cudaEventDisableTiming) == cudaSuccess &&
                    cudaEventCreateWithFlags(&l.join, cudaEventDisableTiming) == cudaSuccess;
    l.state = ok ? 1 : -1;
    if (!ok) (void)cudaGetLastError();
  }
  return l.state == 1 ? &l : nullptr;
}

int fm_overfit_step(const fm_overfit_step_args* a, void* stream) {
  if (!a || !a->depth || !a->fflow || !a->bflow || !a->fmask || !a->bmask || !a->mask_sum ||
      !a->g_depth || !a->rt || !a->loss || !a->ws || !a->k4 || bad_dims(1, a->F, a->H, a->W))
    return fail_msg("fm_overfit_step: bad arguments");
  if (a->weight_logits && !a->g_weights) return fail_msg("fm_overfit_step: g_weights missing");
  if (a->tracks && (!a->extrinsics || !a->g_extrinsics || !a->track_ws || !a->track_loss))
    return fail_msg("fm_overfit_step: tracking needs extrinsics / g_extrinsics / track_ws / track_loss");
  if (a->metrics_log && (a->phase != FM_STEP_ALL || !a->clock || !a->extrinsics || a->metrics_capacity < 1))
    return fail_msg("fm_overfit_step: metrics_log needs FM_STEP_ALL, a clock, extrinsics and metrics_capacity >= 1");
  cudaStream_t s = (cudaStream_t)stream;
  const int F = a->F, H = a->H, W = a->W, BP = F - 1;
  const size_t N = (size_t)H * W;
  Workspace w = carve(a->ws, 1, F);
  int rc;
  cudaError_t e;
  if (a->phase < FM_STEP_ALL || a->phase > FM_STEP_BACKWARD) return fail_msg("fm_overfit_step: unknown phase");
  // the splat plan of this video's backward flows serves the dense path (all-pixel Procrustes)
  void* plan = (a->splat_plan && !a->indices && tiled_shape_ok(F, H, W)) ? a->splat_plan : nullptr;
  // intrinsics from the focal parameter (regressed stage) or as given
  float* k4 = a->k4;
  if (a->phase != FM_STEP_BACKWARD) {
    if (a->focal) {
      k_k4_from_focal<<<(F + 63) / 64, 64, 0, s>>>(a->focal, k4, F, H, W);
      FM_CHECK_LAUNCH("fm_overfit_step: k_k4_from_focal");
    }
    // Model.forward: Procrustes poses (model.py:54-90)
    if ((rc = procrustes_fwd_impl(a->depth, k4, a->bflow, a->weight_logits, a->weight_sensitivity,
                                  a->indices, a->num_indices, a->rt, a->ws, 1, F, H, W, stream, nullptr, plan,
                                  (a->indices || plan) ? nullptr : a->moments_k4)))
      return rc;
    // The flow loss and the tracking sweep both need only the poses: with tracking on they run as
    // two branches of the step (the tracking sweep is issue-bound, the flow kernel waits on memory:
    // where blocks of both share an SM they fill each other's idle slots).
    SideLane* fwd_lane = a->tracks ? side_lane() : nullptr;
    if (fwd_lane) {
      if ((e = cudaEventRecord(fwd_lane->fork, s)) != cudaSuccess) return fail("fm_overfit_step: fork", e);
      if ((e = cudaStreamWaitEvent(fwd_lane->stream, fwd_lane->fork, 0)) != cudaSuccess) return fail("fm_overfit_step: fork", e);
    }
    // LossFlow forward + direct gradients (loss_flow.py:31-70)
    e = cudaMemsetAsync(w.flowacc, 0, (size_t)F * kFlowAcc * sizeof(double), s);
    if (e != cudaSuccess) return fail("fm_overfit_step: memset", e);
    if ((rc = launch_flow(a->depth, k4, a->rt, a->fflow, a->bflow, a->fmask, a->bmask, a->mask_sum,
                          a->mapping, a->delta, a->flow_weight, a->focal ? 1 : 2, a->g_depth, w.flowacc, 1, F,
                          H, W, s)))
      return rc;
    k_flow_finalize<<<(F + 127) / 128, 128, 0, s>>>(w.flowacc, a->rt, a->loss, nullptr, nullptr, 1, F);
    FM_CHECK_LAUNCH("fm_overfit_step: k_flow_finalize");
    // LossTracking (loss_tracking.py:28-61) on the chained poses: the forward sweep belongs to the
    // forward half of a split step, its scaling / scatter to the backward half
    if (a->tracks) {
      const fm_packed_tracks* t = a->tracks;
      void* ts = fwd_lane ? (void*)fwd_lane->stream : stream;
      if ((rc = fm_pose_chain(a->rt, a->extrinsics, 1, F, ts))) return rc;
      // one focal length (or constant intrinsics) for all frames: only the summed K gradient is used
      if ((rc = fm_track_loss_fwd_sharded(a->depth, k4, a->extrinsics, t->segments, t->num_segments, t->max_rows,
                                          t->max_points, t->xy, t->vis, t->total_samples, a->mapping, a->delta,
                                          a->track_weight, a->track_loss, a->track_ws, F, H, W, 0, 0, F, 1, ts)))
        return rc;
      if (fwd_lane) {
        if ((e = cudaEventRecord(fwd_lane->join, fwd_lane->stream)) != cudaSuccess) return fail("fm_overfit_step: join", e);
        if ((e = cudaStreamWaitEvent(s, fwd_lane->join, 0)) != cudaSuccess) return fail("fm_overfit_step: join", e);
      }
    }
  }
  // The metrics row of this step (model_wrapper_overfit.py:63-71 and metrics/ate): it reads only what
  // the forward half produced and the rest of the step does not change (losses, k4, chained poses), so
  // it runs on its own lane beside the backward and Adam and is joined before the call returns.
  SideLane* mlane = nullptr;
  if (a->metrics_log) {
    mlane = side_lane(1);
    cudaStream_t ms = s;
    if (mlane) {
      if ((e = cudaEventRecord(mlane->fork, s)) != cudaSuccess) return fail("fm_overfit_step: fork", e);
      if ((e = cudaStreamWaitEvent(mlane->stream, mlane->fork, 0)) != cudaSuccess) return fail("fm_overfit_step: fork", e);
      ms = mlane->stream;
    }
    // the camera centres: the tracking loss chained the poses already, a flow-only step chains them here
    if (!a->tracks && (rc = fm_pose_chain(a->rt, a->extrinsics, 1, F, ms))) return rc;
    MetricsRow row;
    row.log = a->metrics_log;
    row.capacity = a->metrics_capacity;
    row.clock = (const StepClock*)a->clock;
    row.loss = a->loss;
    row.track_loss = a->tracks ? a->track_loss : nullptr;
    row.k4 = k4;
    row.gt_fx = a->gt_fx;
    row.gt_fy = a->gt_fy;
    k_trajectory_ate<<<1, kAteThreads, 0, ms>>>(a->gt_positions, a->extrinsics + 3, 16, 4, F, nullptr, nullptr, nullptr,
                                                nullptr, row);
    FM_CHECK_LAUNCH("fm_overfit_step: k_trajectory_ate");
    if (mlane && (e = cudaEventRecord(mlane->join, mlane->stream)) != cudaSuccess) return fail("fm_overfit_step: join", e);
  }
  if (a->phase == FM_STEP_FORWARD) return 0;
  // d total / d (flow loss) and d total / d (tracking loss) of a split step (device scalars, NULL = 1)
  const float* fscale = a->phase == FM_STEP_BACKWARD ? a->flow_grad_scale : nullptr;
  const float* tscale = a->phase == FM_STEP_BACKWARD ? a->track_grad_scale : nullptr;
  if (fscale) {  // the direct flow-loss gradient in g_depth was computed for scale 1; scale it before
    // the tracking loss adds its own (differently scaled) part
    k_scale_inplace<<<sm_count_cached() * 4, kThreads, 0, s>>>(a->g_depth, fscale, (size_t)F * N);
    FM_CHECK_LAUNCH("fm_overfit_step: k_scale_inplace");
  }
  const float* g_rt = a->phase == FM_STEP_BACKWARD ? a->g_rt : nullptr;           // the caller's
  const float* track_g_k4 = a->phase == FM_STEP_BACKWARD ? a->track_g_k4 : nullptr;  // tracking part
  SideLane* lane = nullptr;  // carries the tracking loss's depth scatter while the Procrustes backward runs
  if (a->tracks) {
    const fm_packed_tracks* t = a->tracks;
    // REDs into g_depth commute with those of k_distribute; the splat-plan backward instead rewrites
    // g_depth with plain stores, so there the scatter stays in stream order
    if (!plan) lane = side_lane();
    cudaStream_t apply_stream = s;
    if (lane) {
      if ((e = cudaEventRecord(lane->fork, s)) != cudaSuccess) return fail("fm_overfit_step: fork", e);
      if ((e = cudaStreamWaitEvent(lane->stream, lane->fork, 0)) != cudaSuccess) return fail("fm_overfit_step: fork", e);
      apply_stream = lane->stream;
    }
    if ((rc = track_bwd_impl(k4, a->extrinsics, t->segments, t->num_segments, t->max_rows, t->max_points, t->xy,
                             t->total_samples, a->track_weight, tscale, a->g_depth, a->g_extrinsics, a->track_g_k4,
                             a->track_ws, F, H, W, 0, 0, F, s, apply_stream)))
      return rc;
    if (lane && (e = cudaEventRecord(lane->join, lane->stream)) != cudaSuccess) return fail("fm_overfit_step: join", e);
    if ((rc = fm_pose_chain_bwd(a->rt, a->extrinsics, a->g_extrinsics, a->g_rt, 1, F, stream))) return rc;
    g_rt = a->g_rt;
    track_g_k4 = a->track_g_k4;
  }
  // backward through Procrustes: adjoint constants, per-point distribution
  if (a->indices && a->g_weights) {  // subsampled Procrustes: sparse weight gradient, dense buffer
    e = cudaMemsetAsync(a->g_weights, 0, (size_t)BP * N * sizeof(float), s);
    if (e != cudaSuccess) return fail("fm_overfit_step: memset g_weights", e);
  }
  AdamFuse af;
  memset(&af, 0, sizeof(af));
  const bool defer = a->defer_adam != 0;  // softmin stage: the sweep's backward still adds gradients
  const bool fuse_w = a->step > 0 && a->weight_logits && !a->indices && W % 4 == 0;
  const StepClock* clock = (const StepClock*)a->clock;
  if (fuse_w) {  // the weight gradient is final inside k_distribute: update the logits there
    af.consts = clock ? &clock->step_size : nullptr;
    af.on = 1; af.m = a->m_weights; af.v = a->v_weights;
    af.first_pair = a->defer_adam == 1 ? 1 : 0;  // 1: the sweep still touches pair 0; 2: every pair is final
    af.beta1 = (float)a->beta1; af.beta2 = (float)a->beta2;
    af.omb1 = (float)(1.0 - a->beta1); af.omb2 = (float)(1.0 - a->beta2); af.eps = (float)a->eps;
    af.step_size = (float)(a->lr / (1.0 - pow(a->beta1, (double)a->step)));
    af.bc2_sqrt = (float)sqrt(1.0 - pow(a->beta2, (double)a->step));
  }
  if ((rc = procrustes_bwd_impl(a->depth, k4, a->bflow, a->weight_logits, a->weight_sensitivity,
                                a->indices, a->num_indices, g_rt, 1, fscale, a->g_depth, a->g_weights,
                                a->g_k4, a->ws, 1, F, H, W, stream, nullptr, fuse_w ? &af : nullptr, plan,
                                a->splat_overflow_max, /*depth_prescaled=*/fscale != nullptr)))
    return rc;
  if (lane && (e = cudaStreamWaitEvent(s, lane->join, 0)) != cudaSuccess) return fail("fm_overfit_step: join", e);
  // Adam (model_wrapper_overfit.py:104-105)
  if (a->step > 0 && !defer) {
    auto adam = [&](float* p, const float* g, float* m, float* v, size_t n, int step, int focal_clock) -> int {
      return clock ? fm_adam_step_clock(p, g, m, v, n, clock, focal_clock, a->beta1, a->beta2, a->eps, stream)
                   : fm_adam_step(p, g, m, v, n, a->lr, a->beta1, a->beta2, a->eps, step, stream);
    };
    if ((rc = adam(a->depth, a->g_depth, a->m_depth, a->v_depth, (size_t)F * N, a->step, 0))) return rc;
    if (a->weight_logits && !fuse_w &&
        (rc = adam(a->weight_logits, a->g_weights, a->m_weights, a->v_weights, (size_t)BP * N, a->step, 0)))
      return rc;
    if (a->focal) {
      k_focal_grad<<<1, 256, 0, s>>>(w.k4acc, w.flowacc, track_g_k4, a->g_focal, 1, F, H, W, fscale);
      FM_CHECK_LAUNCH("fm_overfit_step: k_focal_grad");
      if ((rc = adam(a->focal, a->g_focal, a->m_focal, a->v_focal, 1, a->focal_step > 0 ? a->focal_step : a->step, 1)))
        return rc;
    }
  } else if (a->focal) {
    k_focal_grad<<<1, 256, 0, s>>>(w.k4acc, w.flowacc, track_g_k4, a->g_focal, 1, F, H, W, fscale);
    FM_CHECK_LAUNCH("fm_overfit_step: k_focal_grad");
  }
  if (defer && a->step > 0 && a->weight_logits && !fuse_w) return fail_msg("fm_overfit_step: defer_adam needs the fused weight update");
  if (mlane && (e = cudaStreamWaitEvent(s, mlane->join, 0)) != cudaSuccess) return fail("fm_overfit_step: join", e);
  return 0;
}

}  // extern "C"
