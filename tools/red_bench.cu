// Micro-benchmark: throughput of fire-and-forget float adds (RED) on the GPU for the access
// patterns of the Procrustes-adjoint scatter (tools only).
#include <cstdio>
#include <cuda_runtime.h>
#include <vector>

__device__ __forceinline__ void red1(float* a, float v) { asm volatile("red.global.add.f32 [%0], %1;" ::"l"(a), "f"(v) : "memory"); }
__device__ __forceinline__ void red2(float* a, float v0, float v1) { asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(a), "f"(v0), "f"(v1) : "memory"); }
__device__ __forceinline__ void red4(float* a, float v0, float v1, float v2, float v3) { asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a), "f"(v0), "f"(v1), "f"(v2), "f"(v3) : "memory"); }

__device__ __forceinline__ unsigned hash(unsigned x) { x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16; return x; }

// mode 0: 4 scalar reds at bilinear taps of a jittered position (jitter +-J px)
// mode 1: v2 when x0 even else 2 scalars (per row)
// mode 2: v4 padded when x0 % 4 != 3 else 2 scalars (per row)
// mode 3: aligned coalesced scalar red (1 per pixel)
// mode 4: aligned coalesced v4 red (1 per 4 pixels)
// mode 5: plain float4 store
// mode 6: 4 scalar reds, but no jitter (smooth flow): taps of neighbouring lanes overlap
template <int MODE>
__global__ void k(float* out, int H, int W, int J, int frames) {
  const int N = H * W;
  for (int f = blockIdx.y; f < frames; f += gridDim.y) {
    float* o = out + (size_t)f * N;
    for (int base = (blockIdx.x * blockDim.x + threadIdx.x) * 4; base < N; base += gridDim.x * blockDim.x * 4) {
      const int r = base / W, c0 = base - r * W;
      if (MODE == 3) { for (int v = 0; v < 4; ++v) red1(o + base + v, 1.f); continue; }
      if (MODE == 4) { red4(o + base, 1.f, 1.f, 1.f, 1.f); continue; }
      if (MODE == 5) { *reinterpret_cast<float4*>(o + base) = make_float4(1.f, 1.f, 1.f, 1.f); continue; }
      for (int v = 0; v < 4; ++v) {
        unsigned h = hash((unsigned)(f * N + base + v));
        int dx = (MODE == 6) ? 3 : (int)(h % (2 * J + 1)) - J, dy = (MODE == 6) ? -2 : (int)((h >> 12) % (2 * J + 1)) - J;
        int x0 = min(max(c0 + v + dx, 0), W - 2), y0 = min(max(r + dy, 0), H - 2);
        float* p0 = o + y0 * W + x0; float* p1 = p0 + W;
        if (MODE == 0 || MODE == 6) { red1(p0, .25f); red1(p0 + 1, .25f); red1(p1, .25f); red1(p1 + 1, .25f); }
        if (MODE == 1) {
          if ((x0 & 1) == 0) { red2(p0, .25f, .25f); red2(p1, .25f, .25f); }
          else { red1(p0, .25f); red1(p0 + 1, .25f); red1(p1, .25f); red1(p1 + 1, .25f); }
        }
        if (MODE == 2) {
          const int k4 = x0 & 3;
          if (k4 != 3) {
            float* b0 = p0 - k4; float* b1 = p1 - k4;
            float a0 = k4 == 0 ? .25f : 0.f, a1 = (k4 == 0 || k4 == 1) ? .25f : 0.f, a2 = (k4 == 1 || k4 == 2) ? .25f : 0.f, a3 = k4 == 2 ? .25f : 0.f;
            red4(b0, a0, a1, a2, a3); red4(b1, a0, a1, a2, a3);
          } else { red1(p0, .25f); red1(p0 + 1, .25f); red1(p1, .25f); red1(p1 + 1, .25f); }
        }
      }
    }
  }
}

// 2-D mapping: a warp covers 16 x 8 pixels (4 px per thread along x), blocks of 256 threads
// cover 64 x 16.  MODE2D 0: scalar reds, 1: v4 padded, 2: shared-memory privatised window
// (float atomics in smem, coalesced v4 flush), 3: same with a 32 x 32 tile.
template <int MODE2D>
__global__ void k2d(float* out, int H, int W, int J, int frames) {
  constexpr int TW = 64, TH = 16, HALO = 16;
  constexpr int WW = TW + 2 * HALO, WH = TH + 2 * HALO;
  __shared__ float win[(MODE2D >= 2) ? WW * WH : 1];
  const int N = H * W;
  const int tiles_x = W / TW, tiles_y = (H + TH - 1) / TH;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int f = blockIdx.y; f < frames; f += gridDim.y) {
    float* o = out + (size_t)f * N;
    for (int tile = blockIdx.x; tile < tiles_x * tiles_y; tile += gridDim.x) {
      const int ty = tile / tiles_x, tx = tile - ty * tiles_x;
      // warp w: x-block (w & 3) * 16, y-block (w >> 2) * 8 ; lane: x = (lane & 3) * 4, y = lane >> 2
      const int c0 = tx * TW + (warp & 3) * 16 + (lane & 3) * 4;
      const int r = ty * TH + (warp >> 2) * 8 + (lane >> 2);
      if (MODE2D >= 2) { for (int i = threadIdx.x; i < WW * WH; i += blockDim.x) win[i] = 0.f; __syncthreads(); }
      if (r < H) {
        for (int v = 0; v < 4; ++v) {
          unsigned h = hash((unsigned)(f * N + r * W + c0 + v));
          int dx = (int)(h % (2 * J + 1)) - J, dy = (int)((h >> 12) % (2 * J + 1)) - J;
          int x0 = min(max(c0 + v + dx, 0), W - 2), y0 = min(max(r + dy, 0), H - 2);
          float* p0 = o + y0 * W + x0; float* p1 = p0 + W;
          if (MODE2D == 0) { red1(p0, .25f); red1(p0 + 1, .25f); red1(p1, .25f); red1(p1 + 1, .25f); }
          if (MODE2D == 1) {
            const int k4 = x0 & 3;
            if (k4 != 3) {
              float a0 = k4 == 0 ? .25f : 0.f, a1 = (k4 == 0 || k4 == 1) ? .25f : 0.f, a2 = (k4 == 1 || k4 == 2) ? .25f : 0.f, a3 = k4 == 2 ? .25f : 0.f;
              red4(p0 - k4, a0, a1, a2, a3); red4(p1 - k4, a0, a1, a2, a3);
            } else { red1(p0, .25f); red1(p0 + 1, .25f); red1(p1, .25f); red1(p1 + 1, .25f); }
          }
          if (MODE2D >= 2) {
            const int wx = x0 - (tx * TW - HALO), wy = y0 - (ty * TH - HALO);
            if (wx >= 0 && wx < WW - 1 && wy >= 0 && wy < WH - 1) {
              float* q = win + wy * WW + wx;
              atomicAdd(q, .25f); atomicAdd(q + 1, .25f); atomicAdd(q + WW, .25f); atomicAdd(q + WW + 1, .25f);
            } else { red1(p0, .25f); red1(p0 + 1, .25f); red1(p1, .25f); red1(p1 + 1, .25f); }
          }
        }
      }
      if (MODE2D >= 2) {
        __syncthreads();
        for (int i = threadIdx.x; i < WW * WH / 4; i += blockDim.x) {
          const int wy = (i * 4) / WW, wx = (i * 4) - wy * WW;
          const int gy = ty * TH - HALO + wy, gx = tx * TW - HALO + wx;
          if (gy >= 0 && gy < H && gx >= 0 && gx + 3 < W) {
            const float4 v = *reinterpret_cast<const float4*>(win + i * 4);
            if (v.x != 0.f || v.y != 0.f || v.z != 0.f || v.w != 0.f) red4(o + gy * W + gx, v.x, v.y, v.z, v.w);
          }
        }
        __syncthreads();
      }
    }
  }
}

template <int MODE2D> float run2d(float* buf, int H, int W, int J, int frames) {
  dim3 grid(74, frames);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  k2d<MODE2D><<<grid, 256>>>(buf, H, W, J, frames);
  cudaDeviceSynchronize();
  cudaEventRecord(a);
  k2d<MODE2D><<<grid, 256>>>(buf, H, W, J, frames);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b); return ms;
}

template <int MODE> float run(float* buf, int H, int W, int J, int frames) {
  dim3 grid((H * W / 4 + 255) / 256 / 4, frames);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  k<MODE><<<grid, 256>>>(buf, H, W, J, frames);
  cudaDeviceSynchronize();
  cudaEventRecord(a);
  k<MODE><<<grid, 256>>>(buf, H, W, J, frames);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b); return ms;
}

// SM-count sweep: one 1024-thread CTA per SM (dynamic shared memory forces exclusivity), S CTAs.
// Tells whether the RED floor is on the SM side (time ~ 1/S) or in the L2 (time flat until S is small).
template <int MODE> float run_sms(float* buf, int H, int W, int J, int frames, int sms) {
  cudaFuncSetAttribute(k<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  dim3 grid(sms, 1);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  k<MODE><<<grid, 1024, 200 * 1024>>>(buf, H, W, J, frames);
  cudaDeviceSynchronize();
  cudaEventRecord(a);
  k<MODE><<<grid, 1024, 200 * 1024>>>(buf, H, W, J, frames);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b); return ms;
}

int main() {
  const int H = 360, W = 640, frames = 149, J = 12;
  float* buf; cudaMalloc(&buf, (size_t)frames * H * W * 4); cudaMemset(buf, 0, (size_t)frames * H * W * 4);
  const double px = (double)frames * H * W;
  const char* names[] = {"4 scalar reds @ jittered taps", "v2 when aligned", "v4 padded", "aligned scalar red", "aligned v4 red", "plain float4 store", "4 scalar reds @ smooth taps"};
  float ms[7] = {run<0>(buf, H, W, J, frames), run<1>(buf, H, W, J, frames), run<2>(buf, H, W, J, frames), run<3>(buf, H, W, J, frames), run<4>(buf, H, W, J, frames), run<5>(buf, H, W, J, frames), run<6>(buf, H, W, J, frames)};
  for (int i = 0; i < 7; ++i) printf("%-32s %8.3f ms  %7.2f Gpx/s\n", names[i], ms[i], px / ms[i] / 1e6);
  const char* n2[] = {"2D patch: 4 scalar reds", "2D patch: v4 padded", "2D patch: smem window + v4 flush"};
  float m2[3] = {run2d<0>(buf, H, W, J, frames), run2d<1>(buf, H, W, J, frames), run2d<2>(buf, H, W, J, frames)};
  for (int i = 0; i < 3; ++i) printf("%-32s %8.3f ms  %7.2f Gpx/s\n", n2[i], m2[i], px / m2[i] / 1e6);
  const int sweep[] = {132, 99, 66, 50, 33, 16};
  for (int sms : sweep)
    printf("SMs %3d: scalar jittered %8.3f ms   v4 padded %8.3f ms   aligned v4 %8.3f ms\n", sms,
           run_sms<0>(buf, H, W, J, frames, sms), run_sms<2>(buf, H, W, J, frames, sms), run_sms<4>(buf, H, W, J, frames, sms));
  cudaError_t e = cudaDeviceSynchronize();
  printf("status: %s\n", cudaGetErrorString(e));
  return 0;
}
