// Tiled, atomic-free form of the Procrustes passes (phase A and phase D), sm_90a.
//
// Included by fm_kernels.cu (inside its anonymous namespace, after the shared helpers).
//
// Why: the backward of align_surfaces (projection.py:235-242) scatters every later-frame
// pixel's adjoint into four bilinear taps of the earlier frame.  As global REDs that scatter
// sits on the L2 atomic path.  The backward flow -- and with it the whole
// tap pattern -- is LOOP-INVARIANT during an overfit run (flow/__init__.py:23,
// model_wrapper_overfit.py:44-49), so the scatter matrix B^T (4 entries per source pixel) is
// transposed ONCE per set of flows into a static "splat plan": for every earlier-frame cell the
// list of (source pixel, bilinear coefficient) that reach it.  Phase D then GATHERS: no atomics,
// deterministic summation order, every depth-gradient value is produced by exactly one thread
// and written with one plain store.
//
// Plan format (per pair, per 64 x 32 tile of the earlier frame): SELL-32-sigma.  The tile's 2048
// cells are sorted by their number of contributors ("slots"); 32 consecutive slots form a slice
// whose entries are stored column-major, padded to the slice's largest count with zero
// coefficients -- a warp walks a slice with a uniform trip count and perfectly coalesced 128-byte
// loads.  An entry is 32 bits: [31:26] row, [25:19] column of the source pixel inside the tile's
// SOURCE WINDOW (128 x 60 pixels of the later frame, placed around the tile shifted by the mean
// flow), [18:0] the bilinear coefficient as unorm19 (absolute error <= 2^-20).  Sources outside
// the window (flow outliers) go to a per-pair overflow list handled by a small RED kernel.
//
// Tile movement: the per-tile windows (earlier-frame depth for the bilinear gather, later-frame
// depth and correspondence weights for the transposed gather) are staged global -> shared memory
// with TMA (cp.async.bulk.tensor.3d + mbarrier complete_tx), one elected thread issuing, software
// pipelined across the tiles of a persistent CTA: the windows of tile t+1 travel while tile t is
// being processed.  Out-of-image parts of a window are zero-filled by the TMA unit and never
// carry weight.
#pragma once
#include <cuda.h>  // CUtensorMap (types only; the encoder is fetched through cudaGetDriverEntryPoint)

namespace tiled {

constexpr int kTW = 64, kTH = 32, kCells = kTW * kTH;        // tile: 2048 cells
constexpr int kWX = 128, kWY = 60, kWinFloats = kWX * kWY;   // window: 7680 floats
constexpr int kWinBytes = kWinFloats * 4;                    // 30720 B
constexpr int kHaloX = (kWX - kTW) / 2, kHaloY = (kWY - kTH) / 2;  // 32, 14
constexpr int kSlices = kCells / 32;                         // 64
constexpr int kT = 256;                                      // threads per CTA
constexpr int kPerThread = kCells / kT;                      // 8 cells per thread
constexpr unsigned kCoefOne = (1u << 19) - 1u;               // unorm19
constexpr float kCoefScale = 524288.0f / 524287.0f;          // decoded value * this = coefficient
constexpr int kPlanMagic = 0x464d5032;                       // "FMP2"
constexpr int kCanonMax = 24;                                // entries per cell sorted for determinism

// status values of PlanHeader (device): 1 = usable, > 1 = fall back to the RED path
enum PlanStatus : int { PLAN_BUILDING = 0, PLAN_OK = 1, PLAN_COUNT_RANGE = 2, PLAN_CAPACITY = 3, PLAN_OVERFLOW = 4 };

struct PlanHeader {
  int magic, F, H, W, tiles_x, tiles_y, status, ovf_cap;
  unsigned long long total_entries, entry_capacity;
  unsigned ovf_max;  // largest per-pair overflow count
  int pad[3];
};
static_assert(sizeof(PlanHeader) == 64, "PlanHeader layout");

struct TileInfo {
  short swx0, swy0;  // source window origin (later frame) for the transposed gather INTO this tile
  short qwx0, qwy0;  // tap window origin (earlier frame) for the bilinear gather OF this tile's pixels
  unsigned entry_base;
  unsigned slice_off[kSlices + 1];  // entry offset of each slice inside the tile (multiples of 32)
};
static_assert(sizeof(TileInfo) == 272, "TileInfo layout");

struct OvfRec { unsigned cell, src; float coef; };

struct Plan {
  PlanHeader* hdr;
  TileInfo* tiles;            // [P * tiles]
  unsigned short* perm;       // [P * tiles * kCells]  slot -> local cell
  unsigned* entries;          // [entry_capacity]
  unsigned* ovf_count;        // [P]
  OvfRec* ovf;                // [P * ovf_cap]
  float* wscratch;            // [P * N] correspondence weights of the current step (phase A -> phase D)
  unsigned* count;            // [P * N] build: contributors per cell, then fill cursor
  unsigned short* slot_of;    // [P * N] build: cell -> slot
  int4* tile_sum;             // [P * tiles] build: sum of (source - cell) displacements
  unsigned* tile_total;       // [P * tiles] build
  size_t entry_capacity;
  int ovf_cap, tiles_x, tiles_y;
  size_t bytes;
};

inline Plan plan_carve(void* base, int F, int H, int W) {
  Plan p;
  const size_t P = (size_t)(F - 1), N = (size_t)H * W;
  p.tiles_x = (W + kTW - 1) / kTW;
  p.tiles_y = (H + kTH - 1) / kTH;
  const size_t T = P * p.tiles_x * p.tiles_y;
  p.entry_capacity = 6 * P * N;
  const size_t cap4 = N / 4 > 1024 ? N / 4 : 1024;
  p.ovf_cap = (int)(cap4 < (1u << 19) ? cap4 : (1u << 19));
  char* b = (char*)base;
  size_t off = 0;
  auto take = [&](size_t bytes) { char* r = b + off; off = align_up(off + bytes, 256); return r; };
  p.hdr = (PlanHeader*)take(sizeof(PlanHeader));
  p.tiles = (TileInfo*)take(T * sizeof(TileInfo));
  p.perm = (unsigned short*)take(T * kCells * sizeof(unsigned short));
  p.entries = (unsigned*)take(p.entry_capacity * sizeof(unsigned) + 8192);  // + slack for the prefetch overrun
  p.ovf_count = (unsigned*)take(P * sizeof(unsigned));
  p.ovf = (OvfRec*)take(P * p.ovf_cap * sizeof(OvfRec));
  p.wscratch = (float*)take(P * N * sizeof(float));
  p.count = (unsigned*)take(P * N * sizeof(unsigned));
  p.slot_of = (unsigned short*)take(P * N * sizeof(unsigned short));
  p.tile_sum = (int4*)take(T * sizeof(int4));
  p.tile_total = (unsigned*)take(T * sizeof(unsigned));
  p.bytes = off;
  return p;
}

// Slice order inside a tile.  Cells are sorted by contributor count (rank 0 = most), rank / 32 is
// the SORTED slice; warp w of the backward kernel walks the STORED slices 8 w .. 8 w + 7, which are
// the sorted slices w, w + 8, w + 16, ...: every warp gets the same mix of long and short lists
// AND its entries form one contiguous stream (prefetchable with unconditional loads).
__host__ __device__ __forceinline__ int stored_slice(int sorted) { return (sorted & 7) * 8 + (sorted >> 3); }
__host__ __device__ __forceinline__ int sorted_slice(int stored) { return (stored & 7) * 8 + (stored >> 3); }

__device__ __forceinline__ unsigned quant_coef(float w) { return __float2uint_rn(w * (float)kCoefOne); }

// The four taps of source pixel (r, c) of a pair: same arithmetic as the per-step kernels.
struct Corners { int cell[4]; float w[4]; int x0, y0; };
__device__ __forceinline__ Corners corners_of(const float* __restrict__ fl, int j, int r, int c, const GridDims& g) {
  const float2 f = __ldg(reinterpret_cast<const float2*>(fl) + j);
  const Taps t = bilinear_taps(pix_coord(c, g.Wf, g.invW) + f.x, pix_coord(r, g.Hf, g.invH) + f.y, g);
  Corners k;
  k.cell[0] = t.y0 * g.W + t.x0; k.w[0] = t.w00;
  k.cell[1] = t.y0 * g.W + t.x1; k.w[1] = t.w01;
  k.cell[2] = t.y1 * g.W + t.x0; k.w[2] = t.w10;
  k.cell[3] = t.y1 * g.W + t.x1; k.w[3] = t.w11;
  k.x0 = t.x0; k.y0 = t.y0;
  return k;
}

__global__ void k_plan_init(PlanHeader* hdr, int F, int H, int W, int tiles_x, int tiles_y, int ovf_cap,
                            unsigned long long capacity) {
  PlanHeader h;
  h.magic = kPlanMagic; h.F = F; h.H = H; h.W = W; h.tiles_x = tiles_x; h.tiles_y = tiles_y;
  h.status = PLAN_BUILDING; h.ovf_cap = ovf_cap; h.total_entries = 0ull; h.entry_capacity = capacity;
  h.ovf_max = 0u; h.pad[0] = h.pad[1] = h.pad[2] = 0;
  *hdr = h;
}

// ---------------------------------------------------------------- plan build, pass 1: count
__global__ void __launch_bounds__(256)
k_plan_count(const float* __restrict__ bflow, unsigned* __restrict__ count, int4* __restrict__ tile_sum,
             int H, int W, int tiles_x, int tiles) {
  const int pair = blockIdx.y, N = H * W;
  const GridDims g = make_grid(H, W);
  const float* fl = bflow + (size_t)pair * N * 2;
  unsigned* cnt = count + (size_t)pair * N;
  int4* ts = tile_sum + (size_t)pair * tiles;
  for (int j0 = blockIdx.x * blockDim.x; j0 < N; j0 += gridDim.x * blockDim.x) {
    const int j = j0 + threadIdx.x;
    const bool live = j < N;
    int tile = -1, dx = 0, dy = 0;
    if (live) {
      const int r = j / W, c = j - r * W;
      const Corners k = corners_of(fl, j, r, c, g);
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (quant_coef(k.w[q]) != 0u) atomicAdd(cnt + k.cell[q], 1u);
      tile = (k.y0 / kTH) * tiles_x + k.x0 / kTW;
      dx = c - k.x0; dy = r - k.y0;
    }
    // displacement statistics of the target tile: one atomic triple per (warp, tile) group
    const unsigned act = __ballot_sync(0xffffffffu, live);
    if (live) {
      const unsigned grp = __match_any_sync(act, tile);
      const int sx = __reduce_add_sync(grp, dx), sy = __reduce_add_sync(grp, dy);
      if ((int)(threadIdx.x & 31) == __ffs(grp) - 1) {
        atomicAdd(&ts[tile].x, sx); atomicAdd(&ts[tile].y, sy); atomicAdd(&ts[tile].z, __popc(grp));
      }
    }
  }
}

// ---------------------------------------------------------------- plan build, pass 2: sort cells
__device__ __forceinline__ int clamp_origin(int o, int extent, int window) {
  const int hi = extent - window;
  return hi <= 0 ? 0 : (o < 0 ? 0 : (o > hi ? hi : o));
}
// Column origin of a window: TMA wants the first byte of a box 16-byte aligned in global memory
// (measured: UTMALDG raises "illegal instruction" otherwise), i.e. a multiple of 4 floats.
__device__ __forceinline__ int clamp_origin_x(int o, int extent, int window) {
  return clamp_origin(o, extent, window) & ~3;
}

__global__ void __launch_bounds__(kT)
k_plan_sort(const float* __restrict__ bflow, const unsigned* __restrict__ count,
            const int4* __restrict__ tile_sum, TileInfo* __restrict__ tiles_out,
            unsigned short* __restrict__ perm, unsigned short* __restrict__ slot_of,
            unsigned* __restrict__ tile_total, PlanHeader* __restrict__ hdr, int H, int W, int tiles_x,
            int tiles) {
  __shared__ unsigned keys[kCells];
  __shared__ int red[2][kT / 32];
  const int tile = blockIdx.x, pair = blockIdx.y, N = H * W;
  const int X0 = (tile % tiles_x) * kTW, Y0 = (tile / tiles_x) * kTH;
  const unsigned* cnt = count + (size_t)pair * N;
  for (int i = threadIdx.x; i < kCells; i += kT) {
    const int gx = X0 + (i & (kTW - 1)), gy = Y0 + (i >> 6);
    unsigned c = (gx < W && gy < H) ? cnt[gy * W + gx] : 0u;
    if (c >= (1u << 20)) { atomicMax(&hdr->status, (int)PLAN_COUNT_RANGE); c = (1u << 20) - 1u; }
    keys[i] = (c << 11) | (unsigned)(kCells - 1 - i);
  }
  __syncthreads();
  // bitonic sort, descending (keys are distinct: ties broken by cell index -> deterministic)
  for (int k = 2; k <= kCells; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < kCells; i += kT) {
        const int p = i ^ j;
        if (p > i) {
          const unsigned a = keys[i], b = keys[p];
          const bool first_larger = (i & k) == 0;
          if (first_larger ? (a < b) : (a > b)) { keys[i] = b; keys[p] = a; }
        }
      }
      __syncthreads();
    }
  const size_t tix = (size_t)pair * tiles + tile;
  for (int rk = threadIdx.x; rk < kCells; rk += kT) {
    const int local = kCells - 1 - (int)(keys[rk] & (kCells - 1));
    const int s = stored_slice(rk >> 5) * 32 + (rk & 31);
    perm[tix * kCells + s] = (unsigned short)local;
    const int gx = X0 + (local & (kTW - 1)), gy = Y0 + (local >> 6);
    if (gx < W && gy < H) slot_of[(size_t)pair * N + gy * W + gx] = (unsigned short)s;
  }
  // tap-window statistics of this tile's own pixels (as later-frame pixels of the pair)
  int sx = 0, sy = 0;
  {
    const GridDims g = make_grid(H, W);
    const float* fl = bflow + (size_t)pair * N * 2;
    for (int i = threadIdx.x; i < kCells; i += kT) {
      const int c = X0 + (i & (kTW - 1)), r = Y0 + (i >> 6);
      if (c < W && r < H) {
        const Corners k = corners_of(fl, r * W + c, r, c, g);
        sx += k.x0 - c; sy += k.y0 - r;
      }
    }
    sx = __reduce_add_sync(0xffffffffu, sx); sy = __reduce_add_sync(0xffffffffu, sy);
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = sx; red[1][threadIdx.x >> 5] = sy; }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    TileInfo ti;
    unsigned off = 0;
    for (int s = 0; s < kSlices; ++s) { ti.slice_off[s] = off; off += 32u * (keys[32 * sorted_slice(s)] >> 11); }
    ti.slice_off[kSlices] = off;
    ti.entry_base = 0;
    tile_total[tix] = off;
    const int4 ts = tile_sum[tix];
    const int n = ts.z > 0 ? ts.z : 1;
    const int mdx = (int)rintf((float)ts.x / (float)n), mdy = (int)rintf((float)ts.y / (float)n);
    ti.swx0 = (short)clamp_origin_x(X0 + mdx - kHaloX, W, kWX);
    ti.swy0 = (short)clamp_origin(Y0 + mdy - kHaloY, H, kWY);
    int qx = 0, qy = 0;
    for (int w = 0; w < kT / 32; ++w) { qx += red[0][w]; qy += red[1][w]; }
    const int cw = (W - X0 < kTW ? W - X0 : kTW), ch = (H - Y0 < kTH ? H - Y0 : kTH);
    const int live = cw * ch > 0 ? cw * ch : 1;
    ti.qwx0 = (short)clamp_origin_x(X0 + (int)rintf((float)qx / (float)live) - kHaloX, W, kWX);
    ti.qwy0 = (short)clamp_origin(Y0 + (int)rintf((float)qy / (float)live) - kHaloY, H, kWY);
    tiles_out[tix] = ti;
  }
}

// ---------------------------------------------------------------- plan build, pass 3: entry bases
__global__ void __launch_bounds__(1024)
k_plan_scan(const unsigned* __restrict__ tile_total, TileInfo* __restrict__ tiles, PlanHeader* __restrict__ hdr,
            int n, unsigned long long capacity) {
  __shared__ unsigned long long warp_tot[32];
  __shared__ unsigned long long carry_s;
  if (threadIdx.x == 0) carry_s = 0ull;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    const unsigned long long v = i < n ? (unsigned long long)tile_total[i] : 0ull;
    unsigned long long incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    unsigned long long before = carry_s;
    for (int w = 0; w < warp; ++w) before += warp_tot[w];
    const unsigned long long excl = before + incl - v;
    if (i < n) tiles[i].entry_base = (unsigned)(excl < 0xffffffffull ? excl : 0xffffffffull);
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = before + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    hdr->total_entries = carry_s;
    if (carry_s > capacity || carry_s >= 0xffffffffull) atomicMax(&hdr->status, (int)PLAN_CAPACITY);
  }
}

// ---------------------------------------------------------------- plan build, pass 4: fill
__global__ void __launch_bounds__(256)
k_plan_fill(const float* __restrict__ bflow, const TileInfo* __restrict__ tiles,
            const unsigned short* __restrict__ slot_of, unsigned* __restrict__ cursor,
            unsigned* __restrict__ entries, unsigned* __restrict__ ovf_count, OvfRec* __restrict__ ovf,
            PlanHeader* __restrict__ hdr, int H, int W, int tiles_x, int ntiles, unsigned long long capacity,
            int ovf_cap) {
  const int pair = blockIdx.y, N = H * W;
  const GridDims g = make_grid(H, W);
  const float* fl = bflow + (size_t)pair * N * 2;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < N; j += gridDim.x * blockDim.x) {
    const int r = j / W, c = j - r * W;
    const Corners k = corners_of(fl, j, r, c, g);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const unsigned qc = quant_coef(k.w[q]);
      if (qc == 0u) continue;
      const int cell = k.cell[q];
      const int cy = cell / W, cx = cell - cy * W;
      const size_t tix = (size_t)pair * ntiles + (cy / kTH) * tiles_x + cx / kTW;
      const unsigned slot = slot_of[(size_t)pair * N + cell];
      const unsigned kth = atomicAdd(cursor + (size_t)pair * N + cell, 1u);
      const TileInfo* ti = tiles + tix;
      const unsigned long long pos = (unsigned long long)ti->entry_base + ti->slice_off[slot >> 5] + kth * 32u + (slot & 31u);
      const int xs = c - (int)ti->swx0, ys = r - (int)ti->swy0;
      unsigned e = 0u;
      if ((unsigned)xs < (unsigned)kWX && (unsigned)ys < (unsigned)kWY) {
        e = ((unsigned)(ys * kWX + xs) << 19) | qc;
      } else {  // flow outlier: the source lies outside the tile's window -> overflow list
        const unsigned idx = atomicAdd(ovf_count + pair, 1u);
        if (idx < (unsigned)ovf_cap) {
          OvfRec rec; rec.cell = (unsigned)cell; rec.src = (unsigned)j; rec.coef = k.w[q];
          ovf[(size_t)pair * ovf_cap + idx] = rec;
        } else {
          atomicMax(&hdr->status, (int)PLAN_OVERFLOW);
        }
      }
      if (pos < capacity) entries[pos] = e;
    }
  }
}

// ---------------------------------------------------------------- plan build, pass 5: canonical order + padding
// One thread per slot: zero the padding behind the cell's entries and sort the entries (the fill
// order depends on the atomic cursor; sorted lists make the plan -- and with it every gradient
// bit -- reproducible from run to run).
__global__ void __launch_bounds__(256)
k_plan_canon(const TileInfo* __restrict__ tiles, const unsigned short* __restrict__ perm,
             const unsigned* __restrict__ cursor, unsigned* __restrict__ entries, unsigned* __restrict__ ovf_count,
             PlanHeader* __restrict__ hdr, int H, int W, int tiles_x, int ntiles, int P,
             unsigned long long capacity) {
  const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t tix = gid / kCells;
  if (gid == 0) {
    unsigned m = 0;
    for (int p = 0; p < P; ++p) m = ovf_count[p] > m ? ovf_count[p] : m;
    hdr->ovf_max = m;
    atomicCAS(&hdr->status, (int)PLAN_BUILDING, (int)PLAN_OK);
  }
  if (tix >= (size_t)P * ntiles) return;
  const int slot = (int)(gid - tix * kCells);
  const int pair = (int)(tix / ntiles), tile = (int)(tix - (size_t)pair * ntiles);
  const TileInfo* ti = tiles + tix;
  const unsigned off = ti->slice_off[slot >> 5], width = (ti->slice_off[(slot >> 5) + 1] - off) >> 5;
  if (width == 0u) return;
  const int local = perm[gid];
  const int gx = (tile % tiles_x) * kTW + (local & (kTW - 1)), gy = (tile / tiles_x) * kTH + (local >> 6);
  unsigned cnt = 0u;
  if (gx < W && gy < H) cnt = cursor[(size_t)pair * (H * W) + gy * W + gx];
  const unsigned long long base = (unsigned long long)ti->entry_base + off + (slot & 31);
  if (base + (unsigned long long)(width - 1) * 32u >= capacity) return;
  unsigned* e = entries + base;
  for (unsigned k = cnt; k < width; ++k) e[k * 32u] = 0u;
  if (cnt >= 2u && cnt <= (unsigned)kCanonMax) {
    unsigned v[kCanonMax];
#pragma unroll 1
    for (unsigned k = 0; k < cnt; ++k) v[k] = e[k * 32u];
#pragma unroll 1
    for (unsigned a = 1; a < cnt; ++a) {
      const unsigned x = v[a];
      int b = (int)a - 1;
      while (b >= 0 && v[b] > x) { v[b + 1] = v[b]; --b; }
      v[b + 1] = x;
    }
#pragma unroll 1
    for (unsigned k = 0; k < cnt; ++k) e[k * 32u] = v[k];
  }
}

// (a & b) | c in one LOP3 (immLut 0xEA); b is expected in a register, c an immediate.
__device__ __forceinline__ unsigned lop3_and_or(unsigned a, unsigned b, unsigned c) {
  unsigned d;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}

// Software prefetch into L2: the streaming operands / entry rows of the NEXT tile are requested a
// whole tile ahead, so that the demand loads find them on chip.
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// ---------------------------------------------------------------- TMA / mbarrier primitives
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy accesses to shared memory (the previous tile's reads) ordered before the async
// proxy's (TMA) writes into the same buffer
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  const unsigned addr = smem_u32(bar);
  unsigned done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(addr), "r"(parity) : "memory");
  } while (!done);
}
// One (kWX x kWY x 1) box of a (W, H, frames) float tensor -> shared memory; completes on `bar`.
__device__ __forceinline__ void tma_load_window(float* dst, const CUtensorMap* map, unsigned long long* bar,
                                                int x, int y, int z) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z) : "memory");
}

}  // namespace tiled

// =================================================================================================
// Per-step kernels
// =================================================================================================
namespace tiled {

// Dynamic shared memory of the tiled kernels: declared 1024-byte aligned so that every buffer sits
// at a compile-time offset of ONE shared-space symbol (pointers rebuilt from integers are generic:
// every window access then costs a 64-bit address computation and a generic LD instead of an LDS).
extern __shared__ __align__(1024) unsigned char tiled_smem[];

// Four taps of the earlier frame: from the staged window when the 2 x 2 patch lies inside it
// (always, up to flow outliers), else from global memory with the clamped indices.
__device__ __forceinline__ void gather_taps(const Taps& t, const float* __restrict__ win, int wx0, int wy0,
                                            const float* __restrict__ da, int W, float& d00, float& d01,
                                            float& d10, float& d11) {
  const int ux = t.x0 - wx0, uy = t.y0 - wy0;
  if ((unsigned)ux < (unsigned)(kWX - 1) && (unsigned)uy < (unsigned)(kWY - 1)) {
    const float* p = win + uy * kWX + ux;  // a clamped second tap has weight 0; the window is fully defined
    d00 = p[0]; d01 = p[1]; d10 = p[kWX]; d11 = p[kWX + 1];
  } else {
    const int r0 = t.y0 * W, r1 = t.y1 * W;
    d00 = __ldg(da + r0 + t.x0); d01 = __ldg(da + r0 + t.x1);
    d10 = __ldg(da + r1 + t.x0); d11 = __ldg(da + r1 + t.x1);
  }
}

// q' (shifted by z0) of one later-frame pixel from its four taps.
__device__ __forceinline__ void q_from_taps(const Taps& t, const GridDims& grid, const Cam& ka, float d00, float d01,
                                            float d10, float d11, float z0, float* q) {
  const float a00 = t.w00 * d00, a01 = t.w01 * d01, a10 = t.w10 * d10, a11 = t.w11 * d11;
  float rx0, ry0, rx1, ry1;
  tap_rays(t, grid, ka, rx0, ry0, rx1, ry1);
  q[0] = (a00 + a10) * rx0 + (a01 + a11) * rx1;
  q[1] = (a00 + a01) * ry0 + (a10 + a11) * ry1;
  q[2] = ((a00 + a01) + (a10 + a11)) - z0;
}

// ---------------------------------------------------------------- phase A, tiled
struct MomArgs {
  const float* depth; const float* k4; const float* bflow; const float* weights;
  float* wscratch; double* moments; const TileInfo* tinfo;
  float wsens;
  int F, H, W, tiles_x, tiles, n_items;
};
constexpr int kMomSmem = 2 * kWinBytes + 16 + 16 + kNumMoments * (kT / 32) * 8;

template <bool HAS_W>
__global__ void __launch_bounds__(kT, 3)
k_moments_tiled(const __grid_constant__ CUtensorMap tm_depth, const MomArgs a) {
  float* win = reinterpret_cast<float*>(tiled_smem);                    // two windows
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(win + 2 * kWinFloats);
  int* s_org = reinterpret_cast<int*>(bars + 2);                         // [2][2]
  double* red = reinterpret_cast<double*>(s_org + 4);
  const int per = (a.n_items + (int)gridDim.x - 1) / (int)gridDim.x;
  const int i0 = (int)blockIdx.x * per, i1 = (i0 + per < a.n_items) ? i0 + per : a.n_items;
  if (i0 >= i1) return;
  const int tid = threadIdx.x, N = a.H * a.W;
  if (tid == 0) {
    mbar_init(&bars[0], 1); mbar_init(&bars[1], 1);
    fence_mbar_init();
    const TileInfo* ti = a.tinfo + i0;
    const int ox = ti->qwx0, oy = ti->qwy0;
    s_org[0] = ox; s_org[1] = oy;
    mbar_expect_tx(&bars[0], kWinBytes);
    tma_load_window(win, &tm_depth, &bars[0], ox, oy, i0 / a.tiles);
  }
  __syncthreads();
  const GridDims grid = make_grid(a.H, a.W);
  float acc[kNumMoments];
#pragma unroll
  for (int k = 0; k < kNumMoments; ++k) acc[k] = 0.f;
  int cur_pair = i0 / a.tiles;
  PairGeom g;
  g.grid = grid;
  int geom_pair = -1;
  unsigned ph0 = 0u, ph1 = 0u;
  int b = 0;
#pragma unroll 1
  for (int i = i0; i < i1; ++i, b ^= 1) {
    if (tid == 0 && i + 1 < i1) {  // next tile's window travels while this one is processed
      const TileInfo* ti = a.tinfo + i + 1;
      const int ox = ti->qwx0, oy = ti->qwy0;
      s_org[(b ^ 1) * 2] = ox; s_org[(b ^ 1) * 2 + 1] = oy;
      fence_proxy_async();
      mbar_expect_tx(&bars[b ^ 1], kWinBytes);
      tma_load_window(win + (b ^ 1) * kWinFloats, &tm_depth, &bars[b ^ 1], ox, oy, (i + 1) / a.tiles);
    }
    if (i + 1 < i1) {  // the next tile's streaming operands: this thread's own future addresses
      const int pn = (i + 1) / a.tiles, tn = (i + 1) - pn * a.tiles;
      const int xn = (tn % a.tiles_x) * kTW + (tid & 15) * 4, yn = (tn / a.tiles_x) * kTH + (tid >> 4);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int gy = yn + 16 * h;
        if (gy < a.H && xn < a.W) {
          const size_t base = (size_t)gy * a.W + xn;
          prefetch_l2(a.depth + (size_t)(pn + 1) * N + base);
          prefetch_l2(a.bflow + ((size_t)pn * N + base) * 2);
          if (HAS_W) prefetch_l2(a.weights + (size_t)pn * N + base);
        }
      }
    }
    const int pair = i / a.tiles, tile = i - pair * a.tiles;
    if (pair != cur_pair) {
      block_accumulate<kNumMoments>(acc, a.moments + (size_t)cur_pair * kNumMoments, red);
#pragma unroll
      for (int k = 0; k < kNumMoments; ++k) acc[k] = 0.f;
      cur_pair = pair;
    }
    if (pair != geom_pair) {
      g.ka = make_cam(load_k4(a.k4, pair));
      g.kb = make_cam(load_k4(a.k4, pair + 1));
      g.z0 = __ldg(a.depth + (size_t)(pair + 1) * N + (size_t)(a.H / 2) * a.W + a.W / 2);
      geom_pair = pair;
    }
    const float* da = a.depth + (size_t)pair * N;
    const float* db = da + N;
    const float* fl = a.bflow + (size_t)pair * N * 2;
    const float* wt = HAS_W ? a.weights + (size_t)pair * N : nullptr;
    float* ws = HAS_W ? a.wscratch + (size_t)pair * N : nullptr;
    const int X0 = (tile % a.tiles_x) * kTW, Y0 = (tile / a.tiles_x) * kTH;
    // operands of this thread's 8 pixels (two rows of 4) are fetched before waiting for the window
    float dv[2][4], wv[2][4], fv[2][8];
    bool live[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int gy = Y0 + (tid >> 4) + 16 * h, gx0 = X0 + (tid & 15) * 4;
      live[h] = gy < a.H && gx0 < a.W;
      if (live[h]) {
        const int base = gy * a.W + gx0;
        load_vec<4>(db + base, dv[h]);
        load_vec2<4>(fl + 2 * base, fv[h]);
        if (HAS_W) {
          load_vec<4>(wt + base, wv[h]);
#pragma unroll
          for (int v = 0; v < 4; ++v) wv[h][v] = weight_of(wv[h][v], a.wsens);
          *reinterpret_cast<float4*>(ws + base) = make_float4(wv[h][0], wv[h][1], wv[h][2], wv[h][3]);
        } else {
#pragma unroll
          for (int v = 0; v < 4; ++v) wv[h][v] = 1.f;
        }
      }
    }
    if (b == 0) { mbar_wait(&bars[0], ph0); ph0 ^= 1u; } else { mbar_wait(&bars[1], ph1); ph1 ^= 1u; }
    const float* w_ = win + b * kWinFloats;
    const int wx0 = s_org[b * 2], wy0 = s_org[b * 2 + 1];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!live[h]) continue;
      const int gy = Y0 + (tid >> 4) + 16 * h, gx0 = X0 + (tid & 15) * 4;
      const float y = pix_coord(gy, grid.Hf, grid.invH);
      float ry_b;
      {
        float rxd;
        ray_of(0.f, y, g.kb, rxd, ry_b);
      }
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        const float x = pix_coord(gx0 + v, grid.Wf, grid.invW);
        const Taps t = bilinear_taps(x + fv[h][2 * v], y + fv[h][2 * v + 1], grid);
        float d00, d01, d10, d11;
        gather_taps(t, w_, wx0, wy0, da, a.W, d00, d01, d10, d11);
        float p[3], q[3];
        q_from_taps(t, grid, g.ka, d00, d01, d10, d11, g.z0, q);
        const float d = dv[h][v];
        p[0] = d * ((x - g.kb.cx) * g.kb.ifx);
        p[1] = d * ry_b;
        p[2] = d - g.z0;
        moments_add(acc, wv[h][v], p, q);
      }
    }
    __syncthreads();  // every read of this window is done before it is refilled (two tiles ahead)
  }
  block_accumulate<kNumMoments>(acc, a.moments + (size_t)cur_pair * kNumMoments, red);
}

// ---------------------------------------------------------------- phase D, tiled (gather form)
struct ItemInfo {
  TileInfo ti;   // target side: pair k (this frame is the earlier one)
  int qwx0, qwy0;  // source side: pair k-1 (this frame is the later one)
  float tgt[12];   // pair k:   cbar[9], kk[3] = qb - cbar (pbar + shift)
  float src[22];   // pair k-1: cbar[9], pb[3], qb[3], qbar[3], pofs[3] = pbar + shift, z0
  Cam cam[3];      // cameras of frames k, k+1, k-1 (the reciprocals are formed once per item, not per thread)
};
static_assert(sizeof(ItemInfo) % 8 == 0, "ItemInfo alignment");

struct BwdArgs {
  const float* depth; const float* k4; const float* bflow;
  float* weights;            // logits / weights of all pairs (updated in place when adam.on), or NULL
  const PairAdjoint* adj; const TileInfo* tinfo; const unsigned short* perm; const unsigned* entries;
  float* g_depth;            // in: direct flow-loss gradient; out: total gradient
  float* g_weights;          // out (or NULL)
  AdamFuse adam;
  float wsens;
  int F, H, W, tiles_x, tiles, n_items;
};
constexpr int kBwdSmem = 3 * kWinBytes + kCells * 4 + 16 + 2 * (int)sizeof(ItemInfo);

__device__ __forceinline__ void stage_item(ItemInfo* dst, const BwdArgs& a, int item, int tid, int N) {
  // threads 128..195: TileInfo of the target side; 200 / 201: per-pair constants
  const int k = item / a.tiles, tile = item - k * a.tiles;
  const bool has_tgt = k <= a.F - 2, has_src = k >= 1;
  if (tid >= 128 && tid < 128 + (int)(sizeof(TileInfo) / 4)) {
    if (has_tgt)
      reinterpret_cast<unsigned*>(&dst->ti)[tid - 128] =
          __ldg(reinterpret_cast<const unsigned*>(a.tinfo + (size_t)k * a.tiles + tile) + (tid - 128));
  } else if (tid == 200) {
    if (has_tgt) {
      const PairAdjoint* ad = a.adj + k;
      float pofs[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) pofs[c] = ad->pbar[c] + ad->shift[c];
#pragma unroll
      for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) dst->tgt[r * 3 + c] = ad->cbar[r * 3 + c];
        dst->tgt[9 + r] = ad->qb[r] - (ad->cbar[r * 3] * pofs[0] + ad->cbar[r * 3 + 1] * pofs[1] + ad->cbar[r * 3 + 2] * pofs[2]);
      }
    }
  } else if (tid == 201) {
    if (has_src) {
      const PairAdjoint* ad = a.adj + (k - 1);
      const TileInfo* ti = a.tinfo + (size_t)(k - 1) * a.tiles + tile;
      dst->qwx0 = ti->qwx0; dst->qwy0 = ti->qwy0;
#pragma unroll
      for (int c = 0; c < 9; ++c) dst->src[c] = ad->cbar[c];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        dst->src[9 + c] = ad->pb[c];
        dst->src[12 + c] = ad->qb[c];
        dst->src[15 + c] = ad->qbar[c];
        dst->src[18 + c] = ad->pbar[c] + ad->shift[c];
      }
      dst->src[21] = ad->shift[2];
    }
  } else if (tid == 202) {
    dst->cam[0] = make_cam(load_k4(a.k4, k));
    dst->cam[1] = make_cam(load_k4(a.k4, has_tgt ? k + 1 : k));
    dst->cam[2] = make_cam(load_k4(a.k4, has_src ? k - 1 : k));
  }
}

template <bool HAS_W>
__global__ void __launch_bounds__(kT, 2)
k_backward_tiled(const __grid_constant__ CUtensorMap tm_depth, const __grid_constant__ CUtensorMap tm_w,
                 const BwdArgs a) {
  float* winQ = reinterpret_cast<float*>(tiled_smem);
  float* winW = winQ + kWinFloats;
  float* winD = winW + kWinFloats;
  float* accs = winD + kWinFloats;                                       // [kCells]
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(accs + kCells);  // [0] W+D, [1] Q
  ItemInfo* info = reinterpret_cast<ItemInfo*>(bars + 2);                // [2]
  const int per = (a.n_items + (int)gridDim.x - 1) / (int)gridDim.x;
  const int i0 = (int)blockIdx.x * per, i1 = (i0 + per < a.n_items) ? i0 + per : a.n_items;
  if (i0 >= i1) return;
  const int tid = threadIdx.x, lane = tid & 31, N = a.H * a.W;
  const GridDims grid = make_grid(a.H, a.W);
  if (tid == 0) {
    mbar_init(&bars[0], 1); mbar_init(&bars[1], 1);
    fence_mbar_init();
  }
  stage_item(&info[0], a, i0, tid, N);
  __syncthreads();
  if (tid == 0) {
    const int k = i0 / a.tiles;
    if (k <= a.F - 2) {
      mbar_expect_tx(&bars[0], (HAS_W ? 2 : 1) * kWinBytes);
      if (HAS_W) tma_load_window(winW, &tm_w, &bars[0], info[0].ti.swx0, info[0].ti.swy0, k);
      tma_load_window(winD, &tm_depth, &bars[0], info[0].ti.swx0, info[0].ti.swy0, k + 1);
    }
    if (k >= 1) {
      mbar_expect_tx(&bars[1], kWinBytes);
      tma_load_window(winQ, &tm_depth, &bars[1], info[0].qwx0, info[0].qwy0, k - 1);
    }
  }
  unsigned phWD = 0u, phQ = 0u;
  int ib = 0;
  // Adam's step-dependent scalars: by value, or from the device step clock (CUDA-graph replays)
  const float adam_step_size = (a.adam.on && a.adam.consts) ? __ldg(a.adam.consts) : a.adam.step_size;
  const float adam_bc2_sqrt = (a.adam.on && a.adam.consts) ? __ldg(a.adam.consts + 1) : a.adam.bc2_sqrt;
#pragma unroll 1
  for (int i = i0; i < i1; ++i, ib ^= 1) {
    const ItemInfo& me = info[ib];
    const int k = i / a.tiles, tile = i - k * a.tiles;
    const bool has_tgt = k <= a.F - 2, has_src = k >= 1;
    const int X0 = (tile % a.tiles_x) * kTW, Y0 = (tile / a.tiles_x) * kTH;
    const bool more = i + 1 < i1;
    if (more) stage_item(&info[ib ^ 1], a, i + 1, tid, N);
    const Cam kk_ = me.cam[0];

    // ---- target side: this tile's cells as the EARLIER frame of pair k (transposed bilinear gather)
    if (has_tgt) {
      const Cam kn = me.cam[1];
      const float axc = grid.invW * kk_.ifx, bxc = (0.5f * grid.invW - kk_.cx) * kk_.ifx;
      const float ayc = grid.invH * kk_.ify, byc = (0.5f * grid.invH - kk_.cy) * kk_.ify;
      const float axn = grid.invW * kn.ifx, ayn = grid.invH * kn.ify;
      const float bxn = fm_fma(axn, (float)me.ti.swx0, (0.5f * grid.invW - kn.cx) * kn.ifx);
      const float byn = fm_fma(ayn, (float)me.ti.swy0, (0.5f * grid.invH - kn.cy) * kn.ify);
      const float axn256 = axn * 256.0f, ayn128 = ayn * 128.0f;
      float cc[12];
#pragma unroll
      for (int q = 0; q < 12; ++q) cc[q] = me.tgt[q];
      const unsigned* ebase = a.entries + me.ti.entry_base + lane;
      const unsigned short* pm = a.perm + ((size_t)k * a.tiles + tile) * kCells + tid;
      // Entry lists are read through registers.  A warp's eight slices are one contiguous stream of
      // 128-byte rows: while slot `it` is processed the first kPF rows of slot it + 1 are already in
      // flight, fetched UNCONDITIONALLY (rows past a short list belong to the following slots and are
      // simply not used; the stream may be overrun by up to 2 kPF rows, the plan leaves slack).
      constexpr int kPF = 8;
      const int sl0 = (tid >> 5) * kPerThread;           // this warp's first stored slice
      const unsigned* p = ebase + me.ti.slice_off[sl0];
      unsigned ec[kPF], en[kPF];
#pragma unroll
      for (int q = 0; q < kPF; ++q) ec[q] = __ldg(p + q * 32);
      int local_c = pm[sl0 * 32 - (tid & ~31)];          // pm already carries + tid: slot = sl0 * 32 + lane
      const unsigned m_cf = opaque_u32(0x7FFFF0u), m_xf = opaque_u32(0x7F0000u), m_yf = opaque_u32(0x7E0000u);
      mbar_wait(&bars[0], phWD);
      phWD ^= 1u;
#pragma unroll 1
      for (int it = 0; it < kPerThread; ++it) {
        const unsigned wc = (me.ti.slice_off[sl0 + it + 1] - me.ti.slice_off[sl0 + it]) >> 5;
        const unsigned* pn = p + wc * 32;
        int local_n = 0;
        if (it + 1 < kPerThread) {
#pragma unroll
          for (int q = 0; q < kPF; ++q) en[q] = __ldg(pn + q * 32);
          local_n = pm[(sl0 + it + 1) * 32 - (tid & ~31)];
        }
        float S1 = 0.f, S2 = 0.f, S3 = 0.f, S4 = 0.f;
        auto add = [&](unsigned e) {
          const unsigned lin = e >> 19;
          const float dj = winD[lin];
          // (x & mask) | exponent as ONE LOP3 each (the mask lives in a register)
          const float cf = __uint_as_float(lop3_and_or(e << 4, m_cf, 0x3F800000u)) - 1.0f;
          const float xf = __uint_as_float(lop3_and_or(e >> 3, m_xf, 0x3F000000u));   // .5 + xs / 256
          const float yf = __uint_as_float(lop3_and_or(e >> 9, m_yf, 0x3F000000u));   // .5 + ys / 128
          const float A = HAS_W ? cf * winW[lin] : cf;
          S1 += A;
          const float t = A * dj;
          S2 += t;
          S3 = fm_fma(t, xf, S3);
          S4 = fm_fma(t, yf, S4);
        };
#pragma unroll
        for (int q = 0; q < kPF; q += 2) {
          if ((unsigned)q < wc) {
            add(ec[q]);
            if ((unsigned)(q + 1) < wc) add(ec[q + 1]);
          }
        }
        for (unsigned q = kPF; q < wc; ++q) add(__ldg(p + q * 32));
        const float gxf = (float)(X0 + (local_c & (kTW - 1))), gyf = (float)(Y0 + (local_c >> 6));
        const float rcx = fm_fma(gxf, axc, bxc), rcy = fm_fma(gyf, ayc, byc);
        // sum_j coef w_j d_j ray_j  (rays of the later frame, from the window coordinates)
        const float T0 = fm_fma(axn256, fm_fma(-0.5f, S2, S3), bxn * S2);
        const float T1 = fm_fma(ayn128, fm_fma(-0.5f, S2, S4), byn * S2);
        const float G0 = fm_fma(cc[0], T0, fm_fma(cc[1], T1, fm_fma(cc[2], S2, cc[9] * S1)));
        const float G1 = fm_fma(cc[3], T0, fm_fma(cc[4], T1, fm_fma(cc[5], S2, cc[10] * S1)));
        const float G2 = fm_fma(cc[6], T0, fm_fma(cc[7], T1, fm_fma(cc[8], S2, cc[11] * S1)));
        accs[local_c] = kCoefScale * fm_fma(rcx, G0, fm_fma(rcy, G1, G2));
#pragma unroll
        for (int q = 0; q < kPF; ++q) ec[q] = en[q];
        p = pn; local_c = local_n;
      }
    } else {
#pragma unroll
      for (int it = 0; it < kPerThread; ++it) accs[it * kT + tid] = 0.f;
    }
    __syncthreads();  // accs complete; winW / winD free; info[ib ^ 1] staged
    if (more) {  // L2 prefetch for the next tile: its entry rows, its slot permutation, its streaming operands
      const ItemInfo& nx = info[ib ^ 1];
      const int kn_ = (i + 1) / a.tiles, tn_ = (i + 1) - kn_ * a.tiles;
      if (kn_ <= a.F - 2) {
        const int sl0 = (tid >> 5) * kPerThread;
        const unsigned r0 = nx.ti.slice_off[sl0] >> 5, r1 = nx.ti.slice_off[sl0 + kPerThread] >> 5;
        const unsigned* eb = a.entries + nx.ti.entry_base;
        for (unsigned r = r0 + lane; r < r1; r += 32) prefetch_l2(eb + (size_t)r * 32);
        prefetch_l2(a.perm + ((size_t)kn_ * a.tiles + tn_) * kCells + tid * 8);
      }
      const int xn = (tn_ % a.tiles_x) * kTW + (tid & 15) * 4, yn = (tn_ / a.tiles_x) * kTH + (tid >> 4);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int gy = yn + 16 * h;
        if (gy < a.H && xn < a.W) {
          const size_t base = (size_t)gy * a.W + xn;
          prefetch_l2(a.g_depth + (size_t)kn_ * N + base);
          if (kn_ >= 1) {
            prefetch_l2(a.depth + (size_t)kn_ * N + base);
            prefetch_l2(a.bflow + ((size_t)(kn_ - 1) * N + base) * 2);
            if (HAS_W) {
              prefetch_l2(a.weights + (size_t)(kn_ - 1) * N + base);
              if (a.adam.on && kn_ - 1 >= a.adam.first_pair) {
                prefetch_l2(a.adam.m + (size_t)(kn_ - 1) * N + base);
                prefetch_l2(a.adam.v + (size_t)(kn_ - 1) * N + base);
              }
            }
          }
        }
      }
    }
    if (tid == 0 && more) {
      const ItemInfo& nx = info[ib ^ 1];
      const int kn_ = (i + 1) / a.tiles;
      if (kn_ <= a.F - 2) {
        fence_proxy_async();
        mbar_expect_tx(&bars[0], (HAS_W ? 2 : 1) * kWinBytes);
        if (HAS_W) tma_load_window(winW, &tm_w, &bars[0], nx.ti.swx0, nx.ti.swy0, kn_);
        tma_load_window(winD, &tm_depth, &bars[0], nx.ti.swx0, nx.ti.swy0, kn_ + 1);
      }
    }

    // ---- source side: this tile's pixels as the LATER frame of pair k-1, + the final gradient
    float* gd = a.g_depth + (size_t)k * N;
    if (has_src) {
      const int ps = k - 1;
      const Cam kp = me.cam[2];
      const float* da = a.depth + (size_t)ps * N;
      const float* db = da + N;
      const float* fl = a.bflow + (size_t)ps * N * 2;
      float* wt = HAS_W ? a.weights + (size_t)ps * N : nullptr;
      float* gw = (HAS_W && a.g_weights) ? a.g_weights + (size_t)ps * N : nullptr;
      const float* c = me.src;
      const float z0 = c[21];
      const bool adam = HAS_W && a.adam.on && ps >= a.adam.first_pair;
      mbar_wait(&bars[1], phQ);
      phQ ^= 1u;
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        const int ly = (tid >> 4) + 16 * h, lx0 = (tid & 15) * 4;
        const int gy = Y0 + ly, gx0 = X0 + lx0;
        if (gy >= a.H || gx0 >= a.W) continue;
        const int base = gy * a.W + gx0;
        float dv[4], fv[8], wraw[4], gdir[4], gout[4], gwv[4], wv[4];
        load_vec<4>(db + base, dv);
        load_vec2<4>(fl + 2 * base, fv);
        {
          const float4 g4 = *reinterpret_cast<const float4*>(gd + base);
          gdir[0] = g4.x; gdir[1] = g4.y; gdir[2] = g4.z; gdir[3] = g4.w;
        }
        if (HAS_W) {
          const float4 w4 = *reinterpret_cast<const float4*>(wt + base);  // coherent: updated in place below
          wraw[0] = w4.x; wraw[1] = w4.y; wraw[2] = w4.z; wraw[3] = w4.w;
        }
        const float4 ac = *reinterpret_cast<const float4*>(accs + ly * kTW + lx0);
        const float acv[4] = {ac.x, ac.y, ac.z, ac.w};
        const float y = pix_coord(gy, grid.Hf, grid.invH);
        const float ry = (y - kk_.cy) * kk_.ify;
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          const float x = pix_coord(gx0 + v, grid.Wf, grid.invW);
          const float rx = (x - kk_.cx) * kk_.ifx;
          const float w = HAS_W ? weight_of(wraw[v], a.wsens) : 1.f;
          wv[v] = w;
          const Taps t = bilinear_taps(x + fv[2 * v], y + fv[2 * v + 1], grid);
          float d00, d01, d10, d11;
          gather_taps(t, winQ, me.qwx0, me.qwy0, da, a.W, d00, d01, d10, d11);
          float q[3];
          q_from_taps(t, grid, kp, d00, d01, d10, d11, z0, q);
          const float dq0 = q[0] - c[15], dq1 = q[1] - c[16], dq2 = q[2] - c[17];
          // u = cbar^T dq + pb ; s = ray . u
          const float u0 = fm_fma(c[0], dq0, fm_fma(c[3], dq1, fm_fma(c[6], dq2, c[9])));
          const float u1 = fm_fma(c[1], dq0, fm_fma(c[4], dq1, fm_fma(c[7], dq2, c[10])));
          const float u2 = fm_fma(c[2], dq0, fm_fma(c[5], dq1, fm_fma(c[8], dq2, c[11])));
          const float s = fm_fma(rx, u0, fm_fma(ry, u1, u2));
          gout[v] = (gdir[v] + acv[v]) + w * s;
          const float pu = fm_fma(c[18], u0, fm_fma(c[19], u1, c[20] * u2));
          const float qd = fm_fma(c[12], dq0, fm_fma(c[13], dq1, c[14] * dq2));
          gwv[v] = fm_fma(dv[v], s, qd - pu);
        }
        *reinterpret_cast<float4*>(gd + base) = make_float4(gout[0], gout[1], gout[2], gout[3]);
        if (HAS_W) {
          if (a.wsens != 0.f) {
#pragma unroll
            for (int v = 0; v < 4; ++v) gwv[v] *= a.wsens * wv[v] * (1.0f - wv[v]);
          }
          if (gw) *reinterpret_cast<float4*>(gw + base) = make_float4(gwv[0], gwv[1], gwv[2], gwv[3]);
          if (adam) {  // torch.optim.Adam on the logits (k_adam's operation order, single-MUFU sqrt / divisions)
            float* am = a.adam.m + (size_t)ps * N + base;
            float* av = a.adam.v + (size_t)ps * N + base;
            float4 mm = *reinterpret_cast<float4*>(am);
            float4 vv = *reinterpret_cast<float4*>(av);
            float* mp = &mm.x; float* vp = &vv.x;
            const float inv_bc2 = fm_rcp(adam_bc2_sqrt);
#pragma unroll
            for (int v = 0; v < 4; ++v) {
              mp[v] = mp[v] + a.adam.omb1 * (gwv[v] - mp[v]);
              vp[v] = vp[v] * a.adam.beta2 + a.adam.omb2 * gwv[v] * gwv[v];
              const float root = vp[v] * fm_rsqrt(fmaxf(vp[v], 1e-37f));
              wraw[v] = wraw[v] - adam_step_size * (mp[v] * fm_rcp(fm_fma(root, inv_bc2, a.adam.eps)));
            }
            *reinterpret_cast<float4*>(am) = mm;
            *reinterpret_cast<float4*>(av) = vv;
            *reinterpret_cast<float4*>(wt + base) = make_float4(wraw[0], wraw[1], wraw[2], wraw[3]);
          }
        }
      }
    } else {  // frame 0: no pair below it
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        const int ly = (tid >> 4) + 16 * h, lx0 = (tid & 15) * 4;
        const int gy = Y0 + ly, gx0 = X0 + lx0;
        if (gy >= a.H || gx0 >= a.W) continue;
        const int base = gy * a.W + gx0;
        float4 g4 = *reinterpret_cast<const float4*>(gd + base);
        const float4 ac = *reinterpret_cast<const float4*>(accs + ly * kTW + lx0);
        g4.x += ac.x; g4.y += ac.y; g4.z += ac.z; g4.w += ac.w;
        *reinterpret_cast<float4*>(gd + base) = g4;
      }
    }
    __syncthreads();  // winQ and accs free
    if (tid == 0 && more) {
      const ItemInfo& nx = info[ib ^ 1];
      const int kn_ = (i + 1) / a.tiles;
      if (kn_ >= 1) {
        fence_proxy_async();
        mbar_expect_tx(&bars[1], kWinBytes);
        tma_load_window(winQ, &tm_depth, &bars[1], nx.qwx0, nx.qwy0, kn_ - 1);
      }
    }
  }
}

// Flow outliers (sources outside their tile's window): the few remaining scatter terms as REDs,
// after k_backward_tiled has stored the gradient.
__global__ void __launch_bounds__(256)
k_backward_overflow(const float* __restrict__ depth, const float* __restrict__ k4,
                    const float* __restrict__ wscratch, const PairAdjoint* __restrict__ adj,
                    const unsigned* __restrict__ ovf_count, const OvfRec* __restrict__ ovf, int ovf_cap,
                    float* __restrict__ g_depth, int H, int W) {
  const int pair = blockIdx.y, N = H * W;
  const unsigned n = ovf_count[pair] < (unsigned)ovf_cap ? ovf_count[pair] : (unsigned)ovf_cap;
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const OvfRec r = ovf[(size_t)pair * ovf_cap + i];
  const PairAdjoint ad = adj[pair];
  const GridDims grid = make_grid(H, W);
  const Cam ka = make_cam(load_k4(k4, pair)), kb = make_cam(load_k4(k4, pair + 1));
  const int sr = (int)r.src / W, sc = (int)r.src - sr * W;
  const int cr = (int)r.cell / W, cc = (int)r.cell - cr * W;
  float rxs, rys, rxc, ryc;
  ray_of(pix_coord(sc, grid.Wf, grid.invW), pix_coord(sr, grid.Hf, grid.invH), kb, rxs, rys);
  ray_of(pix_coord(cc, grid.Wf, grid.invW), pix_coord(cr, grid.Hf, grid.invH), ka, rxc, ryc);
  const float w = wscratch ? wscratch[(size_t)pair * N + r.src] : 1.f;
  const float d = __ldg(depth + (size_t)(pair + 1) * N + r.src);
  const float dp[3] = {d * rxs - ad.pbar[0] - ad.shift[0], d * rys - ad.pbar[1] - ad.shift[1],
                       d - ad.pbar[2] - ad.shift[2]};
  float qb[3];
#pragma unroll
  for (int k = 0; k < 3; ++k)
    qb[k] = w * (ad.cbar[k * 3] * dp[0] + ad.cbar[k * 3 + 1] * dp[1] + ad.cbar[k * 3 + 2] * dp[2] + ad.qb[k]);
  red_add(g_depth + (size_t)pair * N + r.cell, r.coef * (qb[0] * rxc + qb[1] * ryc + qb[2]));
}

}  // namespace tiled
