// TEST INFRASTRUCTURE -- never loaded by flowmap_b200.
//
// Serial host driver for the per-pixel bodies in flowmap_b200/csrc/fm_pixel.cuh and the
// float64 solver in fm_procrustes.cuh.  It exists so that the analytic gradients can be
// checked against the oracle in the build container, which has no GPU; the CUDA kernels
// instantiate the very same inline functions.  Compiled by tests/test_host_emulation.py
// with g++ into tests/host_emulation/_build/ (git-ignored).
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../flowmap_b200/csrc/fm_pixel.cuh"

using namespace fm;

static K4 k4_of(const float* k4, int frame) {
  K4 k; k.fx = k4[frame * 4 + 0]; k.fy = k4[frame * 4 + 1]; k.cx = k4[frame * 4 + 2]; k.cy = k4[frame * 4 + 3];
  return k;
}

// z0: the pair's conditioning shift (pair_shift below in the forward, the saved state's in the backward)
static PairGeom geom(const float* k4, int pair, int F, int H, int W, float z0, int& a) {
  int bi = pair / (F - 1), i = pair - bi * (F - 1);
  a = bi * F + i;
  PairGeom g;
  g.ka = make_cam(k4_of(k4, a)); g.kb = make_cam(k4_of(k4, a + 1)); g.grid = make_grid(H, W);
  g.z0 = z0;
  return g;
}

// k_pair_shift: the weighted mean depth of the later frame db over the shift samples (weights wt or 1)
static float pair_shift(const float* db, const float* wt, int H, int W) {
  double s[3] = {0, 0, 0};
  for (int i = 0; i < kShiftSamples; ++i) {
    const int j = shift_sample(i, H, W);
    const double z = db[j], w = wt ? wt[j] : 1.0;
    s[0] += w * z; s[1] += w; s[2] += z;
  }
  return shift_from_sums(s[0], s[1], s[2]);
}

extern "C" {

size_t emu_state_bytes() { return sizeof(PairState); }

// lean_term (one point) against lean_term2 (two points packed as float32x2, the form k_flow_lean and
// k_track_src evaluate): out[0..1] = 7 values per point from the scalar form, out2 the same from the
// packed form.  dir / off: camera-space direction and offset (P = D * dir + off), k4: intrinsics,
// xy: reference position, fl: flow, mapping / delta: robust map.
void emu_lean_terms(const float* D, const float* dir, const float* off, const float* k4, const float* xy,
                    const float* fl, int mapping, float delta, int H, int W, float* out, float* out2) {
  const RobustCfg rc = make_robust(mapping, delta, H, W);
  K4 kk; kk.fx = k4[0]; kk.fy = k4[1]; kk.cx = k4[2]; kk.cy = k4[3];
  const Cam cam = make_cam(kk);
  for (int i = 0; i < 2; ++i) {
    const LeanTerm t = lean_term(D[i], dir[i * 3 + 0], dir[i * 3 + 1], dir[i * 3 + 2], off[0], off[1], off[2], cam,
                                 xy[i * 2 + 0], xy[i * 2 + 1], fl[i * 2 + 0], fl[i * 2 + 1], 1.0f, rc);
    const float v[7] = {t.loss, t.d0, t.d1, t.d2, t.uvx, t.uvy, t.su};
    for (int k = 0; k < 7; ++k) out[i * 7 + k] = v[k];
  }
  const LeanTerm2 t2 = lean_term2(f2(D[0], D[1]), f2(dir[0], dir[3]), f2(dir[1], dir[4]), f2(dir[2], dir[5]),
                                  f2s(off[0]), f2s(off[1]), f2s(off[2]), cam2(cam, cam), f2(xy[0], xy[2]),
                                  f2(xy[1], xy[3]), f2(fl[0], fl[2]), f2(fl[1], fl[3]), f2s(1.0f), rc);
  const F2 v2[7] = {t2.loss, t2.d0, t2.d1, t2.d2, t2.uvx, t2.uvy, t2.su};
  for (int k = 0; k < 7; ++k) { out2[k] = v2[k].x; out2[7 + k] = v2[k].y; }
}

// item_span (fm_math.cuh): how often every item is covered by the (round, block) spans, and the
// largest / smallest number of items one block receives over all rounds.
void emu_item_cover(long long total, int rounds, int grid, int* cover, long long* per_block_minmax) {
  std::vector<long long> per(grid, 0);
  for (int r = 0; r < rounds; ++r)
    for (int b = 0; b < grid; ++b) {
      const ItemSpan sp = item_span(total, rounds, r, b, grid);
      for (long long i = sp.i0; i < sp.i1; ++i) cover[i] += 1;
      per[b] += sp.i1 - sp.i0;
    }
  per_block_minmax[0] = *std::min_element(per.begin(), per.end());
  per_block_minmax[1] = *std::max_element(per.begin(), per.end());
}

void emu_procrustes_fwd(const float* depth, const float* k4, const float* bflow, const float* weights,
                        const int64_t* indices, int n_idx, float* rt, PairState* state, int B, int F,
                        int H, int W) {
  const int N = H * W, BP = B * (F - 1);
  for (int pair = 0; pair < BP; ++pair) {
    const int bi = pair / (F - 1), a0 = bi * F + pair - bi * (F - 1);
    const float z0 = pair_shift(depth + (size_t)(a0 + 1) * N, weights ? weights + (size_t)pair * N : nullptr, H, W);
    int a;
    PairGeom g = geom(k4, pair, F, H, W, z0, a);
    const float* da = depth + (size_t)a * N; const float* db = da + N;
    double m[kNumMoments] = {0};
    const int cnt = indices ? n_idx : N;
    for (int t = 0; t < cnt; ++t) {
      const int j = indices ? (int)indices[t] : t;
      float acc[kNumMoments] = {0}; float p[3], q[3]; Taps taps;
      point_pq(g, pix_coord(j % W, g.grid.Wf, g.grid.invW), pix_coord(j / W, g.grid.Hf, g.grid.invH), db[j], bflow[((size_t)pair * N + j) * 2], bflow[((size_t)pair * N + j) * 2 + 1],
               [da](int o) { return da[o]; }, p, q, taps);
      moments_add(acc, weights ? weights[(size_t)pair * N + j] : 1.f, p, q);
      for (int k = 0; k < kNumMoments; ++k) m[k] += acc[k];
    }
    double shift[3] = {0, 0, (double)g.z0};
    procrustes_solve(m, shift, rt + (size_t)pair * 12, state[pair]);
  }
}

// flowacc: (B*F, 40) doubles, zero-filled by the caller.
void emu_flow(const float* depth, const float* k4, const float* rt, const float* ff, const float* fb,
              const float* mf, const float* mb, double mask_sum, int mapping, float delta, float weight,
              float* g_depth, double* flowacc, int B, int F, int H, int W) {
  const int N = H * W;
  if (mask_sum == 0.0) mask_sum = 1.0;
  const float g = (float)((double)weight / mask_sum);
  const RobustCfg rc = make_robust(mapping, delta, H, W);
  const GridDims grid = make_grid(H, W);
  for (int frame = 0; frame < B * F; ++frame) {
    int bi = frame / F, i = frame - bi * F;
    FlowFrame f;
    f.hasF = i < F - 1; f.hasB = i > 0;
    f.kk = make_cam(k4_of(k4, frame)); f.kn = make_cam(k4_of(k4, f.hasF ? frame + 1 : frame)); f.kp = make_cam(k4_of(k4, f.hasB ? frame - 1 : frame));
    int pairF = bi * (F - 1) + i, pairB = pairF - 1;
    auto ld = [&](int pair) { Rt t; for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) t.r[r * 3 + c] = rt[(size_t)pair * 12 + r * 4 + c]; t.t[r] = rt[(size_t)pair * 12 + r * 4 + 3]; } return t; };
    if (f.hasF) f.tf = ld(pairF);
    if (f.hasB) f.tb = ld(pairB);
    for (int j = 0; j < N; ++j) {
      float acc[kFlowVals] = {0};
      const size_t jf = (size_t)(f.hasF ? pairF : 0) * N + j, jb = (size_t)(f.hasB ? pairB : 0) * N + j;
      auto fp = f.hasF && f.hasB ? flow_pixel<true, true> : (f.hasF ? flow_pixel<true, false> : flow_pixel<false, true>);
      g_depth[(size_t)frame * N + j] = fp(
          f, pix_coord(j % W, grid.Wf, grid.invW), pix_coord(j / W, grid.Hf, grid.invH), depth[(size_t)frame * N + j], f.hasF ? ff[jf * 2] : 0.f,
          f.hasF ? ff[jf * 2 + 1] : 0.f, f.hasF ? mf[jf] : 0.f, f.hasB ? fb[jb * 2] : 0.f,
          f.hasB ? fb[jb * 2 + 1] : 0.f, f.hasB ? mb[jb] : 0.f, g, rc, acc);
      for (int k = 0; k < kFlowVals; ++k) flowacc[(size_t)frame * 40 + k] += acc[k];
    }
  }
}

// Lean phase C: writes the STANDARD accumulator layout (after lean_to_standard) into flowacc.
void emu_flow_lean(const float* depth, const float* k4, const float* rt, const float* ff, const float* fb,
                   const float* mf, const float* mb, double mask_sum, int mapping, float delta, float weight,
                   int focal_mode, float* g_depth, double* flowacc, int B, int F, int H, int W) {
  const int N = H * W;
  if (mask_sum == 0.0) mask_sum = 1.0;
  const float g = (float)((double)weight / mask_sum);
  const RobustCfg rc = make_robust(mapping, delta, H, W);
  const GridDims grid = make_grid(H, W);
  for (int frame = 0; frame < B * F; ++frame) {
    int bi = frame / F, i = frame - bi * F;
    const bool hasF = i < F - 1, hasB = i > 0;
    FlowFrameLean f;
    f.kk = make_cam(k4_of(k4, frame)); f.kn = make_cam(k4_of(k4, hasF ? frame + 1 : frame)); f.kp = make_cam(k4_of(k4, hasB ? frame - 1 : frame));
    int pairF = bi * (F - 1) + i, pairB = pairF - 1;
    auto ld = [&](int pair) { Rt t; for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) t.r[r * 3 + c] = rt[(size_t)pair * 12 + r * 4 + c]; t.t[r] = rt[(size_t)pair * 12 + r * 4 + 3]; } return t; };
    Rt tf, tb;
    if (hasF) tf = ld(pairF);
    if (hasB) tb = ld(pairB);
    fill_lean(f, hasF ? &tf : nullptr, hasB ? &tb : nullptr);
    double lean[kFlowLeanVals] = {0};
    // even widths: the packed two-pixel code path (what the vector kernel instantiation runs)
    if (W % 2 == 0) {
      for (int j = 0; j < N; j += 2) {
        F2 acc2[kFlowLeanVals];
        for (int k = 0; k < kFlowLeanVals; ++k) acc2[k] = f2s(0.f);
        const size_t jf = (size_t)(hasF ? pairF : 0) * N + j, jb = (size_t)(hasB ? pairB : 0) * N + j;
        const F2 x = f2(pix_coord(j % W, grid.Wf, grid.invW), pix_coord(j % W + 1, grid.Wf, grid.invW));
        const float y = pix_coord(j / W, grid.Hf, grid.invH);
        const F2 D = f2(depth[(size_t)frame * N + j], depth[(size_t)frame * N + j + 1]);
        const F2 z = f2s(0.f);
        F2 o;
#define FM_CALL2(HF, HB) o = focal_mode ? flow_pixel_lean2<HF, HB, true>(f, x, y, D, HF ? f2(ff[jf * 2], ff[jf * 2 + 2]) : z, HF ? f2(ff[jf * 2 + 1], ff[jf * 2 + 3]) : z, HF ? f2(mf[jf], mf[jf + 1]) : z, HB ? f2(fb[jb * 2], fb[jb * 2 + 2]) : z, HB ? f2(fb[jb * 2 + 1], fb[jb * 2 + 3]) : z, HB ? f2(mb[jb], mb[jb + 1]) : z, g, rc, acc2) \
                                   : flow_pixel_lean2<HF, HB, false>(f, x, y, D, HF ? f2(ff[jf * 2], ff[jf * 2 + 2]) : z, HF ? f2(ff[jf * 2 + 1], ff[jf * 2 + 3]) : z, HF ? f2(mf[jf], mf[jf + 1]) : z, HB ? f2(fb[jb * 2], fb[jb * 2 + 2]) : z, HB ? f2(fb[jb * 2 + 1], fb[jb * 2 + 3]) : z, HB ? f2(mb[jb], mb[jb + 1]) : z, g, rc, acc2)
        if (hasF && hasB) { FM_CALL2(true, true); } else if (hasF) { FM_CALL2(true, false); } else { FM_CALL2(false, true); }
#undef FM_CALL2
        g_depth[(size_t)frame * N + j] = o.x;
        g_depth[(size_t)frame * N + j + 1] = o.y;
        for (int k = 0; k < kFlowLeanVals; ++k) lean[k] += (double)acc2[k].x + (double)acc2[k].y;
      }
    } else
    for (int j = 0; j < N; ++j) {
      float acc[kFlowLeanVals] = {0};
      const size_t jf = (size_t)(hasF ? pairF : 0) * N + j, jb = (size_t)(hasB ? pairB : 0) * N + j;
      const float x = pix_coord(j % W, grid.Wf, grid.invW), y = pix_coord(j / W, grid.Hf, grid.invH);
      const float D = depth[(size_t)frame * N + j];
      float out;
#define FM_CALL(HF, HB) out = focal_mode ? flow_pixel_lean<HF, HB, true>(f, x, y, D, HF ? ff[jf * 2] : 0.f, HF ? ff[jf * 2 + 1] : 0.f, HF ? mf[jf] : 0.f, HB ? fb[jb * 2] : 0.f, HB ? fb[jb * 2 + 1] : 0.f, HB ? mb[jb] : 0.f, g, rc, acc) \
                                 : flow_pixel_lean<HF, HB, false>(f, x, y, D, HF ? ff[jf * 2] : 0.f, HF ? ff[jf * 2 + 1] : 0.f, HF ? mf[jf] : 0.f, HB ? fb[jb * 2] : 0.f, HB ? fb[jb * 2 + 1] : 0.f, HB ? mb[jb] : 0.f, g, rc, acc)
      if (hasF && hasB) { FM_CALL(true, true); } else if (hasF) { FM_CALL(true, false); } else { FM_CALL(false, true); }
#undef FM_CALL
      g_depth[(size_t)frame * N + j] = out;
      for (int k = 0; k < kFlowLeanVals; ++k) lean[k] += acc[k];
    }
    const double s = sqrt((double)H * (double)W);
    const double focal = (double)k4[(size_t)frame * 4] * (double)W / s;
    double out_std[kFlowVals];
    lean_to_standard<double>(lean, hasF ? rt + (size_t)pairF * 12 : nullptr, hasB ? rt + (size_t)pairB * 12 : nullptr, focal, (double)W / s, focal_mode != 0, out_std);
    for (int k = 0; k < kFlowVals; ++k) flowacc[(size_t)frame * 40 + k] = out_std[k];
  }
}

// g_rt: (BP, 12) doubles = dL/d[R|t]; g_depth accumulated into; g_weights written/accumulated;
// k4acc: (B*F, 4) doubles accumulated into.
void emu_procrustes_bwd(const float* depth, const float* k4, const float* bflow, const float* weights,
                        const int64_t* indices, int n_idx, const PairState* state, const double* g_rt,
                        float* g_depth, float* g_weights, double* k4acc, int B, int F, int H, int W) {
  const int N = H * W, BP = B * (F - 1);
  for (int pair = 0; pair < BP; ++pair) {
    PairAdjoint ad;
    procrustes_adjoint(state[pair], g_rt + (size_t)pair * 12, ad);
    int a;
    PairGeom g = geom(k4, pair, F, H, W, ad.shift[2], a);
    const float* da = depth + (size_t)a * N; const float* db = da + N;
    float* gda = g_depth + (size_t)a * N; float* gdb = gda + N;
    const int cnt = indices ? n_idx : N;
    for (int t = 0; t < cnt; ++t) {
      const int j = indices ? (int)indices[t] : t;
      float kacc[8] = {0}; float gdj, gwj;
      distribute_point(g, ad, pix_coord(j % W, g.grid.Wf, g.grid.invW), pix_coord(j / W, g.grid.Hf, g.grid.invH), db[j], weights ? weights[(size_t)pair * N + j] : 1.f,
                       bflow[((size_t)pair * N + j) * 2], bflow[((size_t)pair * N + j) * 2 + 1],
                       [da](int o) { return da[o]; }, [gda, W](int y0, int x0, float v0, float v1) { gda[y0 * W + x0] += v0; if (x0 + 1 < W) gda[y0 * W + x0 + 1] += v1; }, gdj, gwj, kacc);
      gdb[j] += gdj;
      if (g_weights) g_weights[(size_t)pair * N + j] += gwj;
      for (int k = 0; k < 8; ++k) k4acc[(size_t)a * 4 + k] += kacc[k];
    }
  }
}

// Phase D2 on every pixel through distribute_point<true> (kgrad 1) or <false> (kgrad 0, the constant-intrinsics
// kernels): per point (pair * N + j) its g_db, its g_w and the two scatter calls in call order (row, x0, v0,
// v1) -> taps[8 per point].  kacc starts at a sentinel for every point; kacc_moved counts the points whose kacc
// changed.
void emu_distribute(const float* depth, const float* k4, const float* bflow, const float* weights,
                    const PairState* state, const double* g_rt, int kgrad, float* g_db, float* g_w, float* taps,
                    long long* kacc_moved, int B, int F, int H, int W) {
  const int N = H * W, BP = B * (F - 1);
  const float sentinel = 0.3125f;
  *kacc_moved = 0;
  for (int pair = 0; pair < BP; ++pair) {
    PairAdjoint ad;
    procrustes_adjoint(state[pair], g_rt + (size_t)pair * 12, ad);
    int a;
    PairGeom g = geom(k4, pair, F, H, W, ad.shift[2], a);
    const float* da = depth + (size_t)a * N; const float* db = da + N;
    for (int j = 0; j < N; ++j) {
      const size_t o = (size_t)pair * N + j;
      float kacc[8];
      for (int k = 0; k < 8; ++k) kacc[k] = sentinel;
      float* tp = taps + o * 8;
      int call = 0;
      auto scatter = [tp, &call](int y0, int x0, float v0, float v1) {
        float* t = tp + 4 * call++;
        t[0] = (float)y0; t[1] = (float)x0; t[2] = v0; t[3] = v1;
      };
      auto load_a = [da](int q) { return da[q]; };
      const float x = pix_coord(j % W, g.grid.Wf, g.grid.invW), y = pix_coord(j / W, g.grid.Hf, g.grid.invH);
      const float w = weights ? weights[o] : 1.f, flx = bflow[o * 2], fly = bflow[o * 2 + 1];
      if (kgrad) distribute_point<true>(g, ad, x, y, db[j], w, flx, fly, load_a, scatter, g_db[o], g_w[o], kacc);
      else distribute_point<false>(g, ad, x, y, db[j], w, flx, fly, load_a, scatter, g_db[o], g_w[o], kacc);
      bool moved = false;
      for (int k = 0; k < 8; ++k) moved |= kacc[k] != sentinel;
      *kacc_moved += moved;
    }
  }
}
}

