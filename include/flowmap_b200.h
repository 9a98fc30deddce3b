/* flowmap_b200 -- C ABI of the B200-native FlowMap optimisation hot path.
 *
 * The reference (dcharatan/flowmap) has no FFI of its own: its boundary is the Python
 * surface of flowmap.model.projection / flowmap.model.procrustes / flowmap.loss, every
 * body being ATen calls.  This header is what those bodies bind to instead.  Each entry
 * point cites the reference code it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless said otherwise; all arrays are contiguous
 *     float32, row-major, in the reference's layouts: depth (B,F,H,W), flows
 *     (B,F-1,H,W,2), masks/weights (B,F-1,H,W).  Intrinsics are passed as k4 (B,F,4) =
 *     (fx, fy, cx, cy) of the normalised matrix of intrinsics/common.py:6-20; relative
 *     poses as rt (B,F-1,3,4) = [R | t] of procrustes.py:45-51 (maps frame i+1 camera
 *     coordinates to frame i camera coordinates).
 *   - every function is asynchronous on `stream` (a cudaStream_t passed as void*), never
 *     allocates or frees device memory, keeps no pointer after returning, is re-entrant
 *     and may be called from any host thread (autograd runs backward on its own thread).
 *   - return value 0 = success; otherwise fm_last_error() (thread-local) describes it.
 *   - `ws` is caller-provided scratch of at least fm_workspace_bytes(...) bytes, 256-byte
 *     aligned; the same ws must be passed to the forward and backward halves of one step.
 */
#ifndef FLOWMAP_B200_H
#define FLOWMAP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FM_MAP_HUBER 0 /* loss/mapping/mapping_huber.py:19-34 */
#define FM_MAP_L1 1    /* loss/mapping/mapping_l1.py:16-20    */
#define FM_MAP_L2 2    /* loss/mapping/mapping_l2.py:16-21    */

#define FM_K_FULL 0
#define FM_K_SHARED_FOCAL 1
#define FM_K_CONST 2

int fm_version(void);
const char* fm_last_error(void);
/* Number of kernels this library has launched in this process (evidence for bench.py's
 * gpu_launches; one count per successful launch). */
unsigned long long fm_launch_count(void);

/* Scratch size for one optimisation step on (B, F, H, W). */
size_t fm_workspace_bytes(int B, int F, int H, int W);
/* Zero the accumulators in ws; call once at the start of every step. */
int fm_workspace_reset(void* ws, int B, int F, int H, int W, void* stream);

/* projection.py:76-90 unproject (+ :93-113 sample_image_grid): depth, k4 -> surfaces
 * (B*F, H, W, 3). */
int fm_unproject(const float* depth, const float* k4, float* surfaces, int BF, int H, int W,
                 void* stream);
/* Adjoint of fm_unproject: g_surfaces -> g_depth (B*F,H,W) and g_k4 (B*F,4). */
int fm_unproject_bwd(const float* depth, const float* k4, const float* g_surfaces, float* g_depth,
                     float* g_k4, void* ws, int B, int F, int H, int W, void* stream);

/* projection.py:116-134 reproject_points + :49-58 project_camera_space: n points per
 * item, one [R|t] (3x4) and one k4 per item -> xy (items, n, 2).  Forward only (used by
 * the visualiser/export callers; the differentiable uses are the fused ops below). */
int fm_reproject(const float* xyz, const float* rt, const float* k4, float* xy,
                 unsigned char* in_front /* optional: z >= 0 after the transform, projection.py:72 */,
                 int items, int n, void* stream);

/* projection.py:76-90 unproject on explicit coordinates: xy (items or 1, n, 2), z (items, n),
 * k4 (items, 4) -> (items, n, 3); xy_shared != 0 means one coordinate set for all items.  The
 * backward returns g_z and g_k4 (coordinates are constants). */
int fm_unproject_points(const float* xy, const float* z, const float* k4, float* out, int items, int n,
                        int xy_shared, void* stream);
int fm_unproject_points_bwd(const float* xy, const float* z, const float* k4, const float* g_out, float* g_z,
                            float* g_k4, void* ws, int items, int n, int xy_shared, void* stream);

/* procrustes.py:7-51 align_rigid on explicit point sets p, q (items, n, 3), weights (items, n)
 * -> rt (items, 3, 4), and its backward (closed-form SVD adjoint).  ws: fm_points_workspace_bytes. */
size_t fm_points_workspace_bytes(int items);
int fm_align_rigid_fwd(const float* p, const float* q, const float* weights, float* rt, void* ws, int items,
                       int n, void* stream);
int fm_align_rigid_bwd(const float* p, const float* q, const float* weights, const float* g_rt, float* g_p,
                       float* g_q, float* g_w, void* ws, int items, int n, void* stream);

/* projection.py:213-249 align_surfaces up to the chain, + procrustes.py:7-51
 * align_rigid: per pair, gather later points / bilinear-sample earlier surface at
 * xy + backward_flow / weights, accumulate weighted moments, 3x3 SVD, det fix.
 * indices: int64 pixel indices (extrinsics_procrustes.py:33-51) or NULL for all pixels.
 * Writes rt (B*(F-1), 3, 4); keeps the solver state in ws for fm_procrustes_bwd. */
int fm_procrustes_fwd(const float* depth, const float* k4, const float* backward_flow,
                      const float* weights, const int64_t* indices, int num_indices, float* rt,
                      void* ws, int B, int F, int H, int W, void* stream);

/* Backward of fm_procrustes_fwd (closed-form SVD adjoint, SURVEY A.7).
 * g_rt: dL/d rt from any consumer, or NULL.  When `include_flow_loss` is non-zero the
 * pose gradient that fm_flow_loss_fwd_bwd left in ws is added, scaled by *flow_scale
 * (device scalar, NULL = 1).  g_depth (B,F,H,W) is ACCUMULATED into (atomics; caller
 * zero-fills or passes the buffer fm_flow_loss_fwd_bwd wrote); g_weights (B,F-1,H,W) is
 * written (all-pixel mode) or accumulated into (index mode; caller zero-fills);
 * g_k4 (B,F,4) is written = procrustes part [+ flow-loss part when included]. */
int fm_procrustes_bwd(const float* depth, const float* k4, const float* backward_flow,
                      const float* weights, const int64_t* indices, int num_indices,
                      const float* g_rt, int include_flow_loss, const float* flow_scale,
                      float* g_depth, float* g_weights, float* g_k4, void* ws, int B, int F, int H,
                      int W, void* stream);

/* loss_flow.py:55-56,67-68 denominators: *out = sum(forward_mask) + sum(backward_mask)
 * (device float64 scalar). */
int fm_mask_sum(const float* forward_mask, const float* backward_mask, double* out, size_t count,
                void* stream);

/* loss_flow.py:31-70 LossFlow + projection.py:143-184 compute_{forward,backward}_flow +
 * mapping/<name>.py, forward and analytic backward in one pass.  Uses the pair-local form of
 * SURVEY A.6 (inv(P_i) P_{i+1} == rt_i).  loss_weight is cfg.weight (loss.py:46).
 * mask_sum: device float64 scalar from fm_mask_sum ("or 1" applied inside).
 * intrinsics_mode: FM_K_FULL = per-frame k4, gradient for every entry; FM_K_SHARED_FOCAL =
 * all frames share one focal length with the principal point fixed (intrinsics_regressed.py,
 * intrinsics_softmin.py): a cheaper kernel, the gradient is returned as the equivalent
 * d/dfx of each frame (g_k4[:, 1:] = 0); FM_K_CONST = constant intrinsics (g_k4 = 0).  In the
 * two cheap modes g_rt is the tangent (rigid) part of the pose gradient.
 * Outputs: loss (device float, = weight * sum / mask_sum); g_depth (B,F,H,W) WRITTEN with
 * the direct (pose-detached) depth gradient; g_rt (B*(F-1),3,4) written; pose and
 * intrinsics partials also stay in ws for fm_procrustes_bwd / fm_flow_k4_grad. */
int fm_flow_loss_fwd_bwd(const float* depth, const float* k4, const float* rt,
                         const float* forward_flow, const float* backward_flow,
                         const float* forward_mask, const float* backward_mask,
                         const double* mask_sum, int mapping, float delta, float loss_weight,
                         int intrinsics_mode, float* loss, float* g_depth, float* g_rt, float* g_k4,
                         void* ws, int B, int F, int H, int W, void* stream);

/* projection.py:187-210 get_extrinsics: rt (B, F-1, 3, 4) -> camera-to-world (B, F, 4, 4),
 * P_0 = I, P_{k+1} = P_k @ T_k, and its adjoint. */
int fm_pose_chain(const float* rt, float* extrinsics, int B, int F, void* stream);
int fm_pose_chain_bwd(const float* rt, const float* extrinsics, const float* g_extrinsics,
                      float* g_rt, int B, int F, void* stream);

/* misc/ate.py:7-25 compute_ate (scipy.spatial.procrustes) on T independent trajectories of F points,
 * gt / pred (T, F, 3), one block per trajectory, float64 inside: both sets centred and scaled to unit
 * Frobenius norm, R = U V^T from the SVD of gt^T pred (reflections allowed), s = sum of the singular
 * values; aligned_pred = s * pred R^T, ate[t] = sqrt(mean((aligned_gt - aligned_pred)^2)).
 * aligned_gt / aligned_pred (T, F, 3) may be NULL.  status[t] = 0, or 1 where scipy raises "Input
 * matrices must contain >1 unique points" (a set is exactly one point after centring in float64);
 * ate[t] is NaN then.  No host synchronisation.  A trajectory's results do not depend on T. */
int fm_trajectory_ate(const float* gt, const float* pred, int T, int F, float* ate, float* aligned_gt,
                      float* aligned_pred, int* status, void* stream);

/* loss_tracking.py:28-61 LossTracking + projection.py:255-298 compute_track_flow, all
 * segments in one launch (batch size 1, as tracking/__init__.py:92-93 asserts).
 * Packing: samples of segment s are stored row-major (frame row, point) starting at
 * segments[s][0]; segments (device int32, num_segments x 4) = (sample_start, rows f_s,
 * points n_s, start_frame); track_xy (total_samples, 2) float; track_vis (total_samples)
 * uint8.  extrinsics: camera-to-world (F, 4, 4).  All (source row, target row) pairs of a
 * segment are evaluated, including source == target; a term is valid when both ends are
 * visible, the source lies in [0,1)^2 and the PREDICTED target lies in [0,1)^2.
 * The count depends on the predicted positions, so fwd makes the single sweep over all
 * (source, target, point) triples, accumulating loss, count AND the unscaled gradient pieces
 * into ws (fm_track_workspace_bytes); bwd only scales them by weight * grad_out / count:
 * it accumulates into g_depth (F,H,W; caller zero-fills or passes the flow-loss gradient)
 * and writes g_extrinsics (F,4,4; tangent part) and g_k4 (F,4).  grad_out: device float
 * scalar dL/dloss or NULL (= 1).  bwd must follow fwd with the same ws and inputs. */
size_t fm_track_workspace_bytes(int F, long long total_samples);
int fm_track_loss_fwd(const float* depth, const float* k4, const float* extrinsics, const int* segments,
                      int num_segments, int max_rows, int max_points, const float* track_xy,
                      const unsigned char* track_vis, long long total_samples, int mapping, float delta,
                      float loss_weight, float* loss, void* ws, int F, int H, int W, void* stream);
int fm_track_loss_bwd(const float* depth, const float* k4, const float* extrinsics, const int* segments,
                      int num_segments, int max_rows, int max_points, const float* track_xy,
                      const unsigned char* track_vis, long long total_samples, int mapping, float delta,
                      float loss_weight, const float* grad_out, float* g_depth, float* g_extrinsics,
                      float* g_k4, void* ws, int F, int H, int W, void* stream);

/* Multi-GPU form (SURVEY 8(e): "shard by source frame"): the reference has no counterpart (its
 * DDP replicas hold the whole problem, overfit.py:99-103).  This rank holds the depth frames
 * starting at global frame `depth_frame0` (depth and g_depth point at that frame) and evaluates
 * only the source frames [src_frame_lo, src_frame_hi); k4 / extrinsics / g_extrinsics / g_k4 and
 * the track arrays are global (F frames).  Between fwd and bwd the caller all-reduces (sum, as
 * float64) the first fm_track_reduce_bytes(F) bytes of `ws` (loss sum, valid count, per-frame
 * pose / intrinsics sums); fm_track_loss_value then gives the global loss, and the backward's
 * g_extrinsics / g_k4 are the global gradients on every rank while g_depth receives this rank's
 * source frames.  loss may be NULL in the sharded forward.
 * shared_intrinsics != 0: the caller guarantees that all frames share one set of intrinsics (one
 * focal length parameter, or constants) and only uses the SUM over frames of g_k4; the per-frame
 * split of g_k4 is then unspecified (the target-frame terms are booked on the source frame, which
 * takes 4 of the 10 values out of the per-row warp reduction).  depth_frame0 = 0, range [0, F) and
 * shared_intrinsics = 0 is exactly fm_track_loss_fwd. */
size_t fm_track_reduce_bytes(int F);
int fm_track_loss_fwd_sharded(const float* depth, const float* k4, const float* extrinsics, const int* segments,
                              int num_segments, int max_rows, int max_points, const float* track_xy,
                              const unsigned char* track_vis, long long total_samples, int mapping, float delta,
                              float loss_weight, float* loss, void* ws, int F, int H, int W, int depth_frame0,
                              int src_frame_lo, int src_frame_hi, int shared_intrinsics, void* stream);
/* fm_track_loss_fwd_sharded for constant intrinsics (ground truth): the sweep accumulates no intrinsics
 * terms (6 values per target-row reduction instead of 10) and leaves in `ws` what the constant-intrinsics
 * backward reads, fm_overfit_step's FM_STEP_BACKWARD with g_k4 == track_g_k4 == NULL.  k4 may differ from
 * frame to frame.  Arguments as in fm_track_loss_fwd_sharded, which shared_intrinsics would not change. */
int fm_track_loss_fwd_const_k(const float* depth, const float* k4, const float* extrinsics, const int* segments,
                              int num_segments, int max_rows, int max_points, const float* track_xy,
                              const unsigned char* track_vis, long long total_samples, int mapping, float delta,
                              float loss_weight, float* loss, void* ws, int F, int H, int W, int depth_frame0,
                              int src_frame_lo, int src_frame_hi, void* stream);
int fm_track_loss_value(const void* ws, float loss_weight, float* loss, void* stream);
int fm_track_loss_bwd_sharded(const float* depth, const float* k4, const float* extrinsics, const int* segments,
                              int num_segments, int max_rows, int max_points, const float* track_xy,
                              const unsigned char* track_vis, long long total_samples, int mapping, float delta,
                              float loss_weight, const float* grad_out, float* g_depth, float* g_extrinsics,
                              float* g_k4, void* ws, int F, int H, int W, int depth_frame0, int src_frame_lo,
                              int src_frame_hi, void* stream);

/* model_wrapper_overfit.py:104-105 optim.Adam(lr): torch's single-tensor Adam update (no
 * amsgrad, no weight decay), one fused pass; `step` is the 1-based step number. */
int fm_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, size_t count,
                 double lr, double beta1, double beta2, double eps, int step, void* stream);

/* ---- step clock: the step-dependent scalars in device memory (CUDA-graph capture of whole steps) --
 * FM_STEP_CLOCK_BYTES of zero-initialised device memory = {u32 step, u32 focal_step, f32 step_size,
 * bc2_sqrt, focal_step_size, focal_bc2_sqrt, u64 seed}.  fm_step_clock_tick advances `step` (and
 * `focal_step` when tick_focal != 0) by one and refreshes torch.optim.Adam's bias-correction scalars
 * lr / (1 - beta1^t), sqrt(1 - beta2^t) (model_wrapper_overfit.py:104-105) and a per-step seed
 * (splitmix64 of base_seed and step) for fm_random_subset_clock (intrinsics_softmin.py:90). */
#define FM_STEP_CLOCK_BYTES 32
int fm_step_clock_tick(void* clock, double lr, double beta1, double beta2, unsigned long long base_seed,
                       int tick_focal, void* stream);
int fm_adam_step_clock(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, size_t count,
                       const void* clock, int focal_clock, double beta1, double beta2, double eps, void* stream);
int fm_random_subset_clock(const void* clock, long long N, int n, int64_t* out, void* stream);

/* intrinsics_softmin.py:84-131, the candidate sweep on the first frame pair.  For each of
 * the num_candidates intrinsics in cand_k4 (B*num_candidates, 2, 4: one k4 row per virtual
 * frame) run Procrustes at the `indices` points (depth frames 0/1, backward flow and weights
 * of pair 0 are SHARED by all candidates: no (n,2,H,W,3) temporary) and sum the weighted
 * backward-flow error err (B, num_candidates) = sum |(uv - xy - flow) * w|.  rt (B*n, 3, 4)
 * receives the per-candidate poses (needed by the backward).  The backward takes d/d err
 * and ACCUMULATES into g_depth (B,F,H,W) and g_weights (B,F-1,H,W) (frames 0/1, pair 0).
 * weights may be stored as logits (weight_sensitivity != 0), see fm_overfit_step. */
size_t fm_softmin_workspace_bytes(int B, int num_candidates);
int fm_softmin_sweep_fwd(const float* depth, const float* weights, float weight_sensitivity,
                         const float* backward_flow, const int64_t* indices, int num_indices,
                         const float* cand_k4, int num_candidates, float* err, float* rt, void* ws, int B,
                         int F, int H, int W, void* stream);
int fm_softmin_sweep_bwd(const float* depth, const float* weights, float weight_sensitivity,
                         const float* backward_flow, const int64_t* indices, int num_indices,
                         const float* cand_k4, int num_candidates, const float* rt, const float* g_err,
                         float* g_depth, float* g_weights, void* ws, int B, int F, int H, int W,
                         void* stream);
/* intrinsics_softmin.py:90 `torch.randperm(h * w)[:n]`: n distinct uniformly random pixel indices
 * (int64) as the head of a keyed pseudo-random permutation of [0, N), O(n) work. */
int fm_random_subset(unsigned long long seed, long long N, int n, int64_t* out, void* stream);

/* intrinsics_softmin.py:126-139: softmin((err - min) * 10) over the candidates and the focal
 * estimate f_hat (B) = sum softmin_n * cand_focal_n; and d f_hat / d err for the backward. */
int fm_softmin_focal(const float* err, const float* cand_focal, int num_candidates, int B, float* softmin,
                     float* focal, void* stream);
int fm_softmin_focal_bwd(const float* softmin, const float* cand_focal, const float* focal,
                         const float* g_focal, int num_candidates, int B, float* g_err, void* stream);

/* Packed tracks (see fm_track_loss_fwd), device pointers. */
typedef struct {
  const int* segments;
  const float* xy;
  const unsigned char* vis;
  int num_segments, max_rows, max_points;
  long long total_samples;
} fm_packed_tracks;

/* One whole optimisation step of the explicit-depth overfit run (batch size 1) without
 * leaving the library: what model_wrapper_overfit.py:51-73 (training_step) + :104-105
 * (Adam) do through autograd, as one sequence of launches on `stream`:
 *   [k4 from the focal parameter] -> Procrustes poses (model.py:54-90) -> flow loss with its
 *   direct gradients (loss_flow.py:31-70) -> [track loss fwd/bwd on the chained poses,
 *   loss_tracking.py:28-61] -> Procrustes backward (SURVEY A.7) -> Adam on depth, weight
 *   logits and focal length.
 * The correspondence weights are sigmoid(weight_sensitivity * weight_logits)
 * (backbone_explicit_depth.py:40), evaluated inside the kernels; weight_logits == NULL means
 * use_correspondence_weights = false (model.py:67-68).  focal == NULL keeps k4 as given
 * (no focal gradient).  focal == NULL together with g_k4 == NULL and track_g_k4 == NULL is the
 * constant-intrinsics step (intrinsics_ground_truth.py: K given per frame, e.g. calibrated data): it
 * computes no intrinsics gradient at all -- the Procrustes backward and the tracking sweep run without
 * their K accumulators; g_k4 == NULL with a focal parameter or a track_g_k4 is refused.  step = 0
 * computes loss and gradients but skips Adam.
 * Gradients of the step are left in g_depth / g_weights / g_focal / g_k4. */
typedef struct {
  int F, H, W;
  float* depth;                 /* (F,H,W) parameter, updated in place            */
  float* weight_logits;         /* (F-1,H,W) parameter or NULL                    */
  float weight_sensitivity;
  float* focal;                 /* device scalar parameter or NULL                */
  float* k4;                    /* (F,4): written from focal, or read if focal == NULL */
  const int64_t* indices;       /* Procrustes point subset or NULL (all pixels)   */
  int num_indices;
  const float *fflow, *bflow, *fmask, *bmask;
  const double* mask_sum;
  int mapping;
  float delta, flow_weight;
  const fm_packed_tracks* tracks; /* host struct with device pointers, or NULL    */
  float track_weight;
  float *m_depth, *v_depth, *m_weights, *v_weights, *m_focal, *v_focal;
  double beta1, beta2, eps;
  int step;                     /* 1: update the parameters with Adam, on the bias corrections of `clock`'s
                                   current tick (needs a clock); 0: no update.  Other values are refused. */
  float *g_depth, *g_weights, *g_focal, *g_k4;  /* gradient buffers (written)     */
  float *rt, *loss;             /* outputs: (F-1,3,4) poses, flow loss             */
  float *extrinsics, *g_extrinsics, *g_rt, *track_g_k4, *track_loss; /* tracking only */
  void *ws, *track_ws;
  int defer_adam;               /* With step = 1.  0: Adam on everything inside the step.  1 (softmin stage):
                                   the sweep's backward (fm_softmin_sweep_bwd) still has to add its gradients
                                   to depth frames 0/1 and to the weights of pair 0, so only the weight logits
                                   of pairs >= 1 are updated here; the caller runs Adam on depth and on pair
                                   0's logits afterwards.  2 (pair sharding): the weight logits of ALL pairs
                                   are updated here (their gradient is rank-local and final), depth and focal
                                   length wait for the caller's collective */
  int phase;                    /* FM_STEP_ALL, or a split step (pair sharding with a tracking loss; the
                                   autograd drop-in surface, where the losses' values are needed before
                                   backward() runs): FM_STEP_FORWARD computes rt, the flow loss with its
                                   direct depth gradient and pose-gradient sums in ws and -- with tracks --
                                   the chained poses and the tracking loss; FM_STEP_BACKWARD resumes with
                                   the tracking backward (with tracks) or the caller's extra pose gradient
                                   g_rt (F-1,3,4) / intrinsics gradient track_g_k4 (F,4) (tracks == NULL,
                                   either may be NULL), then the Procrustes backward; step must be 0 in
                                   the two halves' common use (no parameter may change in between) */
  const float* flow_grad_scale;  /* FM_STEP_BACKWARD only: device scalars d total / d flow loss and     */
  const float* track_grad_scale; /* d total / d tracking loss (autograd's grad_output), or NULL (= 1) */
  const void* clock;             /* device step clock (fm_step_clock_tick), the caller ticks it before an
                                    update step; NULL only with step = 0.  Adam's bias corrections come from
                                    its current tick (the focal length's from its own focal count), so that
                                    consecutive steps are launches with identical arguments: a CUDA graph
                                    can replay them */
  const float* moments_k4;       /* NULL, or the intrinsics (F,4) with which fm_procrustes_moments has ALREADY
                                    accumulated this step's moment sums into `ws` (all-pixel Procrustes only;
                                    same principal points as k4, any focal lengths): the step then starts at the
                                    pose solve and rescales the sums to its own K.  Lets the caller run the
                                    moment pass beside the work that produces the focal length (the softmin sweep). */
  /* Per-step metrics log (model_wrapper_overfit.py:63-71 train/loss/<name>, train/intrinsics/f[xy]_error;
     visualizer_trajectory.py metrics/ate).  metrics_log == NULL: off.  Otherwise (needs FM_STEP_ALL, `clock`
     and `extrinsics`) the step writes row (clock.step - 1) mod metrics_capacity of the (metrics_capacity, 5)
     float ring: weighted flow loss, weighted tracking loss (0 without tracks), |gt_fx - mean_f k4[f,0]|,
     |gt_fy - mean_f k4[f,1]|, and fm_trajectory_ate of the translations of the chained poses (written to
     `extrinsics`, also without tracks) against gt_positions.  The row describes the parameters this step
     evaluated, before its Adam update.  It is computed on a side stream beside the backward half: one
     extra launch with tracks, two without (the pose chain). */
  const float* gt_positions;     /* (F,3) ground-truth camera centres, or NULL: ATE column is NaN */
  float gt_fx, gt_fy;            /* frame means of the normalised GT intrinsics, NaN: columns NaN */
  float* metrics_log;            /* (metrics_capacity, 5) ring, or NULL = off */
  int metrics_capacity;
  /* fm_overfit_step_videos, split step only (FM_STEP_FORWARD / FM_STEP_BACKWARD; fm_overfit_step refuses it):
     0 = flow_grad_scale is ONE device scalar for the whole batch (pretraining) and the step takes no tracks;
     1 = B networks' overfits: flow_grad_scale and track_grad_scale are device (B,) arrays (NULL = all 1),
     d total / d loss_b and d total / d track_loss_b of every video b, and the step may take tracks. */
  int video_grad_scales;
  /* 0 or 1; fm_overfit_step_videos ignores it.  fm_overfit_step optimises one video and refuses B > 1:
     several videos go to fm_overfit_step_videos. */
  int B;
  const float* gt_fxfy;          /* fm_overfit_step_videos with metrics_log: (B, 2) frame means of the GT
                                    intrinsics, NaN: none */
} fm_overfit_step_args;
#define FM_STEP_ALL 0
#define FM_STEP_FORWARD 1
#define FM_STEP_BACKWARD 2
/* Stream semantics: everything is ordered after the work already in `stream` and is complete, in
 * stream order, when later work of `stream` runs.  With `tracks` the call internally forks part of
 * its launches onto a second, library-owned stream (the tracking sweep beside the flow-loss kernel,
 * the tracking loss's depth scatter beside the Procrustes backward) and joins it again with events
 * before it returns; under stream capture (cudaStreamCaptureModeThreadLocal / Relaxed) these become
 * parallel branches of the caller's graph. */
int fm_overfit_step(const fm_overfit_step_args* args, void* stream);

/* Several videos (same H, W; equal or different lengths), packed along the frame axis: video b owns the frames
 * [frame_offset[b], frame_offset[b + 1]) of every per-frame buffer (T, ...) and the pairs
 * [frame_offset[b] - b, frame_offset[b + 1] - b - 1) of every per-pair buffer (P, ...), P = T - B; no pair
 * crosses two videos.  The three tables live in device memory and belong to the caller, who keeps them
 * consistent (frame_offset[0] = 0, frame_offset[B] = T, every video >= 2 frames). */
typedef struct {
  int B;                    /* number of videos */
  int T;                    /* frames of all videos */
  const int* frame_offset;  /* (B + 1) first frame of every video, then T */
  const int* frame_video;   /* (T) the video of every frame */
  const int* pair_video;    /* (T - B) the video of every pair */
} fm_video_layout;
/* fm_overfit_step for B independent videos in one step: args->B and args->F are ignored, every per-frame /
 * per-pair buffer has the packed layout above, and the per-video scalars (focal, mask_sum, loss,
 * track_loss, g_focal, m_focal, v_focal) hold B values.  Video b gets what a one-video step on it gets:
 * its flow loss is normalised by its own mask_sum[b] and its tracking loss by its own valid count ("or 1"
 * per video), and its poses chain from the identity at its own frame 0.  (The reference's LossFlow
 * normalises a batch by ONE pooled mask sum; this is B overfit runs, not a pooled batch.)  Tracks: the
 * segments of video b carry start frames frame_offset[b] + s (they never cross videos); track_ws is
 * fm_track_workspace_bytes(T, total_samples).  Metrics: gt_positions (T, 3), NaN first position of a
 * video = no ground truth; the ring is (metrics_capacity, B, 5).  ws: fm_workspace_bytes_videos(B, T).
 * Refuses defer_adam = 1 together with step = 1 and weight logits (the caller updates the logits after
 * the sweep's backward).
 * Phases: FM_STEP_ALL, or the two halves of a split step, FM_STEP_FORWARD then FM_STEP_BACKWARD (a network
 * backbone's batch, whose depths / weights come from the network and whose update the caller owns).  A
 * split step needs step = 0, defer_adam = 0 and metrics_log == NULL.  With video_grad_scales = 0 it takes no
 * tracks and its flow_grad_scale is ONE device scalar for the whole batch, d total / d loss_b for every video b:
 * the sum of the B losses is the objective.  With video_grad_scales = 1 (B networks, each overfitting its own
 * video) it is B independent split steps: the forward computes each video's flow loss (by its own mask_sum[b])
 * and, with tracks, the chained poses and each video's tracking loss into track_loss[b]; the backward scales
 * video b's flow and tracking gradients, its focal gradient included, by flow_grad_scale[b] and
 * track_grad_scale[b].  The reference's LossFlow at b > 1 (pretraining) is such a sum when every mask_sum[b] holds the
 * pooled normaliser M = sum over all videos of their forward + backward mask sums ("or 1"): loss[b] is then
 * weight * S_b / M and sum_b loss[b] the pooled loss. */
int fm_overfit_step_videos(const fm_overfit_step_args* args, const fm_video_layout* layout, void* stream);
size_t fm_workspace_bytes_videos(int B, int T);
/* fm_procrustes_moments for packed videos (see fm_overfit_step_args.moments_k4). */
int fm_procrustes_moments_videos(const float* depth, const float* k4, const float* backward_flow,
                                 const float* weights, float weight_sensitivity, void* ws,
                                 const fm_video_layout* layout, int H, int W, void* stream);
/* fm_softmin_sweep_fwd / _bwd on pair 0 of every video of a packed layout (cand_k4, err, rt, ws: as
 * there with B = layout->B). */
int fm_softmin_sweep_fwd_videos(const float* depth, const float* weights, float weight_sensitivity,
                                const float* backward_flow, const int64_t* indices, int num_indices,
                                const float* cand_k4, int num_candidates, float* err, float* rt, void* ws,
                                const fm_video_layout* layout, int H, int W, void* stream);
int fm_softmin_sweep_bwd_videos(const float* depth, const float* weights, float weight_sensitivity,
                                const float* backward_flow, const int64_t* indices, int num_indices,
                                const float* cand_k4, int num_candidates, const float* rt, const float* g_err,
                                float* g_depth, float* g_weights, void* ws, const fm_video_layout* layout,
                                int H, int W, void* stream);
/* fm_adam_step_clock on the rows lo <= r < min(hi, rows of video b) of every video b of a packed layout,
 * rows = its frames (pairs = 0: depth) or its pairs (pairs = 1: weight logits): one launch for the same
 * rows of every video (the softmin stage, where the sweep still adds to frames 0 / 1 of each video while
 * the others are final). */
int fm_adam_step_clock_frames_videos(float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                                     size_t frame_elems, const fm_video_layout* layout, int pairs, int frame_lo,
                                     int frame_hi, const void* clock, int focal_clock, double beta1,
                                     double beta2, double eps, void* stream);
/* fm_pose_chain / fm_pose_chain_bwd for a packed layout: rt (T - B, 3, 4), extrinsics (T, 4, 4). */
int fm_pose_chain_videos(const float* rt, float* extrinsics, const fm_video_layout* layout, void* stream);
int fm_pose_chain_bwd_videos(const float* rt, const float* extrinsics, const float* g_extrinsics, float* g_rt,
                             const fm_video_layout* layout, void* stream);

/* Phase A alone (all pixels, one video): the 16 weighted moment sums of every frame pair into `ws`,
 * for intrinsics `k4` (F,4); `weights` are plain weights (weight_sensitivity == 0) or logits.  See
 * fm_overfit_step_args.moments_k4.  (Model.forward's first reduction, model.py:75-90 with
 * projection.py:222-242.) */
int fm_procrustes_moments(const float* depth, const float* k4, const float* backward_flow,
                          const float* weights, float weight_sensitivity, void* ws, int F, int H, int W,
                          void* stream);

/* ---- stages either side of the hot path (SURVEY 8(f) rank 4) ---------------------------- */

/* flow/flow_predictor.py:60-82 compute_consistency_mask: videos (B,F,3,H,W) planar frames, flow
 * (B,F-1,H,W,2) in normalised units -> mask (B,F-1,H,W) = (1 - max_c |I_src - bilinear_zero_pad(
 * I_tgt, xy + flow)|)^8.  reverse = 0: src frame i, tgt frame i+1 (forward flow); reverse = 1:
 * src i+1, tgt i (the backward flow as stored in Flows.backward, :92-99). */
int fm_consistency_mask(const float* videos, const float* flow, float* mask, int B, int F, int H, int W,
                        int reverse, void* stream);

/* flow/flow_predictor.py:40-58 rescale_flow / rescale_mask and misc/cropping.py:19-27
 * resize_batch: F.interpolate(mode="bilinear", align_corners=False) of channels-last images
 * in (items,Hin,Win,C) -> out (items,Hout,Wout,C), C in {1,2,3}. */
int fm_resize_bilinear(const float* in, float* out, int items, int Hin, int Win, int Hout, int Wout,
                       int channels, void* stream);

/* export/colmap.py:84-101 (the point cloud of export_to_colmap): depth (F,H,W), k4 (F,4),
 * camera-to-world extrinsics (F,4,4) -> xyz (F*H*W,3), frames concatenated, row-major pixels. */
int fm_world_points(const float* depth, const float* k4, const float* extrinsics, float* xyz, int F, int H,
                    int W, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FLOWMAP_B200_H */
