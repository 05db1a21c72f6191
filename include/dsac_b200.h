/*
 * dsac_b200.h -- C ABI of the H100-native DSAC soft-argmax hypothesis engine.
 *
 * This is the drop-in boundary for the ONE hot path of cvlab-dresden/DSAC
 * (core/cnn_softam.h processImage :960-1180 and the backward assembled in
 * train_ransac_softam.cpp:288-412).  Plain pointers and sizes only -- no CUDA, torch or
 * OpenCV types -- so the reference's C++ drivers (or any FFI) can bind it directly; see
 * INTEGRATION.md for the binding a DSAC maintainer would add.
 *
 * Each entry point cites the reference interface it replaces.
 *
 * Conventions (identical to the reference):
 *   - scene coordinates: int16 millimetres, [frame][y*40+x][3]     (types.h:43-51, cnn_softam.h:265)
 *   - sampling grid:     int32 pixel (x,y), [frame][y*40+x][2]      (cnn_softam.h:283-309)
 *   - "cv pose": 6 doubles (rvec[3], tvec[3] in mm), scene->camera, OpenCV axes (types.h:91)
 *   - "jp pose": 12 doubles (R row-major 3x3, t[3] in mm) after cv2our (types.h:186-214)
 *   - hypothesis h of a frame owns the 4 cells img_idx[h][0..3] = y*40+x (cnn_softam.h:1037)
 *
 * Error behaviour: every call returns 0 on success, <0 on failure (dsac_last_error gives
 * the text); numeric failures are value-encoded per frame exactly like the reference
 * (zero pose on PnP failure, cnn_softam.h:66-71; NaN translation -> 0, types.h:208-211).
 * The engine never falls back to a CPU path: without a CUDA device dsac_engine_create fails.
 */
#ifndef DSAC_B200_H
#define DSAC_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DSAC_GRID 40                      /* CNN_OBJ_PATCHSIZE, lua_calls.h:33 */
#define DSAC_N (DSAC_GRID * DSAC_GRID)    /* 1600 scene coordinates per frame */
#define DSAC_MAXINPUT 100.0f              /* CNN_OBJ_MAXINPUT, lua_calls.h:36 */
#define DSAC_MAX_HYPS 1024
#define DSAC_MAX_REF_STEPS 16
#define DSAC_MAX_PRIORS 16

#define DSAC_OK 0
#define DSAC_ERR_ARG (-1)
#define DSAC_ERR_CUDA (-2)
#define DSAC_ERR_CAPACITY (-3)
#define DSAC_ERR_NODEVICE (-4)

/* per-frame status bits (dsac_forward_out.status) */
#define DSAC_ST_SAMPLER_EXHAUSTED 1u      /* max_candidates reached before n_hyps accepts */
#define DSAC_ST_BORDER_PATCH 4u           /* dsac_gather_patches_device met a border cell (the reference would skip it, cnn_softam.h:236-240) */
#define DSAC_ST_REFINE_ABORTED 2u         /* refinement stopped early (<50 inliers / NaN), cnn_softam.h:1136,1147 */
#define DSAC_ST_OBJ_DRAW_EXHAUSTED 8u     /* dsac_obj_draw_device: a patch found no valid centre within max_attempts */
#define DSAC_ST_DEPTH_DROPPED 16u         /* dsac_register_depth_device: registration targets outside the image were dropped */
#define DSAC_ST_BAD_WEIGHTS 32u           /* guided sampling: a NaN or +inf logit, or fewer than 4 cells with weight > 0; nothing sampled */
#define DSAC_ST_NO_DEPTH 64u              /* RGB-D pass: fewer than 4 cells with depth; nothing sampled */
#define DSAC_ST_BAD_PRIOR 128u            /* a non-finite prior or an information matrix that is not positive definite; nothing sampled */
#define DSAC_ST_BAD_RIG 256u              /* dsac_forward_rig_device: a non-finite extrinsic; the rig's outputs are zero */

typedef struct dsac_engine dsac_engine;

/* Replaces GlobalProperties::pP / dP as consumed by the drivers
 * (properties.h:40-80, test_ransac_softam.cpp:44-57, train_ransac_softam.cpp:46-66). */
typedef struct dsac_config {
    double focal, cx, cy;     /* getCamMat(), properties.cpp:308-323 */
    int32_t n_hyps;           /* -rI  ransacIterations (256) */
    int32_t thr2d;            /* -rT2D ransacInlierThreshold2D truncated to int (10) */
    int32_t inlier_count;     /* -rB  ransacBatchSize (100) */
    int32_t ref_steps;        /* -rRI ransacRefinementIterations (8) */
    double sub_sample;        /* -rSS ransacSubSample (0.01) */
    double alpha, beta;       /* soft-inlier score s_h = alpha * sum_i sigmoid(beta*(thr2d - e_hi)) */
    uint32_t seed;            /* ThreadRand seed (1305), thread_rand.h:100 */
    int32_t n_streams;        /* sampler streams per frame (= OMP threads of the reference loop) */
    uint32_t stream_skip;     /* raw mt19937 words stream 0 skips first (6400 = stochasticSubSample's drand) */
    int32_t max_candidates;   /* bound on candidates per stream (the reference loops forever) */
    int32_t fix_q4;           /* 0 = bug-compatible dScore column layout (cnn_softam.h:628,641) */
    double grad_clamp;        /* clampE2E of the score backward (train_score_softam.lua:13,97) */
    int32_t write_diffmaps;   /* 1 = materialise the HxN reprojection-error matrix (reference behaviour) */
    int32_t device;           /* CUDA device ordinal */
    int32_t max_frames;       /* frames per call the engine is sized for */
    int32_t hyps_per_cta;     /* scoring tile (hypotheses per CTA); 0 = auto */
} dsac_config;

/* Caller-allocated host outputs of the forward pass; any pointer may be NULL.
 * These are the by-reference outputs of processImage (cnn_softam.h:971-988). */
typedef struct dsac_forward_out {
    double* hyp_pose;         /* [n][H][6]  hyps (cv)                  cnn_softam.h:974 */
    int32_t* img_idx;         /* [n][H][4]  imgIdx                     cnn_softam.h:979 */
    int32_t* cand_idx;        /* [n][H]     index of the accepted candidate in its stream */
    double* scores;           /* [n][H]     scores before softmax      cnn_softam.h:1072 */
    double* sf;               /* [n][H]     sfScores                   cnn_softam.h:981 */
    float* diffmaps;          /* [n][H][N]  diffMaps                   cnn_softam.h:1066 */
    double* entropy;          /* [n]        sfEntropy                  cnn_softam.h:972 */
    double* avg_pose;         /* [n][6]     avgHyp (cv)                cnn_softam.h:976 */
    double* ref_pose;         /* [n][6]     refAvgHyp (cv)             cnn_softam.h:975 */
    int32_t* inlier_map;      /* [n][N]     inlierMap                  cnn_softam.h:985 */
    int32_t* ref_steps_done;  /* [n] */
    int32_t* n_perm_steps;    /* [n]        permutations consumed (non-empty pixelIdxs entries) */
    double* loss;             /* [n]        loss   (needs gt)          cnn_softam.h:971 */
    double* rot_err;          /* [n]        rotErr                     cnn_softam.h:988 */
    double* t_err;            /* [n]        tErr                       cnn_softam.h:987 */
    int32_t* correct;         /* [n]        correct                    cnn_softam.h:973 */
    int64_t* n_candidates;    /* [n]        minimal sets drawn (all streams) */
    uint32_t* status;         /* [n]        DSAC_ST_* */
} dsac_forward_out;

/* Device-side views (valid until the next call on the engine); for zero-copy consumers
 * such as a CNN scorer behind the score seam (lua_calls.h:284-341). */
typedef struct dsac_device_view {
    const float* diffmaps;    /* [n][H][N] or NULL */
    const double* hyp_pose;   /* [n][H][6] */
    const double* scores;     /* [n][H] */
    const double* sf;         /* [n][H] */
    const double* avg_pose;   /* [n][6] */
    const double* ref_pose;   /* [n][6] */
    const int32_t* img_idx;   /* [n][H][4] */
} dsac_device_view;

/* Fills the defaults of GlobalProperties::GlobalProperties() (properties.cpp:39-83). */
int dsac_default_config(dsac_config* cfg);

/* Engine life-cycle.  Replaces the per-process state the drivers set up before the frame
 * loop (test_ransac_softam.cpp:66-82).  One engine per GPU; calls on one engine are not
 * re-entrant, different engines may be driven from different host threads. */
int dsac_engine_create(const dsac_config* cfg, dsac_engine** out);
void dsac_engine_destroy(dsac_engine* e);
const char* dsac_last_error(const dsac_engine* e);   /* e may be NULL: last create error */
int dsac_engine_config(const dsac_engine* e, dsac_config* out);

/* Forward of processImage (cnn_softam.h:960-1180) for n frames, HOST buffers:
 * copies inputs to the device, runs sampling -> HxN reprojection errors -> soft-inlier
 * score -> softmax / soft-argmax -> refinement -> evaluation, copies results back.
 * frame0: global index of the first frame (keys the sampler streams: stream s of frame g
 * is mt19937(seed + g*n_streams + s)), so results do not depend on how a batch is sharded.
 * pix_shared != 0: one sampling grid [N][2] shared by all frames.
 * gt_jp: [n][12] ground-truth jp poses or NULL. */
int dsac_forward(dsac_engine* e, int32_t n_frames, int64_t frame0, const int16_t* coords, const int32_t* pix,
                 int32_t pix_shared, const double* gt_jp, dsac_forward_out* out);

/* The same pass split in two, for drivers that overlap the copies of one batch with the kernels of another
 * (the frame loop of test_ransac_softam.cpp:107-160 with two engines in flight): dsac_forward_submit enqueues
 * H2D -> kernels -> D2H on the engine's streams and returns; dsac_forward_wait blocks until the results are in `out`.
 * coords / pix / gt_jp / out must stay valid (and should be page-locked for the copies to be asynchronous) until the
 * wait returns; one pass per engine may be pending.  dsac_forward == submit + wait. */
int dsac_forward_submit(dsac_engine* e, int32_t n_frames, int64_t frame0, const int16_t* coords, const int32_t* pix,
                        int32_t pix_shared, const double* gt_jp, dsac_forward_out* out);
int dsac_forward_wait(dsac_engine* e);

/* Same pass with inputs already resident in device memory; results stay on the device
 * (dsac_fetch copies them out).  stream: a cudaStream_t cast to void* (NULL = default). */
int dsac_forward_device(dsac_engine* e, int32_t n_frames, int64_t frame0, const int16_t* d_coords,
                        const int32_t* d_pix, int32_t pix_shared, const double* d_gt_jp, void* stream);
/* dsac_fetch copies with cudaMemcpyDefault on `stream` and synchronises it: every destination may be host or device
 * memory, except n_candidates, which is summed on the host and must be host memory. */
int dsac_fetch(dsac_engine* e, int32_t n_frames, dsac_forward_out* out, void* stream);
int dsac_device_view_get(dsac_engine* e, dsac_device_view* view);

/* Per-frame cameras: one batch may mix focal lengths and principal points (images of different sensors, SfM
 * reconstructions, scale augmentation).  The reference has one camera per process (getCamMat(), properties.cpp:308-323);
 * without this call so does the engine (dsac_config's). */
typedef struct dsac_camera { double focal, cx, cy; } dsac_camera;   /* getCamMat(), per frame */

/* Cameras of the frames of the following passes: cams[i] belongs to frame i of the call (local index, like coords --
 * NOT the global frame0 + i).  cams is a HOST array of n entries; it is validated here (focal finite and > 0, cx / cy
 * finite), staged in page-locked memory the engine owns and copied to an engine-owned device buffer on `stream`
 * (a cudaStream_t, NULL = default), after the engine's last forward pass; the passes that follow wait for the copy on
 * whichever stream they run.  The setting is sticky: every later forward on this engine (dsac_forward, _submit, _device,
 * dsac_forward_dsac, _device) must have n_frames == n (else DSAC_ERR_ARG) until it is changed.  cams == NULL (n
 * ignored): back to dsac_config's camera.
 * DSAC_ERR_ARG, with the engine left as it was: n outside [1, max_frames], a bad entry (dsac_last_error names its
 * index), or a submitted pass that has not been awaited.
 * A backward pass, and dsac_refined_jp6_device, belong to the forward pass before them and so to its cameras: after a
 * dsac_set_cameras they return DSAC_ERR_ARG until the next forward.
 * dsac_score_maps_device and the pre-training data paths do not use this table: their frame index is a dataset index, not
 * a pass index, and their per-frame cameras come from dsac_set_dataset_cameras.  No distortion and no separate fx / fy:
 * the reference has neither. */
int dsac_set_cameras(dsac_engine* e, int32_t n, const dsac_camera* cams, void* stream);

/* Guided sampling (Neural-Guided RANSAC, Brachmann & Rother, ICCV 2019): the minimal sets of the following passes are drawn
 * from learned per-cell weights instead of uniformly.  d_logits: DEVICE float32 [n][1600], cell y*40+x, read on `stream`
 * into engine-owned tables (sized once for max_frames); the buffer may be reused once `stream` has passed this call.  Per frame w = softmax(logits) in fp64 and the sampler draws from the integer
 * weights q_j = floor(w_j 2^31): each point of a candidate is cell j with probability q_j / (Q - sum of the q already in the
 * candidate), Q = sum q; the random numbers are Philox4x32-10, key (seed, 0), counter (block, candidate index, lo32(z),
 * hi32(z)) for slot z = global frame * n_streams + stream (INTEGRATION.md, "Guided sampling").  -inf logits are allowed
 * (q = 0); a NaN or +inf logit, or fewer than 4 cells with q > 0, gives the frame DSAC_ST_BAD_WEIGHTS and no hypotheses
 * (zero poses, img_idx -1).  Acceptance, quotas and every later stage are the uniform path's; the DSAC variant's random
 * draw reads MT19937 stream 0 of the frame right after stream_skip.  Sticky like dsac_set_cameras: later passes must have
 * n frames; d_logits == NULL (n ignored) returns to the reference sampler.  The redraw of a repeated cell is unbounded as
 * in the reference: weights with nearly all mass on <= 3 cells and tiny nonzero weights elsewhere make a frame run for a
 * long time (INTEGRATION.md).  DSAC_ERR_ARG, with the engine left as it was:
 * n outside [1, max_frames], or a submitted pass that has not been awaited. */
int dsac_set_sampling_logits_device(dsac_engine* e, int32_t n, const float* d_logits, void* stream);
/* RGB-D localisation (Brachmann & Rother, TPAMI 2021): the hypotheses of the following passes are Kabsch fits of three
 * cells' scene coordinates to their eye coordinates instead of P3P solves, and the refinement fits the selected inliers
 * the same way instead of LM PnP.  d_depth: DEVICE float32 [n][1600], the depth in mm at each cell's grid pixel, cell
 * y*40+x; a cell has depth iff its value is finite and > 0.  Copied on `stream` into an engine-owned buffer (sized once
 * for max_frames); the buffer may be reused once `stream` has passed this call.  Cell c of frame g has the eye point
 * ((u - cx) d / f, (v - cy) d / f, d) in fp64, (u, v) its pix and (f, cx, cy) the frame's camera.  The candidate streams
 * (MT19937, or Philox when guided), quotas and max_candidates are unchanged; a candidate is accepted iff all four cells
 * have depth, neither triangle of cells 0..2 (scene, eye) is degenerate (|(P1 - P0) x (P2 - P0)| >= 1 mm^2), all four
 * points lie in front of the camera under the Kabsch fit of cells 0..2, and all four pass the reprojection check.  A
 * frame with fewer than 4 cells with depth gets DSAC_ST_NO_DEPTH and no hypotheses (zero poses, img_idx -1).  Scoring is
 * unchanged: every cell is scored, with or without depth.  Sticky like dsac_set_cameras: later passes must have n frames;
 * d_depth == NULL (n ignored) returns to RGB.  Every backward entry point differentiates an RGB-D pass with the same jobs
 * and central differences, the Kabsch fit in place of P3P and LM (depth is not differentiated); they,
 * dsac_refined_jp6_device and dsac_sampling_log_prob*_device refuse a pass after which the setting changed.
 * DSAC_ERR_ARG, with the engine left as it was: n outside [1, max_frames], or a submitted pass that has not been awaited. */
int dsac_set_cell_depth_device(dsac_engine* e, int32_t n, const float* d_depth, void* stream);
/* Pose priors (INTEGRATION.md, "Pose priors"): k caller poses per frame join the hypothesis pool of the following passes, for
 * a tracker's prediction or the last frame's refined pose.  d_poses: DEVICE float64 [n][k][6] cv poses (rvec, tvec mm,
 * scene->camera, the representation of hyp_pose and ref_pose).  Prior j of frame f takes hypothesis slot n_hyps - k + j:
 * hyp_pose its bits, img_idx (all four) and cand_idx -1; slots 0 .. n_hyps - k - 1 are drawn exactly as an engine with
 * n_hyps - k draws them (quotas stream_chunk(n_hyps - k, n_streams, s)); k == n_hyps samples nothing.  Everything after
 * sampling (scoring, the score seam, softmax, refinement, the DSAC draw, refine-all, every backward and the pose queries)
 * sees n_hyps hypotheses.  d_info: DEVICE float64 [n][k][6][6] or NULL.  If set, an information matrix Lambda_j (an inverse
 * covariance) per prior in the chart R = exp([w]x) R_j, t = t_j + tau (w rad, tau mm; inv(cov_xi + Q) of
 * dsac_pose_uncertainty_device is one), lower triangle read; a candidate the sampler would accept (the P3P pose after the
 * 4-point check, or the RGB-D Kabsch fit after its tests) is accepted only if min_j xi^T Lambda_j xi <= gate, xi =
 * (log(R_h R_j^T) principal, t_h - t_j) in fp64; a gated-out candidate is an ordinary rejection (counts, quotas,
 * max_candidates, DSAC_ST_SAMPLER_EXHAUSTED, the used candidates of dsac_sampling_log_prob_device).  gate: a chi^2 bound,
 * finite and > 0 with d_info, else ignored.  A frame with a non-finite prior entry, or a Lambda_j whose Cholesky has a pivot
 * below 1e-12 of its diagonal entry, gets DSAC_ST_BAD_PRIOR, samples nothing and has all n_hyps slots empty (zero pose,
 * img_idx -1); decided on the device, other frames unaffected.  Priors are constants of the backward passes: a prior's
 * dPNP is zero, its score is differentiated directly, and in the DSAC variant a selected prior has its inlier-cell
 * refinement jobs and no minimal-set jobs.  Copied on `stream` into engine-owned buffers (sized once for max_frames x
 * DSAC_MAX_PRIORS); the caller's buffers may be reused once `stream` has passed this call.  Sticky like dsac_set_cell_depth_device:
 * later passes must have n frames; d_poses == NULL (n, k ignored) clears the setting.  Every backward entry point,
 * dsac_refined_jp6_device, dsac_pose_uncertainty_device and dsac_sampling_log_prob*_device refuse a pass after which the
 * setting changed.  DSAC_ERR_ARG, with the engine left as it was: n outside [1, max_frames], k outside
 * [1, min(n_hyps, DSAC_MAX_PRIORS)], a bad gate, or a submitted pass that has not been awaited. */
int dsac_set_pose_priors_device(dsac_engine* e, int32_t n, int32_t k, const double* d_poses, const double* d_info, double gate,
                                void* stream);

/* Scene-coordinate derivatives of the backward passes (INTEGRATION.md, "Implicit-function gradients").
 * DSAC_DERIV_CENTRAL (the default): the reference's central differences.  DSAC_DERIV_IMPLICIT: two quantities change.
 *   dRefineObj  the implicit-function derivative of the refined pose with respect to the cells the last accepted refinement
 *               step fitted (LM reprojection or, for RGB-D, Kabsch objective over that frozen set, full Hessian), dense
 *               over those cells, zero elsewhere, with no sub-sampling: sub_sample neither limits nor affects the backward.
 *               A pose with no accepted step, a Hessian that is not positive definite or a non-finite result gives zeros.
 *               DSAC variant: per selected hypothesis, the support cells excluded; only the 9 minimal-set pairs remain jobs.
 *   dPNP        the implicit-function derivative of the P3P equations of points 0..2 at the hypothesis (RGB-D: of the
 *               3-point Kabsch fit); the 4th point's columns are zero; a singular or non-finite solve zeroes the hypothesis.
 * Everything else (dRefineHyp, the minimal-set pairs, dScore, the score seam, fix_q4) is unchanged.  Sticky; read when a
 * backward call starts (dsac_backward, _device, _pose_device, dsac_backward_dsac, _device, _pose_device), so it may change
 * between a forward and its backward.  DSAC_ERR_ARG, with the engine left as it was: any other mode, or a submitted pass
 * that has not been awaited. */
#define DSAC_DERIV_CENTRAL 0
#define DSAC_DERIV_IMPLICIT 1
int dsac_set_coord_derivatives(dsac_engine* e, int32_t mode);

/* The integer weights q [n][1600] of the setting in force (DEVICE uint32), the distribution the sampler draws from.
 * Waits for the setting's table; n must equal its frame count. */
int dsac_sampling_table_device(dsac_engine* e, int32_t n, uint32_t* d_q);
/* Log-probability of the last pass's draw, d_logp DEVICE float64 [n]: per frame the sum over the used candidates (stream s:
 * candidates 0 .. the one of its last accepted hypothesis, or all it drew if it ran out; accepted and rejected alike) of
 * sum_k [log w_{c_k} - log(1 - sum_{i<k} w_{c_i})].  _backward_device: d_grad_logits [n][1600] float32 = d_grad_logp[f] *
 * d log p_f / d logits_f, deterministic.  Both recompute the candidates from their counters.  DSAC_ERR_ARG if the last
 * pass was not guided, n differs from its frame count, the logits were set again since, or a submitted pass is pending. */
int dsac_sampling_log_prob_device(dsac_engine* e, int32_t n, double* d_logp, void* stream);
int dsac_sampling_log_prob_backward_device(dsac_engine* e, int32_t n, const double* d_grad_logp, float* d_grad_logits, void* stream);

/* Stage control for measurement: which stages dsac_forward_device runs. */
#define DSAC_STAGE_SAMPLE 1u
#define DSAC_STAGE_SCORE 2u
#define DSAC_STAGE_REFINE 4u
#define DSAC_STAGE_EVAL 8u
#define DSAC_STAGE_ALL 15u
int dsac_set_stages(dsac_engine* e, uint32_t mask);

/* Tail split of a batch (scheduling only, results are identical): the sampler runs one CTA per (frame, stream) in
 * waves of as many CTAs as the GPU holds; with the split on, the frames of the whole waves run on an internal
 * high-priority stream and the frames of the last, partial wave on the caller's stream, so that scoring / refinement
 * of the former fill the SMs the partial wave leaves idle.  mode 0: off; 1 (default): dsac_forward_device and the
 * blocking dsac_forward; 2: dsac_forward_submit as well.  Environment override at creation: DSAC_TAIL_SPLIT. */
int dsac_set_tail_split(dsac_engine* e, int32_t mode);

/* Number of kernels the engine launched since creation (bench.py's gpu_launches). */
int64_t dsac_launch_count(const dsac_engine* e);

/* Measurement aid for the sampler (the round-based pipeline of sampler_split.cuh): with the profile on, the engine records
 * a CUDA event after every sampler launch of a forward pass and counts the candidates per round.
 * dsac_sampler_profile_read waits for the last pass and returns
 *   ms[0..3]     device time in: generation + selection (k1_cells, k1_slot), conservative filter (k1_filter),
 *                full P3P solve (k1_solve), resume tail (k_sample; normally an empty launch);
 *   counts[0..3] candidates generated, candidates flagged by the filter, candidates accepted, rounds that had work. */
int dsac_sampler_profile(dsac_engine* e, int32_t enable);
int dsac_sampler_profile_read(dsac_engine* e, double ms[4], uint64_t counts[4]);
/* Development aid: per stream (first 8 of the last pass), the number of windows the speculative first round of a few streams
 * (k1_spec / k1_stitch, DESIGN.md section 5) stitched; 0 = speculation abandoned (the ordinary round generated the stream) or not used. */
int dsac_debug_spec_result(dsac_engine* e, int32_t out8[8]);

/* Score seam: replaces forward(diffMaps, stateObj) (lua_calls.h:284-300; call site
 * cnn_softam.h:1072).  If set, the engine materialises the diffmaps and calls the hook with
 * DEVICE pointers instead of evaluating the closed-form soft-inlier score.
 * diffmaps [n][H][N] float (row-major 40x40 images, lua_calls.h:98-104), scores [n][H] double. */
typedef int (*dsac_score_hook)(const float* d_diffmaps, int32_t n_frames, int32_t n_hyps, double* d_scores,
                               void* stream, void* user);
int dsac_set_score_hook(dsac_engine* e, dsac_score_hook fn, void* user);

/* The seam's adjoint: replaces backward(maps, stateObj, scoreOutputGradients, gradients) (lua_calls.h:312-341; call site
 * cnn_softam.h:607 in dScore, cnn.h:672 in dSMScore).  Called by dsac_backward / dsac_backward_dsac with DEVICE pointers:
 * the diffmaps of the preceding forward [n][H][N], the score output-gradients [n][H] already clamped to +-grad_clamp
 * (the clamp of train_score_softam.lua:97), and the buffer to fill: diffmap_grads [n][H][40][40] doubles, element (y, x) =
 * d score_h / d diffmap_h(y, x) -- what the reference holds in gradients[c](y, x) after lua_calls.h:326-338.
 * A forward hook and a backward hook must be registered together: with only one of them set the backward entry points
 * return DSAC_ERR_ARG (they would otherwise differentiate a score the forward did not compute). */
typedef int (*dsac_score_backward_hook)(const float* d_diffmaps, const double* d_score_grads, int32_t n_frames, int32_t n_hyps,
                                        double* d_diffmap_grads, void* stream, void* user);
int dsac_set_score_backward_hook(dsac_engine* e, dsac_score_backward_hook fn, void* user);

/* Backward of one training round (train_ransac_softam.cpp:288-394) for the n frames of the
 * preceding dsac_forward call: dLoss/dY, [n][N][3] doubles, row p = y*40+x
 * (what the driver hands to the coordinate-CNN backward, train_ransac_softam.cpp:412).
 * Optional diagnostics may be NULL. */
typedef struct dsac_backward_out {
    double* dloss_dobj;       /* [n][N][3] */
    double* dloss_dref;       /* [n][6]   dLossMax              maxloss.h:87 */
    double* dref_dhyp;        /* [n][36]  dRefineHyp            cnn_softam.h:738 */
    double* dref_dobj;        /* [n][6][N*3] dRefineObj         cnn_softam.h:853 (DSAC_DERIV_IMPLICIT: the dense IFT matrix) */
    double* score_grads;      /* [n][H]   scoreOutputGradients  train_ransac_softam.cpp:361-376 */
    double* dpnp;             /* [n][H][6][12] dPNP             cnn_softam.h:101 (DSAC_DERIV_IMPLICIT: by the IFT) */
} dsac_backward_out;
int dsac_backward(dsac_engine* e, int32_t n_frames, const int16_t* coords, const int32_t* pix, int32_t pix_shared,
                  const double* gt_jp, dsac_backward_out* out);

/* Soft-argmax backward of the preceding dsac_forward / dsac_forward_device / dsac_forward_submit pass over the same
 * n_frames, on the caller's `stream` (a cudaStream_t; ordered after that pass by an event), with the inputs that pass
 * read (they must still be valid).  All pointers are DEVICE pointers; nothing is synchronised.
 *   d_loss_grad   [n] dOuter/dLoss_f, the gradient arriving at the per-frame losses; NULL = 1
 *   d_dloss_dobj  [n][N][3] dLoss/dObj, exactly what dsac_backward returns; NULL = not written
 *   d_dloss_dpred [n][N][3] the coordinate CNN's gradient as lua/train_obj_softam.lua:101-105 hands it to model:backward:
 *                 float(d_loss_grad[f] * clamp(dLoss/dObj, +-clamp)), clamp before the scale, row y*40+x; NULL = not
 *                 written.  clamp <= 0: no clamp.  Like the reference it is per millimetre of the int16 grid (the network
 *                 predicts metres) and passes straight through the rounding and saturation of
 *                 dsac_coords_from_prediction_device (DESIGN.md quirk Q12). */
int dsac_backward_device(dsac_engine* e, int32_t n_frames, const double* d_loss_grad, double* d_dloss_dobj,
                         float* d_dloss_dpred, float clamp, void* stream);

/* Forward of the DSAC / RANSAC variant (SURVEY.md section 8f row N1): processImage of core/cnn.h:1028-1257 -- same sampling and
 * scoring, then draw() of the winning hypothesis (cnn.h:102-126), refinement of ALL hypotheses, per-hypothesis
 * losses and the expectation of the loss (cnn.h:137-151).  random_draw != 0 draws with the stream-0 generator
 * continuing after the sampler (pP.randomDraw, -rdraw), else arg-max.  Any output may be NULL. */
typedef struct dsac_dsac_out {
    double* hyp_pose;         /* [n][H][6]  hyps                     cnn.h:1042 */
    int32_t* img_idx;         /* [n][H][4]  imgIdx                   cnn.h:1046 */
    double* sf;               /* [n][H]     sfScores                 cnn.h:1048 */
    double* entropy;          /* [n]        sfEntropy                cnn.h:1040 */
    double* ref_pose;         /* [n][H][6]  refHyps                  cnn.h:1043 */
    double* losses;           /* [n][H]     losses                   cnn.h:1052 */
    int32_t* inlier_maps;     /* [n][H][N]  inlierMaps (support cells zeroed, cnn.h:1221-1227) */
    int32_t* steps_done;      /* [n][H] */
    double* expected_loss;    /* [n]        expectedLoss             cnn.h:1039 */
    int32_t* hyp_idx;         /* [n]        hypIdx                   cnn.h:1057 */
    double* rot_err;          /* [n]        of the drawn hypothesis  cnn.h:1056 */
    double* t_err;            /* [n]                                 cnn.h:1055 */
    int32_t* correct;         /* [n]                                 cnn.h:1041 */
    uint32_t* status;         /* [n] */
} dsac_dsac_out;
int dsac_forward_dsac(dsac_engine* e, int32_t n_frames, int64_t frame0, const int16_t* coords, const int32_t* pix,
                      int32_t pix_shared, const double* gt_jp, int32_t random_draw, dsac_dsac_out* out);
/* The same forward on device-resident inputs, on the caller's `stream`: every non-NULL field of d_out is a DEVICE pointer,
 * nothing is copied to the host or synchronised.  The inputs must stay valid until dsac_backward_dsac_device. */
int dsac_forward_dsac_device(dsac_engine* e, int32_t n_frames, int64_t frame0, const int16_t* d_coords, const int32_t* d_pix,
                             int32_t pix_shared, const double* d_gt_jp, int32_t random_draw, const dsac_dsac_out* d_out,
                             void* stream);

/* Backward of the DSAC / RANSAC variant (replaces the gradient block of train_ransac.cpp:304-381; must follow a
 * dsac_forward_dsac over the same n_frames with ground truth):
 *   path I  : sum over the hypotheses with sf_h > 1e-4 of sf_h * dLossMax(refined_h, gt) (maxloss.h:87) * dRefine_h
 *             (cnn.h:866-990: central differences with eps = 2 through refine(), cnn.h:787-852 -- 18 evaluations on the
 *             perturbed minimal set plus 6 per sub-sampled inlier pixel, all of them jobs of the refinement kernel);
 *   path II : dSMScore (cnn.h:726-767) with scoreOutputGradients_i = sf_i * (loss_i - sum_j sf_j loss_j)
 *             (cnn.h:733-741) and the closed-form score backward at the score seam, rows in row-major order.
 * dloss_dobj = path I + path II is what train_ransac.cpp:399 hands to backward() of the coordinate CNN. */
typedef struct dsac_backward_dsac_out {
    double* dloss_dobj;       /* [n][N][3]  dLoss_dObj               train_ransac.cpp:353-377 */
    double* path1;            /* [n][N][3]  nullable */
    double* path2;            /* [n][N][3]  nullable */
    double* score_grads;      /* [n][H]     scoreOutputGradients, nullable  cnn.h:733-741 */
    int32_t* n_selected;      /* [n]        hypotheses with sf > 1e-4, nullable */
    int32_t* n_refine_jobs;   /* [n]        refine() evaluations of path I, nullable (DSAC_DERIV_IMPLICIT: 18 per selected hypothesis,
                                 0 per selected pose prior) */
} dsac_backward_dsac_out;
int dsac_backward_dsac(dsac_engine* e, int32_t n_frames, dsac_backward_dsac_out* out);
/* The same backward after a dsac_forward_dsac(_device), on the caller's `stream` (ordered after that forward by an event):
 * every non-NULL field of d_out (NULL: none) is a DEVICE pointer.  d_loss_grad, d_dloss_dpred and clamp as in
 * dsac_backward_device, with dLoss/dObj = path I + path II.  The call reads back one pair of totals -- selected
 * hypotheses and refinement jobs, which size the finite-difference k_refine launch -- and so synchronises `stream` once
 * in the middle; no per-hypothesis or per-cell array crosses to the host. */
int dsac_backward_dsac_device(dsac_engine* e, int32_t n_frames, const double* d_loss_grad, const dsac_backward_dsac_out* d_out,
                              float* d_dloss_dpred, float clamp, void* stream);

/* Pose-valued outputs (INTEGRATION.md, "Pose-valued outputs").  All pointers are DEVICE pointers, the calls run on the
 * caller's `stream`, ordered after the preceding forward by an event, and need no ground truth.  A pose is the jp 6-vector
 * [rodrigues(R_jp); t_jp in mm] of Hypothesis(cv2our(pose)).getRodVecAndTrans() (Hypothesis.cpp:274-290): the vector
 * refine() and dLossMax work on.  A seeded backward is the reference's chain with the seed in place of dLossMax (with its
 * quirks, DESIGN.md), not a finite-difference-exact derivative of the pose.
 *
 * jp 6-vectors of the refined poses of the preceding pass: [n][6] after dsac_forward(_device/_submit),
 * [n][H][6] after dsac_forward_dsac(_device). */
int dsac_refined_jp6_device(dsac_engine* e, int32_t n_frames, double* d_jp6, void* stream);

/* Pose uncertainty of the refined poses of the preceding pass (INTEGRATION.md, "Pose uncertainty"): one job per frame after
 * dsac_forward(_device/_submit), one per hypothesis ([n][H], h fastest) after dsac_forward_dsac(_device).  Stream ordering
 * and input lifetime as in dsac_backward_device: ordered after the pass by an event, whose coords and pix must still be
 * valid; no ground truth.  S is the set of cells the job's last accepted refinement step fitted, m = |S|, r_i the residual
 * of that fit (RGB: reprojection with the frame's camera, px; RGB-D: R Y_i + t - e_i, mm) and J_i = dr_i/dxi at the refined
 * pose in the chart xi = (w, tau) of R = exp([w]x) R*, t = t* + tau (w rad, tau mm):
 *   cov_xi  = sigma2 (sum_S J_i^T J_i)^-1, the Gauss-Newton covariance of the fit over S held fixed,
 *   sigma2  = sum_S |r_i|^2 / (2m - 6) (RGB, px^2) or / (3m - 6) (RGB-D, mm^2),
 *   cov_jp6 = M cov_xi M^T in the jp 6-vector of dsac_refined_jp6_device, M = d jp6 / d xi.
 * ok = 0, with the covariances and sigma2 zero, when no step was accepted (n_fit = 0: DSAC_ST_NO_DEPTH, DSAC_ST_BAD_WEIGHTS,
 * empty hypotheses), the degrees of freedom are <= 0, the information is not positive definite, or a result is not
 * finite.  support is filled whatever ok is: the cells of all 1600, with or without depth, whose reprojection error at the
 * refined pose, in k_score's arithmetic with the frame's camera, is below thr2d.  The call changes no later result.
 * DSAC_ERR_ARG, with the engine left as it was: not after a forward over the same n_frames, a submitted pass that has not
 * been awaited, cameras or cell depth changed since the pass, or d_out NULL.  The outputs are not differentiated. */
typedef struct dsac_pose_uncertainty_out {   /* DEVICE pointers, each nullable; jobs = n or n*H */
    double* cov_jp6;          /* [jobs][6][6] covariance in the jp 6-vector */
    double* cov_xi;           /* [jobs][6][6] covariance in the left-perturbation chart (w rad, tau mm) */
    double* sigma2;           /* [jobs]       residual variance estimate (px^2 RGB, mm^2 RGB-D) */
    int32_t* n_fit;           /* [jobs]       m: cells of the last accepted step, 0 if none */
    int32_t* support;         /* [jobs]       cells with reprojection error < thr2d at the refined pose */
    int32_t* ok;              /* [jobs]       1 if the covariance is defined */
} dsac_pose_uncertainty_out;
int dsac_pose_uncertainty_device(dsac_engine* e, int32_t n_frames, const dsac_pose_uncertainty_out* d_out, void* stream);
/* The pipeline of the forward pass over n_frames whose refined poses the engine holds, i.e. whose poses
 * dsac_pose_uncertainty_device reads: DSAC_PASS_SOFTAM (n_frames jobs) or DSAC_PASS_DSAC (n_frames * n_hyps jobs, h fastest).
 * A caller that sizes the outputs of dsac_pose_uncertainty_device asks here rather than tracking its own forward calls,
 * since a refused forward leaves the engine's pass as it was.  DSAC_ERR_ARG (*pipeline untouched) when the engine holds no
 * pass over n_frames. */
#define DSAC_PASS_SOFTAM 1
#define DSAC_PASS_DSAC 2
#define DSAC_PASS_RIG 3            /* dsac_forward_rig_device: read by the rig backward, dsac_rig_refined_jp6_device and
                                      dsac_rig_pose_uncertainty_device only */
int dsac_last_pass(dsac_engine* e, int32_t n_frames, int32_t* pipeline);

/* Pose modes of the preceding pass (INTEGRATION.md, "Pose modes"): per frame up to M = max_modes distinct refined poses of
 * its hypothesis pool, each with the pool's probability behind it, its covariance and its support; a frame's modes fit one
 * dsac_set_pose_priors_device setting.  After either pipeline's forward over n_frames (the pass dsac_last_pass names):
 *   1. occupied slots: img_idx[f][h][0] >= 0, or a prior slot of a pass with priors whose frame lacks DSAC_ST_BAD_PRIOR;
 *   2. they are ranked by scores (the hook's, with a score hook) descending, ties to the lower slot, NaN after every score;
 *   3. walking the ranking, a slot near a seed joins the first such seed in seed order, else becomes a new seed while fewer
 *      than M exist, else joins nothing.  Two poses are near iff theta <= rot_rad and |t_a - t_b| <= trans_mm, theta the
 *      angle of R_a R_b^T (atan2 of its skew part's norm and (tr - 1) / 2, fp64).  A seed's mass is the sum of its
 *      members' sf in rank order, members their number;
 *   4. each seed is refined from its own hypothesis pose as dsac_forward_dsac refines that slot (pose, steps_done), and has
 *      the covariance of dsac_pose_uncertainty_device's entry for that DSAC-variant job (cov_xi .. ok);
 *   5. in seed order, a seed whose refined pose is near the refined pose of an earlier surviving seed adds its mass and
 *      members to the first such one and is dropped.  The survivors are entries 0 .. n_modes - 1 in seed order; every
 *      later entry has hyp -1 and zeros.
 * Stream ordering, input lifetime and "changes no later result" as in dsac_pose_uncertainty_device; the pass's outputs are
 * untouched.  DSAC_ERR_ARG, with the engine left as it was: not after a forward over the same n_frames, a submitted pass
 * that has not been awaited, cameras, cell depth or priors changed since the pass, a pass that skipped the sample or
 * score stage (dsac_set_stages), max_modes outside [1, min(n_hyps, DSAC_MAX_MODES)], rot_rad or trans_mm not finite or
 * negative, or d_out NULL.  The outputs are not differentiated. */
#define DSAC_MAX_MODES 16          /* = DSAC_MAX_PRIORS: a frame's modes fit one priors setting */
typedef struct dsac_pose_modes_out {   /* DEVICE pointers, each nullable; M = max_modes */
    int32_t* n_modes;     /* [n]           modes found, 0 .. M */
    int32_t* hyp;         /* [n][M]        hypothesis slot of the mode's seed, -1 unused */
    double*  pose;        /* [n][M][6]     refined cv pose (rvec, tvec mm), as hyp_pose / ref_pose */
    double*  score;       /* [n][M]        the seed's score (before softmax) */
    double*  mass;        /* [n][M]        sum of sf over the mode's members */
    int32_t* members;     /* [n][M]        hypotheses in the mode */
    int32_t* steps_done;  /* [n][M] */
    double*  cov_xi;      /* [n][M][6][6]  as dsac_pose_uncertainty_out.cov_xi */
    double*  sigma2;      /* [n][M] */
    int32_t* n_fit;       /* [n][M] */
    int32_t* support;     /* [n][M] */
    int32_t* ok;          /* [n][M] */
} dsac_pose_modes_out;
int dsac_pose_modes_device(dsac_engine* e, int32_t n_frames, int32_t max_modes, double rot_rad, double trans_mm,
                           const dsac_pose_modes_out* d_out, void* stream);

/* Multi-camera rigs (INTEGRATION.md, "Multi-camera rigs"): one pose per rig from several cameras with known extrinsics.
 * The n_frames frames are R = n_frames / C rigs of C = n_cameras cameras; frame f = r*C + c is camera c of rig r, with the
 * camera of frame f (dsac_set_cameras) and the extrinsic d_cam_from_rig[f] [n][6], a cv pose (rvec, tvec mm):
 * X_cam = R_c X_rig + t_c.  H = n_hyps.
 *   sample: every frame as dsac_forward_device samples it (hyp_pose, img_idx, cand_idx and n_candidates bit-identical);
 *   lift:   camera c's hypothesis h becomes the rig pose R_r = R_c^T R_h, t_r = R_c^T (t_h - t_c), slot j = c*H + h of the
 *           rig's pool of C*H (an extrinsic whose rvec is exactly zero keeps the hypothesis' rvec);
 *   score:  score[r][j] = sum over c' = 0 .. C-1, in order, in fp64, of k_score's soft-inlier score of camera c' for the
 *           pose T_c' o T_r (so at the same alpha the softmax is about C times sharper than one camera's); softmax,
 *           entropy and soft-argmax over the pool as dsac_forward_device;
 *   refine: from the soft-argmax pose, ref_steps steps: per camera in order its first <= inlier_count cells of the step's
 *           permutation with reprojection error < thr2d under its composed pose, concatenated (fewer than 50 in all stop,
 *           DSAC_ST_REFINE_ABORTED), then CvLevMarq's fit of the rig's 6 parameters over their reprojections;
 *   eval:   with d_gt_rig_jp [R][12] (jp of the rig frame) and DSAC_STAGE_EVAL, loss, rot_err, t_err, correct per rig.
 * status[r]: the OR of its frames' sampler bits, DSAC_ST_REFINE_ABORTED, and DSAC_ST_BAD_RIG when one of its extrinsics is
 * not finite (all of that rig's outputs but hyp_pose are then zero).  C = 1 with zero extrinsics gives dsac_forward_device's
 * results bit for bit.  Ordered on `stream`; the engine's pass becomes DSAC_PASS_RIG, which the ordinary backward passes,
 * dsac_refined_jp6_device, dsac_pose_uncertainty_device and dsac_pose_modes_device refuse; the rig backward below and
 * dsac_rig_refined_jp6_device read it, and the sampling log-probability stays valid.  DSAC_ERR_ARG, with the engine left
 * as it was: n_frames % C != 0, C outside [1, DSAC_MAX_RIG_CAMERAS], C * n_hyps > DSAC_MAX_HYPS, a score hook, cell depth
 * or pose priors set, a stage mask without sample, score or refine, a submitted pass that has not been awaited, or a NULL
 * input or d_out. */
#define DSAC_MAX_RIG_CAMERAS 8
typedef struct dsac_rig_out {   /* DEVICE pointers, each nullable; R = n_frames / C, P = C * n_hyps */
    double*   hyp_pose;    /* [n][H][6]  the frames' sampled hypotheses */
    double*   rig_hyp;     /* [R][P][6]  the pool: rig poses (cv) */
    double*   scores;      /* [R][P] */
    double*   sf;          /* [R][P]     softmax */
    double*   entropy;     /* [R] */
    double*   avg_pose;    /* [R][6]     soft-argmax rig pose */
    double*   ref_pose;    /* [R][6]     refined rig pose */
    int32_t*  inlier_map;  /* [n][1600]  per camera frame */
    int32_t*  steps_done;  /* [R] */
    uint32_t* status;      /* [R]        DSAC_ST_* */
    double*   loss;        /* [R] */
    double*   rot_err;     /* [R] */
    double*   t_err;       /* [R] */
    int32_t*  correct;     /* [R] */
} dsac_rig_out;
int dsac_forward_rig_device(dsac_engine* e, int32_t n_frames, int32_t n_cameras, int64_t frame0, const int16_t* d_coords,
                            const int32_t* d_pix, int32_t pix_shared, const double* d_cam_from_rig, const double* d_gt_rig_jp,
                            const dsac_rig_out* d_out, void* stream);

/* Rig gradients (INTEGRATION.md, "Rig gradients"): the backward of the preceding dsac_forward_rig_device over the same
 * n_frames, whose inputs (coords, pix, extrinsics, gt) must still be valid.  The soft-argmax backward's chain in implicit
 * mode (dsac_set_coord_derivatives does not apply: a rig is always differentiated by the implicit function theorem), with
 * every per-hypothesis quantity lifted to the rig's pool of P = C * n_hyps: dRefineHyp by 12 replays of the rig
 * refinement, the direct term by the IFT of its last accepted step over every camera's cells, the support term of each
 * pool slot through the lift's Jacobian and the frame's dPNP, and the score term of every camera frame against its rig's
 * pool (its support part crossing to the camera whose hypothesis the slot lifts).  Quirks Q3, Q4 (fix_q4), Q7, Q10 and
 * Q12 as in dsac_backward_device.  A rig with DSAC_ST_BAD_RIG gets zero rows for all its frames.
 * All pointers are DEVICE pointers, ordered on `stream` after the pass by an event; nothing is synchronised.
 *   dsac_backward_rig_device: dLossMax of the refined rig pose against the pass's d_gt_rig_jp, times d_loss_grad [R]
 *     (NULL = 1 per rig); the pass must have had d_gt_rig_jp and DSAC_STAGE_EVAL.
 *   dsac_backward_rig_pose_device: seeded by d_grad_ref [R][6] = dOuter / d(refined rig jp6) (dsac_rig_refined_jp6_device).
 *   d_dloss_dobj [n][N][3] and d_dloss_dpred [n][N][3], clamp: as dsac_backward_device, per camera frame; NULL = not written.
 *   d_diag (nullable, each field nullable) as dsac_backward_out, per rig.
 * The calls have their own scratch: they change no output of the pass and no result of a later call.  DSAC_ERR_ARG, with the
 * engine left as it was: not after a dsac_forward_rig_device over the same n_frames, cameras, cell depth or pose priors
 * changed since the pass, a submitted pass that has not been awaited, the loss form after a pass without ground truth or
 * without DSAC_STAGE_EVAL, or a NULL d_grad_ref. */
typedef struct dsac_rig_backward_out {   /* DEVICE pointers, each nullable; R = n_frames / C, P = C * n_hyps */
    double* dloss_dref;       /* [R][6]   dLossMax of the refined rig pose, or the seed */
    double* dref_dhyp;        /* [R][36]  d refined jp6 / d soft-argmax rig pose (cv) */
    double* score_grads;      /* [R][P]   score output gradients over the pool */
    double* dref_dobj;        /* [R][6][C*N*3] d refined jp6 / d scene coordinates, camera c's columns at c*N*3 */
} dsac_rig_backward_out;
int dsac_backward_rig_device(dsac_engine* e, int32_t n_frames, const double* d_loss_grad, double* d_dloss_dobj,
                             float* d_dloss_dpred, float clamp, const dsac_rig_backward_out* d_diag, void* stream);
int dsac_backward_rig_pose_device(dsac_engine* e, int32_t n_frames, const double* d_grad_ref, double* d_dloss_dobj,
                                  float* d_dloss_dpred, float clamp, const dsac_rig_backward_out* d_diag, void* stream);
/* jp 6-vectors [R][6] of the refined rig poses of the preceding dsac_forward_rig_device over n_frames (refusals as the rig
 * backward's, and a NULL d_jp6). */
int dsac_rig_refined_jp6_device(dsac_engine* e, int32_t n_frames, double* d_jp6, void* stream);

/* Rig tracking (INTEGRATION.md, "Rig tracking"): the covariance of each refined rig pose, and rig pose priors, so that a rig
 * runs the tracker loop of "Pose priors".
 *
 * dsac_rig_pose_uncertainty_device: "Pose uncertainty" lifted to the rig, one job per rig (jobs = R = n_frames / C) after a
 * dsac_forward_rig_device over the same n_frames and n_cameras = C.  S is the set of cells, over all the rig's cameras, that
 * the rig refinement's last accepted step fitted (a recording replay from the soft-argmax rig pose), m = |S|; r_i the
 * reprojection residual of cell i in its own camera at the composed pose T_c o T_rig with its frame's camera (px); J_i =
 * dr_i/dxi in the rig chart R = exp([w]x) R*, t = t* + tau.  cov_xi = sigma2 (sum_S J_i^T J_i)^-1, sigma2 = sum_S |r_i|^2 /
 * (2m - 6), cov_jp6 = M cov_xi M^T at the rig pose (the jp 6-vector of dsac_rig_refined_jp6_device); support counts the
 * cells of all C cameras (at most 1600 C) whose error in k_score's fp32 arithmetic at the composed pose is below thr2d; n_fit
 * = m; ok as in dsac_pose_uncertainty_device.  A rig with DSAC_ST_BAD_RIG or DSAC_ST_BAD_PRIOR gets zeros in every output,
 * ok, n_fit and support included.  C = 1 with a zero extrinsic gives dsac_pose_uncertainty_device's outputs after the
 * ordinary pass bit for bit.  Ordered after the pass by an event, own scratch: it changes no later result.  DSAC_ERR_ARG,
 * with the engine left as it was: not after a dsac_forward_rig_device over n_frames, n_cameras not the pass's C, cameras,
 * cell depth, pose priors or rig pose priors changed since the pass, a submitted pass that has not been awaited, or d_out
 * NULL.  The outputs are not differentiated. */
int dsac_rig_pose_uncertainty_device(dsac_engine* e, int32_t n_frames, int32_t n_cameras, const dsac_pose_uncertainty_out* d_out,
                                     void* stream);
/* dsac_rig_pose_modes_device (INTEGRATION.md, "Rig pose modes"): dsac_pose_modes_device lifted to each rig's pool of
 * P = C * n_hyps slots after a dsac_forward_rig_device over the same n_frames and n_cameras = C.  Every field of d_out is
 * per rig: n_modes [R], the others [R][M](...), R = n_frames / C, M = max_modes.
 *   1. slot j = c*H + h of rig r is occupied when frame r*C + c sampled hypothesis h (img_idx[f][h][0] >= 0), or when the
 *      pass had rig pose priors (k of them) and h >= H - k; a rig with DSAC_ST_BAD_RIG or DSAC_ST_BAD_PRIOR has none and
 *      gets n_modes 0;
 *   2. the slots are ranked by the rig's scores (dsac_rig_out.scores: the hooks' with rig score hooks), descending, ties
 *      to the lower slot, NaN after every score;
 *   3. the walk, the nearness and the mass of dsac_pose_modes_device over the rig poses rig_hyp (rig frame) and the
 *      pool's sf; hyp is the pool slot j of the seed (the index into rig_hyp, scores and sf), -1 unused;
 *   4. each seed is refined from its rig pose as the rig pass refines its soft-argmax rig pose (pose, steps_done), over all
 *      C cameras' cells (with rig cell depth, the Kabsch refinement of RGB-D rigs), and has the covariance that
 *      dsac_rig_pose_uncertainty_device computes for a rig pose refined from there (cov_xi .. ok);
 *   5. the merge of dsac_pose_modes_device.
 * C = 1 with a zero extrinsic gives dsac_pose_modes_device's outputs after the ordinary pass bit for bit.  The score hooks
 * are not read: the call keeps working after they change.  Ordered after the pass by an event, own scratch: it changes no
 * output of the pass and no later result.  DSAC_ERR_ARG, with the engine left as it was: not after a
 * dsac_forward_rig_device over n_frames, n_cameras not the pass's C, cameras, cell depth, pose priors, rig pose priors or rig
 * cell depth changed since the pass, a submitted pass that has not been awaited, max_modes outside
 * [1, min(n_hyps, DSAC_MAX_MODES)] (a rig's modes fit one rig pose priors setting), rot_rad or trans_mm not finite or
 * negative, or d_out NULL.  The outputs are not differentiated. */
int dsac_rig_pose_modes_device(dsac_engine* e, int32_t n_frames, int32_t n_cameras, int32_t max_modes, double rot_rad,
                               double trans_mm, const dsac_pose_modes_out* d_out, void* stream);
/* dsac_set_rig_pose_priors_device: k rig poses per rig join the pools of the following dsac_forward_rig_device passes over
 * n_frames frames of n_cameras = C cameras.  d_poses: DEVICE float64 [R][k][6] cv rig poses (X_cam = R_c (R_j Y + t_j) +
 * t_c); d_info: DEVICE float64 [R][k][6][6] information matrices in the rig chart R = exp([w]x) R_j, t = t_j + tau
 * (inv(cov_xi + Q) of dsac_rig_pose_uncertainty_device is one), or NULL; gate a chi^2 bound, finite and > 0 with d_info.
 * At each rig pass, with the pass's extrinsic (R_c, t_c) of frame f = r C + c, prior j of rig r becomes frame f's prior
 * T_c o T_j = (R_c R_j, R_c t_j + t_c) (an extrinsic whose rvec is exactly zero keeps the prior's rvec bits) with
 * information B Lambda_j B^T, B = blockdiag(R_c, R_c); frame f then samples exactly as dsac_forward_device samples it under
 * dsac_set_pose_priors_device with those priors (quotas stream_chunk(n_hyps - k, n_streams, s), the gate an ordinary
 * rejection, prior slot n_hyps - k + j of hyp_pose holding the composed pose).  Since xi_cam = B xi_rig for a camera
 * hypothesis lifted to the rig, the camera-frame gate equals the rig-frame gate of the lifted hypothesis up to rounding.
 * Camera c's prior slot lifts to pool slot c n_hyps + n_hyps - k + j, which holds rig prior j's own bits: the pool has C
 * copies of each prior.  A rig whose extrinsics are not all finite, or one of whose composed entries has a non-finite
 * value or a Lambda whose Cholesky has a pivot below 1e-12 of its diagonal entry, gets DSAC_ST_BAD_PRIOR in all its frames
 * (nothing sampled) and in its status, and is treated as a DSAC_ST_BAD_RIG rig: its outputs but hyp_pose are zero, its
 * backward rows are zero and its covariance is zeros; other rigs are unaffected.  Priors are constants of the rig backward.
 * Copied on `stream` into engine-owned buffers; sticky; d_poses == NULL (other arguments ignored) clears the setting.  A rig
 * pass over other n_frames or C refuses, and every other forward entry point (dsac_forward, _submit, _device,
 * dsac_forward_dsac, _device) refuses while the setting is on.  The rig backward, dsac_rig_refined_jp6_device,
 * dsac_rig_pose_uncertainty_device and dsac_sampling_log_prob*_device refuse a rig pass after which the setting changed.
 * DSAC_ERR_ARG, with the engine left as it was: n_frames outside [1, max_frames] or not a multiple of C, C outside
 * [1, DSAC_MAX_RIG_CAMERAS], k outside [1, min(n_hyps, DSAC_MAX_PRIORS)], a bad gate, or a submitted pass that has not been
 * awaited. */
int dsac_set_rig_pose_priors_device(dsac_engine* e, int32_t n_frames, int32_t n_cameras, int32_t k, const double* d_poses,
                                    const double* d_info, double gate, void* stream);
/* RGB-D rigs (INTEGRATION.md, "RGB-D rigs"): dsac_set_rig_cell_depth_device makes the following dsac_forward_rig_device
 * passes over n_frames frames of n_cameras = C cameras RGB-D passes.  d_depth: DEVICE float32 [n_frames][1600], the depth in
 * mm at each cell of camera frame f = r C + c, with the rules of dsac_set_cell_depth_device (a cell has depth iff its value
 * is finite and > 0).  Copied on `stream` into an engine-owned buffer of its own (sized once for max_frames), so neither
 * depth setting changes the other's values.  With it:
 *   sample: every camera frame samples exactly as an RGB-D dsac_forward_device samples it (Kabsch minimal sets,
 *           DSAC_ST_NO_DEPTH and no hypotheses for a frame with fewer than 4 cells with depth, rig pose priors composed as
 *           before); a NO_DEPTH frame's H zero hypotheses are lifted and scored as any other, and the rig status ORs in
 *           DSAC_ST_NO_DEPTH without spoiling the rig;
 *   score:  unchanged (reprojection);
 *   refine: per camera in order its first <= inlier_count cells of the step's permutation with reprojection error < thr2d
 *           under its composed pose AND depth in its own frame (fewer than 50 in all stop, DSAC_ST_REFINE_ABORTED), then the
 *           Kabsch fit of the rig pose from their scene coordinates to their rig-frame eye points R_c^T (e - t_c), the
 *           minimiser of sum |R_c (R Y + t) + t_c - e|^2 (e - t_c exactly for an extrinsic whose rotation is exactly I).
 * The rig backward differentiates it with the Kabsch refinement's replays, the IFT of the RGB-D residual for the direct
 * term and the Kabsch dPNP per frame (depth is not differentiated); dsac_rig_pose_uncertainty_device uses the 3-vector
 * residual in mm and sigma2 = sum |r|^2 / (3m - 6), the support still counting reprojection inliers.  C = 1 with a zero
 * extrinsic gives an RGB-D dsac_forward_device's results and its covariance bit for bit (the backward's direct term to
 * rounding).  Sticky; d_depth == NULL (other arguments ignored)
 * clears it.  A rig pass over other n_frames or C refuses; while per-frame cell depth (dsac_set_cell_depth_device) is set
 * the rig pass still refuses.  Every other forward entry point refuses while the setting is on.  The rig backward,
 * dsac_rig_refined_jp6_device, dsac_rig_pose_uncertainty_device and dsac_sampling_log_prob*_device refuse a rig pass after
 * which the setting changed.  DSAC_ERR_ARG, with the engine left as it was: n_frames outside [1, max_frames] or not a
 * multiple of C, C outside [1, DSAC_MAX_RIG_CAMERAS], or a submitted pass that has not been awaited. */
int dsac_set_rig_cell_depth_device(dsac_engine* e, int32_t n_frames, int32_t n_cameras, const float* d_depth, void* stream);
/* Rig score hooks (INTEGRATION.md, "Rig score hooks"): the score seam for the rig passes.  With fwd and bwd registered, each
 * dsac_forward_rig_device over n frames of C cameras, P = C * n_hyps:
 *   score:  k_score_rig also writes the error image of camera frame f = r C + c against slot j of its rig's pool at the
 *           composed pose T_c o T_j, diffmaps [n][P][N] float (k_score's arithmetic, clamped at 100; in an engine-owned
 *           buffer, so write_diffmaps is not needed), then calls fwd(diffmaps, n, P, cam_scores, stream, user), which
 *           overwrites the camera scores [n][P] double; the rig score of slot j is still their fp64 sum in camera order,
 *           followed by the softmax, entropy and soft-argmax over the pool.  A nonzero return gives DSAC_ERR_ARG and the
 *           engine then holds no pass.
 *   backward: dsac_backward_rig_device and dsac_backward_rig_pose_device clamp the rig's score output gradients [R][P] to
 *           +-grad_clamp, give them to each of its camera frames (d rig score / d camera score = 1) and call
 *           bwd(diffmaps, score_grads [n][P], n, P, diffmap_grads [n][P][N] double, stream, user); the score term then reads
 *           diffmap_grads in place of the closed-form soft-inlier derivative.  A nonzero return gives DSAC_ERR_ARG.  Both
 *           refuse a rig pass that called other hooks, or none, than those registered now.
 * dsac_rig_refined_jp6_device and dsac_rig_pose_uncertainty_device do not read the score and keep working after the hooks
 * change; the covariance's support stays the closed-form reprojection count.  fwd and bwd are set together; both NULL clears
 * them.  Sticky.  While they are registered every other forward entry point (dsac_forward, _submit, _device,
 * dsac_forward_dsac, _device) refuses, naming this setter; the per-frame score hook (dsac_set_score_hook) still makes the rig
 * pass refuse.  DSAC_ERR_ARG, with the engine left as it was: exactly one of fwd and bwd NULL, or a submitted pass that has
 * not been awaited. */
int dsac_set_rig_score_hooks(dsac_engine* e, dsac_score_hook fwd, dsac_score_backward_hook bwd, void* user);

/* Soft-argmax backward seeded by d_grad_ref [n][6] = dOuter/d(refined jp6) instead of dLossMax.
 * No ground truth needed. dloss_dobj / dloss_dpred / clamp as in dsac_backward_device; clamp applies to the total. */
int dsac_backward_pose_device(dsac_engine* e, int32_t n_frames, const double* d_grad_ref,
                              double* d_dloss_dobj, float* d_dloss_dpred, float clamp, void* stream);

/* DSAC-variant backward seeded by d_grad_ref [n][H][6] (path I, over hypotheses with sf > 1e-4 and a nonzero seed)
 * and d_grad_sf [n][H] (path II through the softmax Jacobian); either may be NULL. d_out as in dsac_backward_dsac_device. */
int dsac_backward_dsac_pose_device(dsac_engine* e, int32_t n_frames, const double* d_grad_ref, const double* d_grad_sf,
                                   const dsac_backward_dsac_out* d_out, float* d_dloss_dpred, float clamp, void* stream);

/* Upstream step on the device (SURVEY.md section 8f row N3), so that frames never leave HBM between the image and the
 * hypothesis engine.  All pointers are DEVICE pointers; `stream` is a cudaStream_t (NULL: default stream).
 * dsac_gather_patches_device replaces the patch assembly of getCoordImg (cnn_softam.h:221-256) fused with forward()'s
 * normalisation (lua/train_obj.lua:117-124, mean = 127) and pushMaps' layout (lua_calls.h:65-82):
 *   patches[f][cell][c][y][x] = frames[f][oy-21+y][ox-21+x][c] - mean,   (ox, oy) = pix[f or 0][cell]
 * frames: [n][height][width][3] uint8 BGR (jp::img_bgr_t); patches: [n][N][3][42][42] float.  A border cell (which
 * stochasticSubSample never produces) yields a zero patch and DSAC_ST_BORDER_PATCH in status[f] (nullable).
 * dsac_coords_from_prediction_device replaces "modeImg(y,x) = prediction[i] * 1000" (cnn_softam.h:262-268):
 * prediction [n][N][3] float metres -> coords [n][N][3] int16 mm with cv::saturate_cast<short>. */
int dsac_gather_patches_device(dsac_engine* e, int32_t n_frames, const uint8_t* d_frames, int32_t width, int32_t height,
                               const int32_t* d_pix, int32_t pix_shared, float mean, float* d_patches, uint32_t* d_status,
                               void* stream);
int dsac_coords_from_prediction_device(dsac_engine* e, int32_t n_frames, const float* d_prediction, int16_t* d_coords,
                                       void* stream);

/* Batched Kabsch (Hypothesis::calcRigidBodyTransform, Hypothesis.cpp:145-200):
 * for each of n problems with m correspondences, b ~ R a + t.  a,b: [n][m][3] doubles. */
int dsac_kabsch(dsac_engine* e, int32_t n, int32_t m, const double* a, const double* b, double* R /* [n][9] */,
                double* t /* [n][3] */);

/* Host-side helpers that carry the reference's RNG contract (libstdc++ <random>). */
/* stochasticSubSample (cnn_softam.h:283-309) with ThreadRand thread-0 semantics
 * (thread_rand.cpp:40-81): mt19937(seed), 3200 uniform_real draws. */
int dsac_stochastic_subsample(uint32_t seed, int32_t width, int32_t height, int32_t* pix /* [N][2] */);
/* Synthetic frames of SURVEY.md section 8(d): GT pose, 40x40 int16 scene coordinates with inlier
 * ratio rho, inlier noise sigma (mm); sampling grid of frame g from mt19937(seed + g*n_streams).
 * traj != 0: smooth 7Scenes-like camera trajectory instead of i.i.d. poses. */
int dsac_synth_frames(uint32_t data_seed, uint32_t sampler_seed, int32_t n_streams, int64_t frame0, int32_t n_frames,
                      double rho, double sigma, int32_t traj, double focal, double cx, double cy, int16_t* coords,
                      int32_t* pix, double* gt_cv /* [n][6] */, double* gt_jp /* [n][12] */);

/* Pre-training of the coordinate CNN (train_obj.cpp): the data path on the device.  All pointers are DEVICE pointers
 * except the camera; `stream` is a cudaStream_t (NULL: default stream).
 *
 * The RGB-D camera of jp::Dataset (properties.h dP): the RGB camera (focal, x_shift, y_shift; the principal point is
 * width / 2.f + x_shift in float, so the shifts are kept apart from a cx), the depth camera (secondary_focal,
 * raw_x_shift, raw_y_shift), sensor_trans (row-major 4x4, depth -> RGB, the file sensorTrans.dat), raw_data (1:
 * depth is registered to the RGB camera, dataset.h:180-202) and the frame size. */
typedef struct dsac_rgbd_camera {
    float focal, x_shift, y_shift;
    float secondary_focal, raw_x_shift, raw_y_shift;
    double sensor_trans[16];
    int32_t raw_data, width, height;
} dsac_rgbd_camera;
/* The reference's defaults, which the shipped 7-Scenes default.config repeats: focal 525, secondary focal 585, no shifts,
 * raw_data 1, 640 x 480; sensor_trans identity (the reference's value when sensorTrans.dat is absent). */
int dsac_default_rgbd_camera(dsac_rgbd_camera* cam);
/* Per-frame cameras of a dataset (frames with their own intrinsics: SfM reconstructions, several sensors), indexed by
 * DATASET frame -- unlike dsac_set_cameras' table, which is indexed by the frame of a forward pass; the two are separate.
 * cams: HOST array [n_frames], one RGB-D camera per dataset frame; NULL clears the table (n_frames ignored).  Validated
 * here: n_frames >= 1; focal finite and > 0; secondary_focal finite and > 0 where raw_data is set; the shifts and
 * sensor_trans finite; width, height and raw_data the same in every entry (the dataset arrays are [F][H][W]).  On failure
 * DSAC_ERR_ARG, dsac_last_error names the index, and the table in force stays as it was.  The table is staged in
 * page-locked memory and copied to an engine-owned device buffer on `stream` (a cudaStream_t, NULL = default), after the
 * last call that read the previous table; the calls that read it wait for the copy on whichever stream they run.
 * With a table set:
 *   - dsac_register_depth_device, dsac_obj_coords_device and dsac_obj_draw_device take cam == NULL to mean the table;
 *     their n / n_frames must then equal its size (else DSAC_ERR_ARG, as for cam == NULL without a table);
 *   - dsac_score_maps_device projects image i with the camera of frame img[i] (see there). */
int dsac_set_dataset_cameras(dsac_engine* e, int32_t n_frames, const dsac_rgbd_camera* cams, void* stream);
/* getDepth for n frames: raw [n][H][W] uint16 -> depth [n][H][W] uint16 (raw_data 0: a copy).  cam == NULL: frame f
 * is registered with dataset camera f (dsac_set_dataset_cameras; n must equal the table's size).  Where several depth
 * pixels land on one RGB pixel the last in the reference's order (x outer, y inner) wins.  Targets outside the image are
 * dropped; dropped [n] (nullable) counts them and status [n] (nullable; needs dropped) gets DSAC_ST_DEPTH_DROPPED.
 * With raw_data the scatter uses a per-pixel buffer the engine owns and grows on demand (growing frees the old one,
 * which waits for the device): registrations on one engine must be issued on one stream at a time, as its forward
 * passes are; use one engine per concurrent stream. */
int dsac_register_depth_device(dsac_engine* e, const dsac_rgbd_camera* cam, int32_t n_frames, const uint16_t* d_raw,
                               uint16_t* d_depth, int32_t* d_dropped, uint32_t* d_status, void* stream);
/* getObj: registered depth [n_frames][H][W] and jp poses [n_frames][12] (dsac_forward's gt_jp: row-major rotation,
 * translation in mm; taken through float as jp::info_t holds it) -> int16 scene coordinates [n][H][W][3] in mm of
 * frames idx[0..n) (idx NULL: frames 0..n, n <= n_frames).  A listed index outside [0, n_frames) gives a zero image.
 * cam == NULL: frame idx[k] uses dataset camera idx[k] (n_frames must equal the table's size). */
int dsac_obj_coords_device(dsac_engine* e, const dsac_rgbd_camera* cam, int32_t n_frames, int32_t n, const int32_t* d_idx,
                           const uint16_t* d_depth, const double* d_poses, int16_t* d_coords, void* stream);
/* ThreadRand::init(seed) for n_streams threads: state [n_streams][625] = std::mt19937(seed + t) words and position. */
int dsac_obj_rng_init_device(dsac_engine* e, uint32_t seed, int32_t n_streams, uint32_t* d_state, void* stream);
/* assembleData's draw (train_obj.cpp:47-102) over n_streams OpenMP threads: image i (of n_images, static schedule) draws
 * its frame from [0, n_frames), then n_patches centres (x, y) whose getObj label is nonzero.  Writes img [n_images *
 * n_patches], centre [..][2], label [..][3] (metres, Vec3f /= 1000) and status [n_images].  state is read and advanced,
 * so consecutive calls continue like the reference's rounds.  A patch not found within max_attempts (>= 32) pairs ends
 * its image: the remaining centres are (-1, -1) and status gets DSAC_ST_OBJ_DRAW_EXHAUSTED.  The frame must exceed 42 px
 * in both dimensions.  cam == NULL: an image's labels use the dataset camera of the frame it drew (n_frames must equal
 * the table's size); the random words consumed are the same. */
int dsac_obj_draw_device(dsac_engine* e, const dsac_rgbd_camera* cam, int32_t n_frames, const uint16_t* d_depth,
                         const double* d_poses, int32_t n_images, int32_t n_patches, int32_t n_streams,
                         int32_t max_attempts, uint32_t* d_state, int32_t* d_img, int32_t* d_centre, float* d_label,
                         uint32_t* d_status, void* stream);
/* dsac_gather_patches_device at listed centres: patch k = frames[frame[k]] around centre[k] = (x, y), minus mean,
 * [n][3][42][42].  A centre whose patch leaves the frame, or a frame index outside [0, n_frames), yields a zero patch and
 * DSAC_ST_BORDER_PATCH in status[0] (nullable). */
int dsac_gather_patches_at_device(dsac_engine* e, int32_t n, const uint8_t* d_frames, int32_t n_frames, int32_t width,
                                  int32_t height, const int32_t* d_frame, const int32_t* d_centre, float mean,
                                  float* d_patches, uint32_t* d_status, void* stream);
/* train_obj.cpp:266-270: out = std::shuffle(iota(n), std::mt19937(seed)); the reference uses seed 5489 (default). */
int dsac_shuffle_permutation(int32_t n, uint32_t seed, int32_t* out);

/* Pre-training of the score CNN (train_score.cpp): the data path on the device.  Pointers are DEVICE pointers;
 * `stream` is a cudaStream_t (NULL: default stream).
 *
 * assembleData's draw over n_streams OpenMP threads on ThreadRand state [n_streams][625] (dsac_obj_rng_init_device),
 * read and advanced so that consecutive calls continue like the reference's rounds.  Per image i: stream 0 draws the
 * frame img[i] from [0, n_frames) and the sampling grid pix [i][1600][2] of a width x height frame (stochasticSubSample,
 * cell y * 40 + x); then hypothesis h (static schedule over the streams) draws drift [i * hyps + h] (0: small, 1: large
 * pose error) and getRandHyp's 6-vector noise [i * hyps + h][6] (rotation vector in radians, translation in mm).  The
 * frame must be at least 83 px in both dimensions, where stochasticSubSample's loop runs exactly 40 times per axis
 * (below that the reference writes past its sampling grid). */
int dsac_score_draw_device(dsac_engine* e, int32_t n_frames, int32_t width, int32_t height, int32_t n_images,
                           int32_t hyps_per_image, int32_t n_streams, uint32_t* d_state, int32_t* d_img, int32_t* d_pix,
                           int32_t* d_drift, double* d_noise, void* stream);
/* The training samples of a draw: pose k = i * hyps + h is poseGT(gt_jp[img[i]]) * Hypothesis(noise[k]); maps [k][1600]
 * is its reprojection-error image against coords [i][1600][3] (mm, the coordinate CNN's grid at pix [i]) with the
 * engine's camera (config focal / cx / cy), clamped at 100 and computed like the forward's diffmaps; labels [k] =
 * -temperature * max(angular error in degrees, translation error in mm / 10); correct [k] (nullable) = 1 where the
 * errors are below 5 degrees and 50 mm.  img must index gt_jp (as dsac_score_draw_device writes it).
 * With a dataset camera table set (dsac_set_dataset_cameras), image i uses the camera of frame img[i] as train_score.cpp
 * takes it from getCamMat(): focal, cx = float(width / 2 + x_shift) with the INTEGER width / 2, cy likewise (not
 * getObj's width / 2.f; DESIGN.md quirk Q27).  An img[i] outside the table is not read: its maps and labels are NaN and
 * correct 0. */
int dsac_score_maps_device(dsac_engine* e, int32_t n_images, int32_t hyps_per_image, const int32_t* d_img,
                           const double* d_gt_jp, const int16_t* d_coords, const int32_t* d_pix, const double* d_noise,
                           float temperature, float* d_maps, double* d_labels, int32_t* d_correct, void* stream);
/* train_score.cpp:286,381-384: out [n_rounds][n] = the permutations of rounds first_round .. of one continuing
 * std::mt19937(seed), each round std::shuffle of a fresh iota(n); the reference uses seed 5489 (default). */
int dsac_shuffle_permutations(int32_t n, uint32_t seed, int32_t first_round, int32_t n_rounds, int32_t* out);

const char* dsac_version(void);

#ifdef __cplusplus
}
#endif
#endif
