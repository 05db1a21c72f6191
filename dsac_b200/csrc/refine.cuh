// refine.cuh -- K4: batched refinement of pose hypotheses (one CTA per job).
//
// Restates the refinement loop of processImage (cnn_softam.h:1099-1154) and its replay
// refine() (cnn_softam.h:663-723): per step walk a fixed permutation of the 1600 cells,
// take the first <= inlierCount cells whose reprojection error is below the threshold, stop
// if fewer than 50, run cv::solvePnP(CV_ITERATIVE, useExtrinsicGuess) -- Levenberg-Marquardt
// on the 6 pose parameters with CvLevMarq's schedule -- and recompute the error map.
//
// A "job" is (frame, initial cv pose, optional +-delta on one int16 scene coordinate), so
// the same kernel serves the forward pass (1 job per frame) and the central differences of
// dRefineHyp / dRefineObj (cnn_softam.h:738-923; 12 + 6*k jobs per frame).
//
// The pose arithmetic is fp64 (the reference runs this in double).  The error maps are only ever compared with
// the inlier threshold, so they are kept as bit maps, decided in fp32 with a rigorous error bound and in the
// reference's exact arithmetic where the bound does not separate the error from the threshold.
#pragma once
#include <cuda_runtime.h>

#include "camera.cuh"
#include "lm_math.cuh"
#include "pose_math.cuh"
#include "rigid.cuh"

namespace dsac {

#ifndef K4_THREADS_DEF
#define K4_THREADS_DEF 64
#endif
#ifndef K4_MIN_BLOCKS
#define K4_MIN_BLOCKS 8
#endif
constexpr int K4_THREADS = K4_THREADS_DEF;   // 2 warps per job: the work per job is small and mostly sequential
constexpr int K4_WARPS = K4_THREADS / 32;
constexpr int K4_MAX_INLIERS = 128;
constexpr int RIG_MAX_CAMERAS = 8;            // DSAC_MAX_RIG_CAMERAS
constexpr uint32_t RIG_ST_BAD = 256u;          // DSAC_ST_BAD_RIG
// a rig whose outputs are zero: a non-finite extrinsic, or a bad rig prior (DSAC_ST_BAD_RIG | DSAC_ST_BAD_PRIOR)
constexpr uint32_t RIG_ST_SPOILED = RIG_ST_BAD | 128u;
static_assert(K4_THREADS % 32 == 0 && K4_THREADS >= 32 && K4_THREADS <= 256, "k_refine block size");

struct RefineParams {
    const int16_t* coords;      // [n][N][3]
    const int32_t* pix;         // [n or 1][N][2]
    int pix_stride;
    const uint16_t* perm;       // [ref_steps][N]  (std::shuffle with default mt19937, cnn_softam.h:1104-1114)
    double f, cx, cy;
    const Cam* cams;            // [n_frames] or null: the camera of every frame is f, cx, cy
    int thr, inlier_count, ref_steps;
    // jobs
    int n_jobs;
    const int32_t* job_frame;   // [n_jobs] or null (job j -> frame j)
    const double* job_init;     // [n_jobs][6] cv pose
    const int32_t* job_pert;    // [n_jobs][2] {cell*3+chan or -1, delta} or null
    const int32_t* max_steps;   // [n_frames] replay limit (n_perm_steps of the forward) or null
    const int32_t* job_max_steps;   // [n_jobs] replay limit per job (DSAC variant: per hypothesis) or null
    // outputs
    double* out_pose;           // [n_jobs][6] refined cv pose
    double* out_jp6;            // [n_jobs][6] Hypothesis(cv2our(pose)).getRodVecAndTrans() or null
    int32_t* inlier_map;        // [n_jobs][N] or null
    int32_t* steps_done;        // [n_jobs] or null
    int32_t* n_perm_steps;      // [n_jobs] or null
    uint32_t* status;           // [n_frames] or null
    // evaluation (cnn_softam.h:1160-1179)
    const double* gt_jp;        // [n_frames][12] or null
    double* loss;
    double* rot_err;
    double* t_err;
    int32_t* correct;
};

// A multi-camera rig's refinement (k_refine_rig): job r refines rig r over the camera frames r C .. r C + C - 1.
struct RigRefine {
    int C;
    const double* ext;          // [n_frames][12] Rc (row-major) and tc of each camera frame (k_rig_lift)
};

__device__ __forceinline__ double dot3_plain(double a0, double b0, double a1, double b1, double a2, double b2, double c) {
    // left-to-right, no FMA contraction: matches the scalar double code of cv::projectPoints
    return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1)), __dmul_rn(a2, b2)), c);
}

// jp::cv2our, types.h:186-214
__device__ void cv2our_dev(const double pose[6], double R[9], double t[3]) {
    rodrigues_v2m(pose, R);
    t[0] = pose[3]; t[1] = -pose[4]; t[2] = -pose[5];
    for (int j = 0; j < 3; j++) {
        R[3 + j] = -R[3 + j];
        R[6 + j] = -R[6 + j];
    }
    double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) + R[2] * (R[3] * R[7] - R[4] * R[6]);
    if (det < 0) {
        for (int k = 0; k < 9; k++) R[k] = -R[k];
        for (int k = 0; k < 3; k++) t[k] = -t[k];
    }
    if (t[0] != t[0] || t[1] != t[1] || t[2] != t[2]) t[0] = t[1] = t[2] = 0;
}

// getInvHyp, maxloss.h:39-61
__device__ void inv_pose_dev(const double R[9], const double t[3], double Ri[9], double ti[3]) {
    double d = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) + R[2] * (R[3] * R[7] - R[4] * R[6]);
    double id = 1.0 / d;
    Ri[0] = (R[4] * R[8] - R[5] * R[7]) * id; Ri[1] = (R[2] * R[7] - R[1] * R[8]) * id; Ri[2] = (R[1] * R[5] - R[2] * R[4]) * id;
    Ri[3] = (R[5] * R[6] - R[3] * R[8]) * id; Ri[4] = (R[0] * R[8] - R[2] * R[6]) * id; Ri[5] = (R[2] * R[3] - R[0] * R[5]) * id;
    Ri[6] = (R[3] * R[7] - R[4] * R[6]) * id; Ri[7] = (R[1] * R[6] - R[0] * R[7]) * id; Ri[8] = (R[0] * R[4] - R[1] * R[3]) * id;
    ti[0] = -(Ri[0] * t[0] + Ri[1] * t[1] + Ri[2] * t[2]);
    ti[1] = -(Ri[3] * t[0] + Ri[4] * t[1] + Ri[5] * t[2]);
    ti[2] = -(Ri[6] * t[0] + Ri[7] * t[1] + Ri[8] * t[2]);
}

// maxLoss (maxloss.h:69-79) + the errors of cnn_softam.h:1166-1170
__device__ double max_loss_dev(const double R1[9], const double t1[3], const double R2[9], const double t2[3],
                               double* rot_err, double* t_err) {
    double Ri1[9], ti1[3], Ri2[9], ti2[3], Ri2inv[9], z[3] = {0, 0, 0}, zz[3];
    inv_pose_dev(R1, t1, Ri1, ti1);
    inv_pose_dev(R2, t2, Ri2, ti2);
    inv_pose_dev(Ri2, z, Ri2inv, zz);
    double tr = 0;
    for (int i = 0; i < 3; i++)
        for (int k = 0; k < 3; k++) tr += Ri1[i * 3 + k] * Ri2inv[k * 3 + i];
    tr = fmin(3.0, fmax(-1.0, tr));
    double re = 180 * acos((tr - 1.0) / 2.0) / kPi;
    double dx = ti1[0] - ti2[0], dy = ti1[1] - ti2[1], dz = ti1[2] - ti2[2];
    double te = sqrt(dx * dx + dy * dy + dz * dz);
    *rot_err = re;
    *t_err = te;
    return fmin(fmax(re, te / 10), 10000000.0);
}

// One CTA per job.  Structure of a refinement step:
//   flags    all threads: "error < threshold" per cell as a bit map -- fp32 with a rigorous error bound, the exact
//            reference arithmetic (reproj_error_exact) only for cells within the bound of the threshold;
//   select   warp 0 walks the step's permutation with ballots (no block barrier) and takes the first
//            inlier_count flagged cells in order;
//   LM       CvLevMarq's state machine with ONE pass over the selected points per trial parameter vector: the pass
//            accumulates the error norm AND the normal equations at the trial point (which the reference would
//            compute in its next CALC_J if the trial is accepted -- the same numbers); warp 0 reduces, decides,
//            solves the damped 6x6 system in registers and builds the next R / dR/dr across its lanes.  Two block
//            barriers per trial.
// RGBD (k_refine_rgbd): the selection takes the first inlier_count flagged cells that have depth (eye [n_frames][N][3], NaN
// without), and the pose update is the Kabsch fit of the selected cells, scene to eye (kabsch_fit), in place of LM.
// RECORD (the recording replay of dsac_set_coord_derivatives(DSAC_DERIV_IMPLICIT)): the cells the last accepted step fitted,
// in selection order, go to rec_sel [n_jobs][K4_MAX_INLIERS] and their number to rec_count [n_jobs] (0: no step accepted).
// RIG (k_refine_rig): the job is a rig of rig.C cameras, the pose the rig's.  The flags are those of every camera under its
// composed pose (rig_compose), the selection is each camera's first inlier_count flagged cells in turn (entries cam << 11 |
// cell), an LM point is reprojected in its own camera (lm_point_contrib_ext), and the inlier maps are the cameras' frames.
// The cells are read from global memory rather than staged: C frames do not fit in shared memory.  A rig with
// DSAC_ST_BAD_RIG or DSAC_ST_BAD_PRIOR in status gets zero outputs.  RIG with RECORD (k_refine_rig_rec, the rig backward) records those entries
// at a stride of C K4_MAX_INLIERS per rig.
// RIG with RGBD (k_refine_rig_rgbd, RGB-D rigs): eye holds every camera frame's eye points, each camera's selection takes
// the cells with depth in its own frame, and the Kabsch fit maps the scene coordinates to the rig-frame eye points
// Rc^T (e - tc) (rig_point), the exact minimiser of sum |Rc (R Y + t) + tc - e|^2.  Its C K4_MAX_INLIERS point pairs are
// staged in dynamic shared memory of rig_kabsch_smem(C) bytes.
template <bool PER_FRAME, bool RGBD = false, bool RECORD = false, bool RIG = false>
__device__ __forceinline__ void k_refine_body(const RefineParams& p, const double* eye = nullptr, uint16_t* rec_sel = nullptr,
                                              int32_t* rec_count = nullptr, RigRefine rig = RigRefine{}) {
    constexpr int NC = RIG ? RIG_MAX_CAMERAS : 1;   // camera frames per job, at most
    // the frame's scene coordinates (int16 mm, this job's perturbation applied) and pixel positions, staged once per job:
    // every refinement step reads all of them for the inlier flags and the selected ones in each LM pass
    __shared__ short s_cX[RIG ? 1 : DSAC_N_CONST], s_cY[RIG ? 1 : DSAC_N_CONST], s_cZ[RIG ? 1 : DSAC_N_CONST];
    __shared__ float s_fu[RIG ? 1 : DSAC_N_CONST], s_fv[RIG ? 1 : DSAC_N_CONST];
    __shared__ uint32_t s_bits[NC * DSAC_N_CONST / 32];
    __shared__ unsigned char s_imap[NC * DSAC_N_CONST];
    __shared__ unsigned short s_sel[NC * K4_MAX_INLIERS];
    __shared__ double s_R[9], s_J[27], s_param[6], s_prev[6], s_pose[6], s_Rd[RIG ? NC * 12 : 9];
    __shared__ float s_Pf[NC * 12];
    __shared__ double s_red[K4_WARPS][32];
    __shared__ double s_sum[2][32];
    __shared__ int s_count, s_ctl;
    __shared__ int s_rec_count;                               // (RECORD only)
    __shared__ unsigned short s_rec[RECORD ? NC * K4_MAX_INLIERS : 1];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int job = blockIdx.x;
    const int frame = p.job_frame ? p.job_frame[job] : job;   // (RIG: the rig)
    if (frame < 0) return;  // unused job slot
    const int n_cams = RIG ? rig.C : 1;
    if constexpr (RIG) {
        if (p.status[frame] & RIG_ST_SPOILED) {   // (uniform over the CTA)
            if (tid < 6) p.out_pose[(size_t)job * 6 + tid] = 0.0;
            if (p.inlier_map)
                for (int i = tid; i < n_cams * DSAC_N_CONST; i += K4_THREADS) p.inlier_map[(size_t)job * n_cams * DSAC_N_CONST + i] = 0;
            if (tid == 0) {
                if (p.steps_done) p.steps_done[job] = 0;
                if (p.n_perm_steps) p.n_perm_steps[job] = 0;
                if (p.gt_jp) { p.loss[job] = 0; p.rot_err[job] = 0; p.t_err[job] = 0; p.correct[job] = 0; }
                if constexpr (RECORD) rec_count[job] = 0;
            }
            return;
        }
    }
    const Cam cam = frame_cam<PER_FRAME>(p, frame);
    const int16_t* coords = p.coords + (size_t)frame * DSAC_N_CONST * 3;
    const int32_t* pix = p.pix + (size_t)frame * p.pix_stride;
    int pert_idx = -1, pert_delta = 0;
    if (p.job_pert) {
        pert_idx = p.job_pert[job * 2];
        pert_delta = p.job_pert[job * 2 + 1];
    }
    const int step_limit = p.job_max_steps ? min(p.ref_steps, p.job_max_steps[job])
                                           : (p.max_steps ? min(p.ref_steps, p.max_steps[frame]) : p.ref_steps);

    if (tid < 6) s_pose[tid] = p.job_init[(size_t)job * 6 + tid];
    if constexpr (RIG)
        for (int i = tid; i < n_cams * DSAC_N_CONST; i += K4_THREADS) s_imap[i] = 0;
    else
    for (int i = tid; i < DSAC_N_CONST; i += K4_THREADS) {
        s_imap[i] = 0;
        int v[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            v[k] = __ldg(coords + i * 3 + k);
            if (i * 3 + k == pert_idx) v[k] = (int)(short)(v[k] + pert_delta);  // short += float eps (cnn_softam.h:887)
        }
        s_cX[i] = (short)v[0]; s_cY[i] = (short)v[1]; s_cZ[i] = (short)v[2];
        s_fu[i] = (float)__ldg(pix + i * 2);
        s_fv[i] = (float)__ldg(pix + i * 2 + 1);
    }
    __syncthreads();

    const float thrf = (float)p.thr;
    const float cxf = (float)cam.cx, cyf = (float)cam.cy, c_abs = fabsf(cxf) + fabsf(cyf);

    // inlier flags of the current pose s_pose (getDiffMap, cnn_softam.h:319-362, reduced to "< threshold")
    auto inlier_flags = [&]() {
        if constexpr (RIG) {
            // every camera's composed pose (lane k < 12 stores element k: R row-major, then t) and its fp32 rows
            if (warp == 0) {
                double pose[6], R[9];
#pragma unroll
                for (int k = 0; k < 6; k++) pose[k] = s_pose[k];
                rodrigues_v2m(pose, R);
                for (int c = 0; c < n_cams; c++) {
                    const int fr = frame * n_cams + c;
                    const double* E = rig.ext + (size_t)fr * 12;
                    double Rk[9], tk[3];
                    rig_compose(E, E + 9, R, pose + 3, Rk, tk);
                    const double fc = frame_cam<PER_FRAME>(p, fr).f;
#pragma unroll
                    for (int k = 0; k < 12; k++) {
                        const int row = k >> 2, col = k & 3;
                        const double v = (col < 3) ? Rk[row * 3 + col] : tk[row];
                        if (lane == k) {
                            s_Rd[c * 12 + k] = k < 9 ? Rk[k] : tk[k - 9];
                            s_Pf[c * 12 + k] = (float)(row < 2 ? fc * v : v);
                        }
                    }
                }
            }
            __syncthreads();
            for (int base = 0; base < n_cams * DSAC_N_CONST; base += K4_THREADS) {
                const int ci = base + tid;
                bool flag = false;
                if (ci < n_cams * DSAC_N_CONST) {   // (a warp never straddles two cameras: 1600 = 50 x 32)
                    const int c = ci / DSAC_N_CONST, cell = ci - c * DSAC_N_CONST, fr = frame * n_cams + c;
                    const Cam cm = frame_cam<PER_FRAME>(p, fr);
                    const int16_t* co = p.coords + ((size_t)fr * DSAC_N_CONST + cell) * 3;
                    const int32_t* px = p.pix + (size_t)fr * p.pix_stride + cell * 2;
                    const float X = (float)__ldg(co), Y = (float)__ldg(co + 1), Z = (float)__ldg(co + 2);
                    const float fu = (float)__ldg(px), fv = (float)__ldg(px + 1);
                    const float ccx = (float)cm.cx, ccy = (float)cm.cy;
                    float P[12];
#pragma unroll
                    for (int k = 0; k < 12; k++) P[k] = s_Pf[c * 12 + k];
                    const int r = reproj_below_thr_fast(P, X, Y, Z, fu - ccx, fv - ccy, fabsf(ccx) + fabsf(ccy), thrf);
                    if (r >= 0) {
                        flag = (r != 0);
                    } else {
                        double Rd[9], t[3];
#pragma unroll
                        for (int k = 0; k < 9; k++) Rd[k] = s_Rd[c * 12 + k];
                        t[0] = s_Rd[c * 12 + 9]; t[1] = s_Rd[c * 12 + 10]; t[2] = s_Rd[c * 12 + 11];
                        flag = reproj_error_exact(Rd, t, (double)X, (double)Y, (double)Z, cm.f, cm.cx, cm.cy, fu, fv) < thrf;
                    }
                }
                const uint32_t m = __ballot_sync(0xffffffffu, flag);
                if (lane == 0 && base + warp * 32 < n_cams * DSAC_N_CONST) s_bits[(base >> 5) + warp] = m;
            }
            __syncthreads();
            return;
        }
        if (warp == 0) {
            double pose[6], R[9];
#pragma unroll
            for (int k = 0; k < 6; k++) pose[k] = s_pose[k];
            rodrigues_v2m(pose, R);   // (every lane computes the same R; lane k stores element k)
#pragma unroll
            for (int k = 0; k < 9; k++)
                if (lane == k) s_Rd[k] = R[k];
#pragma unroll
            for (int k = 0; k < 12; k++) {
                const int row = k >> 2, col = k & 3;
                const double v = (col < 3) ? R[row * 3 + col] : pose[3 + row];
                if (lane == k) s_Pf[k] = (float)(row < 2 ? cam.f * v : v);
            }
        }
        __syncthreads();
        float P[12];
#pragma unroll
        for (int k = 0; k < 12; k++) P[k] = s_Pf[k];
        for (int base = 0; base < DSAC_N_CONST; base += K4_THREADS) {
            const int c = base + tid;
            bool flag = false;
            if (c < DSAC_N_CONST) {
                const float X = (float)s_cX[c], Y = (float)s_cY[c], Z = (float)s_cZ[c];
                const float fu = s_fu[c], fv = s_fv[c];
                const int r = reproj_below_thr_fast(P, X, Y, Z, fu - cxf, fv - cyf, c_abs, thrf);
                if (r >= 0) {
                    flag = (r != 0);
                } else {
                    double Rd[9], t[3];
#pragma unroll
                    for (int k = 0; k < 9; k++) Rd[k] = s_Rd[k];
                    t[0] = s_pose[3]; t[1] = s_pose[4]; t[2] = s_pose[5];
                    flag = reproj_error_exact(Rd, t, (double)X, (double)Y, (double)Z, cam.f, cam.cx, cam.cy, fu, fv) < thrf;
                }
            }
            const uint32_t m = __ballot_sync(0xffffffffu, flag);
            if (lane == 0 && base + warp * 32 < DSAC_N_CONST) s_bits[(base >> 5) + warp] = m;
        }
        __syncthreads();
    };

    // this thread's selected points of the current refinement step (constant over its LM loop), loaded once
    constexpr int K4_PPT = (K4_MAX_INLIERS + K4_THREADS - 1) / K4_THREADS;
    float selX[K4_PPT], selY[K4_PPT], selZ[K4_PPT], selU[K4_PPT], selV[K4_PPT];
    auto load_selected = [&](int n) {
        if constexpr (!RIG) {   // (RIG: read from global memory in each pass)
#pragma unroll
            for (int k = 0; k < K4_PPT; k++) {
                const int i = tid + k * K4_THREADS;
                const int c = (i < n) ? s_sel[i] : 0;
                selX[k] = (float)s_cX[c]; selY[k] = (float)s_cY[c]; selZ[k] = (float)s_cZ[c];
                selU[k] = s_fu[c]; selV[k] = s_fv[c];
            }
        }
    };

    // per-thread contribution of the selected points to [0..20] upper triangle of JtJ, [21..26] JtErr, [27] |err|^2
    // at (s_param, s_R, s_J), reduced over the block into s_red[warp][0..31] (lane L holds sum L)
    auto normal_equations_pass = [&](int n) {
        double v[32];
#pragma unroll
        for (int k = 0; k < 32; k++) v[k] = 0;
        if constexpr (RIG) {   // (the points of each thread in the order of the loop below)
            for (int i = tid; i < n; i += K4_THREADS) {
                const int code = s_sel[i], c = code >> 11, cell = code & 2047, fr = frame * n_cams + c;
                const Cam cm = frame_cam<PER_FRAME>(p, fr);
                const int16_t* co = p.coords + ((size_t)fr * DSAC_N_CONST + cell) * 3;
                const int32_t* px = p.pix + (size_t)fr * p.pix_stride + cell * 2;
                const double* E = rig.ext + (size_t)fr * 12;
                lm_point_contrib_ext(s_R, s_J, s_param, E, E + 9, (double)__ldg(co), (double)__ldg(co + 1), (double)__ldg(co + 2),
                                     (double)(float)__ldg(px), (double)(float)__ldg(px + 1), cm.f, cm.cx, cm.cy, v);
            }
        } else {
#pragma unroll
            for (int k = 0; k < K4_PPT; k++)
                if (tid + k * K4_THREADS < n)
                    lm_point_contrib(s_R, s_J, s_param, (double)selX[k], (double)selY[k], (double)selZ[k], (double)selU[k], (double)selV[k],
                                     cam.f, cam.cx, cam.cy, v);
        }
        // transposed butterfly: after the step with offset `off` every lane keeps half of its values; lane L ends with sum L
#pragma unroll
        for (int half = 16, off = 16; half >= 1; half >>= 1, off >>= 1) {
            const bool up = (lane & off) != 0;
#pragma unroll
            for (int i = 0; i < 16; i++) {
                if (i < half) {
                    const double send = up ? v[i] : v[i + half];
                    const double keep = up ? v[i + half] : v[i];
                    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
                }
            }
        }
        s_red[warp][lane] = v[0];
    };

    inlier_flags();

    if constexpr (RECORD) {
        if (tid == 0) s_rec_count = 0;
    }
    int steps_done = 0, n_perm = 0;
    for (int rStep = 0; rStep < step_limit; rStep++) {
        n_perm++;
        // ---- ordered selection of the first inlier_count flagged cells of the step's permutation (cnn_softam.h:1117-1134)
        // (RIG: every camera in turn, its cells appended to the previous cameras')
        if (warp == 0) {
            const uint16_t* perm = p.perm + (size_t)rStep * DSAC_N_CONST;
            int total = 0;
            for (int cc = 0; cc < n_cams; cc++) {
                const uint32_t* bits = s_bits + cc * (DSAC_N_CONST / 32);
                unsigned char* imap = s_imap + cc * DSAC_N_CONST;
                unsigned short* sel = s_sel + total;
                int count = 0;
                for (int k0 = 0; k0 < DSAC_N_CONST && count < p.inlier_count; k0 += 32) {
                    const int c = __ldg(perm + k0 + lane);
                    bool flag = (bits[c >> 5] >> (c & 31)) & 1u;
                    if constexpr (RGBD) {   // (NaN: no depth; RIG: in camera cc's frame)
                        const size_t ef = RIG ? (size_t)frame * n_cams + cc : (size_t)frame;
                        flag = flag && __ldg(eye + (ef * DSAC_N_CONST + c) * 3 + 2) > 0.0;
                    }
                    const uint32_t m = __ballot_sync(0xffffffffu, flag);
                    const int rank = count + __popc(m & ((1u << lane) - 1u));
                    if (flag && rank < p.inlier_count) {
                        sel[rank] = (unsigned short)(RIG ? (cc << 11 | c) : c);
                        imap[c] += 1;  // cnn_softam.h:1129 (each cell appears once per permutation)
                    }
                    count = min(count + __popc(m), p.inlier_count);
                }
                total += count;
            }
            if (lane == 0) s_count = total;
        }
        __syncthreads();
        const int count = s_count;
        if (count < 50) break;  // cnn_softam.h:1136

        if constexpr (RGBD && RIG) {
            // ---- Kabsch fit of the selected cells of every camera, scene to rig-frame eye point, in selection order
            extern __shared__ double s_kdyn[];   // [C K4_MAX_INLIERS * 3] scene, then as many rig-frame eye coordinates
            double* ka = s_kdyn;
            double* kb = s_kdyn + (size_t)n_cams * K4_MAX_INLIERS * 3;
            for (int i = tid; i < count; i += K4_THREADS) {
                const int code = s_sel[i], fr = frame * n_cams + (code >> 11), cell = code & 2047;
                const int16_t* co = p.coords + ((size_t)fr * DSAC_N_CONST + cell) * 3;
                const double* E = rig.ext + (size_t)fr * 12;
                ka[i * 3] = (double)__ldg(co); ka[i * 3 + 1] = (double)__ldg(co + 1); ka[i * 3 + 2] = (double)__ldg(co + 2);
                rig_point(E, E + 9, eye + ((size_t)fr * DSAC_N_CONST + cell) * 3, kb + i * 3);
            }
            __syncthreads();
            if (tid == 0) {
                double R[9], t[3], r[3];
                kabsch_fit(count, ka, kb, R, t);
                rodrigues_m2v(R, r);
                s_param[0] = r[0]; s_param[1] = r[1]; s_param[2] = r[2];
                s_param[3] = t[0]; s_param[4] = t[1]; s_param[5] = t[2];
            }
            __syncthreads();
        } else if constexpr (RGBD) {
            // ---- Kabsch fit of the selected cells: gathered in selection order, one thread fits
            __shared__ double s_ka[K4_MAX_INLIERS * 3], s_kb[K4_MAX_INLIERS * 3];
            for (int i = tid; i < count; i += K4_THREADS) {
                const int c = s_sel[i];
                const double* e = eye + ((size_t)frame * DSAC_N_CONST + c) * 3;
                s_ka[i * 3] = (double)s_cX[c]; s_ka[i * 3 + 1] = (double)s_cY[c]; s_ka[i * 3 + 2] = (double)s_cZ[c];
                s_kb[i * 3] = e[0]; s_kb[i * 3 + 1] = e[1]; s_kb[i * 3 + 2] = e[2];
            }
            __syncthreads();
            if (tid == 0) {
                double R[9], t[3], r[3];
                kabsch_fit(count, s_ka, s_kb, R, t);
                rodrigues_m2v(R, r);
                s_param[0] = r[0]; s_param[1] = r[1]; s_param[2] = r[2];
                s_param[3] = t[0]; s_param[4] = t[1]; s_param[5] = t[2];
            }
            __syncthreads();
        } else {
        // ---- Levenberg-Marquardt, CvLevMarq(6, 2n, max_iter 20, eps FLT_EPSILON)
        load_selected(count);
        // (state used by warp 0 only, uniform across its lanes; trial / base parameter vectors live in s_param / s_prev)
        LMState lm;
        if (warp == 0) {
            double r0[3] = {s_pose[0], s_pose[1], s_pose[2]};
            if (lane < 6) s_param[lane] = s_pose[lane];
            rodrigues_jac_warp(r0, lane, s_R, s_J);
            if (lane == 0) s_ctl = 0;
        }
        __syncthreads();
        for (;;) {
            if (s_ctl) break;
            normal_equations_pass(count);
            __syncthreads();
            if (warp == 0) {
                const int buf = lm_next_buf(lm);
                {
                    double t = 0;
#pragma unroll
                    for (int w = 0; w < K4_WARPS; w++) t += s_red[w][lane];
                    s_sum[buf][lane] = t;
                }
                __syncwarp();
                const int action = lm_advance(lm, buf, s_sum[buf][27], s_param, s_prev);
                if (action != LM_DONE) {
                    __syncwarp();             // every lane has read s_prev / s_param in lm_advance
                    if (action == LM_SOLVE_NEWBASE && lane < 6) s_prev[lane] = s_param[lane];
                    __syncwarp();
                    double x[6], trial[6];
                    lm_solve6_fast(s_sum[lm.cur], c_lm_lambda[lm.lambdaLg10 + 16], x);
#pragma unroll
                    for (int k = 0; k < 6; k++) trial[k] = s_prev[k] - x[k];
                    __syncwarp();
#pragma unroll
                    for (int k = 0; k < 6; k++)
                        if (lane == k) s_param[k] = trial[k];
                    rodrigues_jac_warp(trial, lane, s_R, s_J);
                }
                if (lane == 0) s_ctl = (action == LM_DONE) ? 1 : 0;
            }
            __syncthreads();
        }
        }
        // NaN -> abort without accepting (cnn_softam.h:1147)
        bool nan = false;
        for (int a = 0; a < 6; a++)
            if (s_param[a] != s_param[a]) nan = true;
        if (nan) break;
        __syncthreads();
        if (tid < 6) s_pose[tid] = s_param[tid];
        if constexpr (RECORD) {
            for (int i = tid; i < count; i += K4_THREADS) s_rec[i] = s_sel[i];
            if (tid == 0) s_rec_count = count;
        }
        __syncthreads();
        steps_done++;
        inlier_flags();
    }

    // ---- outputs
    if (tid < 6) p.out_pose[(size_t)job * 6 + tid] = s_pose[tid];
    if constexpr (RECORD) {
        const int rc = s_rec_count;
        const size_t stride = RIG ? (size_t)n_cams * K4_MAX_INLIERS : (size_t)K4_MAX_INLIERS;
        for (int i = tid; i < rc; i += K4_THREADS) rec_sel[(size_t)job * stride + i] = s_rec[i];
        if (tid == 0) rec_count[job] = rc;
    }
    if (p.inlier_map)
        for (int i = tid; i < n_cams * DSAC_N_CONST; i += K4_THREADS) p.inlier_map[(size_t)job * n_cams * DSAC_N_CONST + i] = s_imap[i];
    if (tid == 0) {
        if (p.steps_done) p.steps_done[job] = steps_done;
        if (p.n_perm_steps) p.n_perm_steps[job] = n_perm;
        if (p.status && steps_done < p.ref_steps) atomicOr(p.status + frame, 2u /* DSAC_ST_REFINE_ABORTED */);
        double pose[6], R[9], t[3];
        for (int k = 0; k < 6; k++) pose[k] = s_pose[k];
        if (p.out_jp6 || p.gt_jp) cv2our_dev(pose, R, t);
        if (p.out_jp6) {
            double r[3];
            rodrigues_m2v(R, r);
            double* o = p.out_jp6 + (size_t)job * 6;
            o[0] = r[0]; o[1] = r[1]; o[2] = r[2]; o[3] = t[0]; o[4] = t[1]; o[5] = t[2];
        }
        if (p.gt_jp) {
            const double* g = p.gt_jp + (size_t)frame * 12;
            double re, te;
            double l = max_loss_dev(g, g + 9, R, t, &re, &te);
            p.loss[job] = l;
            p.rot_err[job] = re;
            p.t_err[job] = te;
            p.correct[job] = (re < 5 && te < 50) ? 1 : 0;
        }
    }
}

__global__ void __launch_bounds__(K4_THREADS, K4_MIN_BLOCKS) k_refine(RefineParams p) { k_refine_body<false>(p); }
// the same with the per-frame camera table (RefineParams::cams)
__global__ void __launch_bounds__(K4_THREADS, K4_MIN_BLOCKS) k_refine_cam(RefineParams p) { k_refine_body<true>(p); }

// the same for RGB-D passes: eye [n_frames][N][3] eye coordinates of the cells (rgbd.cuh)
__global__ void __launch_bounds__(K4_THREADS, K4_MIN_BLOCKS) k_refine_rgbd(RefineParams p, const double* eye) { k_refine_body<false, true>(p, eye); }
__global__ void __launch_bounds__(K4_THREADS, K4_MIN_BLOCKS) k_refine_rgbd_cam(RefineParams p, const double* eye) { k_refine_body<true, true>(p, eye); }

// the recording replays (RECORD: rec_sel [n_jobs][K4_MAX_INLIERS], rec_count [n_jobs])
__global__ void __launch_bounds__(K4_THREADS, K4_MIN_BLOCKS) k_refine_rec(RefineParams p, uint16_t* rec_sel, int32_t* rec_count) {
    k_refine_body<false, false, true>(p, nullptr, rec_sel, rec_count);
}
__global__ void __launch_bounds__(K4_THREADS, K4_MIN_BLOCKS) k_refine_rec_cam(RefineParams p, uint16_t* rec_sel, int32_t* rec_count) {
    k_refine_body<true, false, true>(p, nullptr, rec_sel, rec_count);
}
__global__ void __launch_bounds__(K4_THREADS, K4_MIN_BLOCKS) k_refine_rgbd_rec(RefineParams p, const double* eye, uint16_t* rec_sel,
                                                                               int32_t* rec_count) {
    k_refine_body<false, true, true>(p, eye, rec_sel, rec_count);
}
__global__ void __launch_bounds__(K4_THREADS, K4_MIN_BLOCKS) k_refine_rgbd_rec_cam(RefineParams p, const double* eye, uint16_t* rec_sel,
                                                                                   int32_t* rec_count) {
    k_refine_body<true, true, true>(p, eye, rec_sel, rec_count);
}

// multi-camera rigs: one job per rig (RefineParams::status, gt_jp and the outputs per rig; cams, coords and pix per frame)
// (one CTA per rig, so a few hundred CTAs at most: the register budget of two CTAs per SM keeps the C-camera loops out of
// local memory)
__global__ void __launch_bounds__(K4_THREADS, 2) k_refine_rig(RefineParams p, RigRefine rig) {
    k_refine_body<false, false, false, true>(p, nullptr, nullptr, nullptr, rig);
}
__global__ void __launch_bounds__(K4_THREADS, 2) k_refine_rig_cam(RefineParams p, RigRefine rig) {
    k_refine_body<true, false, false, true>(p, nullptr, nullptr, nullptr, rig);
}
// the rig's recording replay (rec_sel [n_jobs][C K4_MAX_INLIERS] of entries cam << 11 | cell, rec_count [n_jobs])
__global__ void __launch_bounds__(K4_THREADS, 2) k_refine_rig_rec(RefineParams p, RigRefine rig, uint16_t* rec_sel, int32_t* rec_count) {
    k_refine_body<false, false, true, true>(p, nullptr, rec_sel, rec_count, rig);
}
__global__ void __launch_bounds__(K4_THREADS, 2) k_refine_rig_rec_cam(RefineParams p, RigRefine rig, uint16_t* rec_sel, int32_t* rec_count) {
    k_refine_body<true, false, true, true>(p, nullptr, rec_sel, rec_count, rig);
}

// the instantiations by per-frame camera (RefineParams::cams), one table per signature
constexpr void (*k_refine_tab[2])(RefineParams) = {k_refine, k_refine_cam};
constexpr void (*k_refine_rgbd_tab[2])(RefineParams, const double*) = {k_refine_rgbd, k_refine_rgbd_cam};
constexpr void (*k_refine_rec_tab[2])(RefineParams, uint16_t*, int32_t*) = {k_refine_rec, k_refine_rec_cam};
constexpr void (*k_refine_rgbd_rec_tab[2])(RefineParams, const double*, uint16_t*, int32_t*) = {k_refine_rgbd_rec, k_refine_rgbd_rec_cam};
constexpr void (*k_refine_rig_tab[2])(RefineParams, RigRefine) = {k_refine_rig, k_refine_rig_cam};
constexpr void (*k_refine_rig_rec_tab[2])(RefineParams, RigRefine, uint16_t*, int32_t*) = {k_refine_rig_rec, k_refine_rig_rec_cam};

// RGB-D rigs: eye [n_frames][N][3] of every camera frame, and the dynamic shared memory of the Kabsch fit
// (rig_kabsch_smem(rig.C) bytes; 48 KB at C = 8)
constexpr size_t rig_kabsch_smem(int C) { return (size_t)2 * C * K4_MAX_INLIERS * 3 * sizeof(double); }
__global__ void __launch_bounds__(K4_THREADS, 2) k_refine_rig_rgbd(RefineParams p, RigRefine rig, const double* eye) {
    k_refine_body<false, true, false, true>(p, eye, nullptr, nullptr, rig);
}
__global__ void __launch_bounds__(K4_THREADS, 2) k_refine_rig_rgbd_cam(RefineParams p, RigRefine rig, const double* eye) {
    k_refine_body<true, true, false, true>(p, eye, nullptr, nullptr, rig);
}
__global__ void __launch_bounds__(K4_THREADS, 2) k_refine_rig_rgbd_rec(RefineParams p, RigRefine rig, const double* eye, uint16_t* rec_sel,
                                                                       int32_t* rec_count) {
    k_refine_body<false, true, true, true>(p, eye, rec_sel, rec_count, rig);
}
__global__ void __launch_bounds__(K4_THREADS, 2) k_refine_rig_rgbd_rec_cam(RefineParams p, RigRefine rig, const double* eye, uint16_t* rec_sel,
                                                                           int32_t* rec_count) {
    k_refine_body<true, true, true, true>(p, eye, rec_sel, rec_count, rig);
}
constexpr void (*k_refine_rig_rgbd_tab[2])(RefineParams, RigRefine, const double*) = {k_refine_rig_rgbd, k_refine_rig_rgbd_cam};
constexpr void (*k_refine_rig_rgbd_rec_tab[2])(RefineParams, RigRefine, const double*, uint16_t*, int32_t*) = {k_refine_rig_rgbd_rec,
                                                                                                          k_refine_rig_rgbd_rec_cam};

// one CTA per job, with the instantiation the parameters ask for; eye != null: an RGB-D pass
inline void launch_refine(const RefineParams& p, unsigned jobs, cudaStream_t stream, const double* eye = nullptr) {
    if (eye) k_refine_rgbd_tab[p.cams != nullptr]<<<jobs, K4_THREADS, 0, stream>>>(p, eye);
    else k_refine_tab[p.cams != nullptr]<<<jobs, K4_THREADS, 0, stream>>>(p);
}
inline void launch_refine_record(const RefineParams& p, unsigned jobs, cudaStream_t stream, const double* eye, uint16_t* rec_sel,
                                 int32_t* rec_count) {
    if (eye) k_refine_rgbd_rec_tab[p.cams != nullptr]<<<jobs, K4_THREADS, 0, stream>>>(p, eye, rec_sel, rec_count);
    else k_refine_rec_tab[p.cams != nullptr]<<<jobs, K4_THREADS, 0, stream>>>(p, rec_sel, rec_count);
}
// one CTA per rig (p.n_jobs jobs), with the instantiation the parameters ask for: eye != null an RGB-D rig, rec_sel != null the
// recording replay.  (The engine raises the RGB-D forms' dynamic shared memory limit to rig_kabsch_smem(RIG_MAX_CAMERAS) at
// creation: with their static shared memory it exceeds the default at C = 8.)
inline void launch_refine_rig(const RefineParams& p, RigRefine rig, cudaStream_t stream, const double* eye = nullptr,
                              uint16_t* rec_sel = nullptr, int32_t* rec_count = nullptr) {
    const int cam = p.cams != nullptr;
    const unsigned jobs = (unsigned)p.n_jobs;
    const size_t smem = rig_kabsch_smem(rig.C);
    if (eye && rec_sel) k_refine_rig_rgbd_rec_tab[cam]<<<jobs, K4_THREADS, smem, stream>>>(p, rig, eye, rec_sel, rec_count);
    else if (eye) k_refine_rig_rgbd_tab[cam]<<<jobs, K4_THREADS, smem, stream>>>(p, rig, eye);
    else if (rec_sel) k_refine_rig_rec_tab[cam]<<<jobs, K4_THREADS, 0, stream>>>(p, rig, rec_sel, rec_count);
    else k_refine_rig_tab[cam]<<<jobs, K4_THREADS, 0, stream>>>(p, rig);
}

}  // namespace dsac
