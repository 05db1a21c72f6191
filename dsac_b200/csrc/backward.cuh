// backward.cuh -- K5/K6: backward of the soft-argmax pipeline, the chain rule assembled in
// train_ransac_softam.cpp:288-394 with the closed-form soft-inlier score in place of the Score CNN:
//
//   path I   dLoss/dY += dLossMax . dRefineObj                      (maxloss.h:87, cnn_softam.h:853)
//            dLoss/dY += dLossMax . dRefineHyp . sum_h sf_h dPNP_h   (cnn_softam.h:738, :101)
//   path II  dLoss/dY += sum_h dScore_h(scoreOutputGradients_h)      (train_ransac_softam.cpp:361-383,
//                                                                     cnn_softam.h:564-646)
//
// dRefineObj / dRefineHyp are central differences through the whole refinement: they are batched
// as jobs of the forward's k_refine kernel (refine.cuh).  dPNP is 24 full P3P solves per
// hypothesis.  dScore keeps a thread per scene coordinate, loops over the hypotheses in
// registers and reduces the per-hypothesis 1x6 with warp shuffles (all fp64, like the reference).
#pragma once
#include <cuda_runtime.h>

#include "ift.cuh"
#include "pose_math.cuh"
#include "refine.cuh"
#include "rigid.cuh"

struct dsac_engine;
struct dsac_backward_out;

namespace dsac {

constexpr int BW_MAX_OBJ_PIX = 16;                       // ceil(1600 / skip) with skip = 1/rSS = 100
constexpr int BW_JOBS = 12 + BW_MAX_OBJ_PIX * 6;         // refine jobs per frame (dRefineHyp + dRefineObj)

// Views into the engine's backward scratch block (dsac_engine::bw_buf); passed to the kernels by value, so it owns nothing.
struct BackwardScratch {
    int n_cap = 0;
    int32_t* job_frame = nullptr;    // [n][BW_JOBS]
    double* job_init = nullptr;      // [n][BW_JOBS][6]
    int32_t* job_pert = nullptr;     // [n][BW_JOBS][2]
    double* job_pose = nullptr;      // [n][BW_JOBS][6]
    double* job_jp6 = nullptr;       // [n][BW_JOBS][6]
    int32_t* obj_cells = nullptr;    // [n][BW_MAX_OBJ_PIX]  cell of each processed pixel, -1 unused
    double* dl = nullptr;            // [n][6]   dLossMax
    double* dldavg = nullptr;        // [n][6]   dLossMax . dRefineHyp
    double* drefhyp = nullptr;       // [n][36]
    double* sog = nullptr;           // [n][H]   scoreOutputGradients
    double* dpnp = nullptr;          // [n][H][72]
    double* hypjp = nullptr;         // [n][H][39]  R(9) t(3) J(27) of every hypothesis in jp convention
    double* row = nullptr;           // [n][N*3]  dLoss_dObj_1row
    double* drefobj = nullptr;       // [n][6][N*3] (diagnostic, optional)
    double* part = nullptr;          // [n][groups][N*3] partial rows of k_dscore
    int groups = 1;
};

// Hypothesis(cv2our(pose)).getRodVecAndTrans()  (Hypothesis.cpp:274-290)
__device__ __forceinline__ void jp6_from_cv_dev(const double pose[6], double out[6]) {
    double R[9], t[3];
    cv2our_dev(pose, R, t);
    rodrigues_m2v(R, out);
    out[3] = t[0]; out[4] = t[1]; out[5] = t[2];
}

// jp 6-vectors of `count` refined cv poses (dsac_refined_jp6_device): the vector refine(), dLossMax and the
// finite-difference jobs (job_jp6) work on, so the seed of a pose backward is the gradient with respect to it
__global__ void k_pose_jp6(const double* __restrict__ pose, size_t count, double* __restrict__ jp6) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    double o[6];
    jp6_from_cv_dev(pose + i * 6, o);
    for (int k = 0; k < 6; k++) jp6[i * 6 + k] = o[k];
}

// dLossMax, maxloss.h:87-198
__device__ void dloss_max_dev(const double est[6], const double gt[6], double jac[6]) {
    for (int i = 0; i < 6; i++) jac[i] = 0;
    double rot1[9], rot2[9], dRod[27];
    rodrigues_jac(est, rot1, dRod);
    rodrigues_v2m(gt, rot2);
    double diag = 0;  // trace(rot1 * rot2^T)
    for (int i = 0; i < 3; i++)
        for (int k = 0; k < 3; k++) diag += rot1[i * 3 + k] * rot2[i * 3 + k];
    double trace = fmin(3.0, fmax(-1.0, diag));
    double rotErr = rot_err_deg(trace);
    double a1[3] = {-est[3] / 10, -est[4] / 10, -est[5] / 10}, a2[3] = {-gt[3] / 10, -gt[4] / 10, -gt[5] / 10};
    double invT1[3], invT2[3];
    for (int r = 0; r < 3; r++) {  // invRot = rot^T
        invT1[r] = rot1[0 * 3 + r] * a1[0] + rot1[1 * 3 + r] * a1[1] + rot1[2 * 3 + r] * a1[2];
        invT2[r] = rot2[0 * 3 + r] * a2[0] + rot2[1 * 3 + r] * a2[1] + rot2[2 * 3 + r] * a2[2];
    }
    double d[3] = {invT1[0] - invT2[0], invT1[1] - invT2[1], invT1[2] - invT2[2]};
    double tErr = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    if (fmax(rotErr, tErr) > 10000000.0) return;
    if ((tErr + rotErr) < 1e-8) return;
    if (tErr > rotErr) {
        double dDist[3] = {d[0] / tErr, d[1] / tErr, d[2] / tErr};
        // cols 3..5 = dDist * (-invRot1), invRot1[i][j] = rot1[j][i]
        for (int j = 0; j < 3; j++) jac[3 + j] = -(dDist[0] * rot1[j * 3 + 0] + dDist[1] * rot1[j * 3 + 1] + dDist[2] * rot1[j * 3 + 2]);
        // dInvT1_dInvRot1 (3x9): row r has a1[0], a1[1], a1[2] at columns r, 3+r, 6+r   (maxloss.h:146-158)
        double v9[9];
        for (int k = 0; k < 9; k++) v9[k] = dDist[k % 3] * a1[k / 3];
        for (int j = 0; j < 3; j++) {
            double s = 0;
            for (int k = 0; k < 9; k++) s += v9[k] * dRod[j * 9 + k];
            jac[j] = s;
        }
    } else {
        // dTrace * dRotDiff: v9[k] = sum over the three diagonal blocks of invRot2 (maxloss.h:168-188)
        double v9[9];
        for (int blk = 0; blk < 3; blk++)
            for (int r = 0; r < 3; r++) v9[blk * 3 + r] = rot2[blk * 3 + r];  // invRot2[r][blk] = rot2[blk][r]
        double coef = 180 / kPi * -1 / sqrt(3 - trace * trace + 2 * trace);
        for (int j = 0; j < 3; j++) {
            double s = 0;
            for (int k = 0; k < 9; k++) s += v9[k] * dRod[j * 9 + k];
            jac[j] = coef * s;
        }
    }
    for (int i = 0; i < 6; i++)
        if (jac[i] != jac[i]) {
            for (int k = 0; k < 6; k++) jac[k] = 0;
            return;
        }
}

struct BwParams {
    const int16_t* coords;
    const int32_t* pix;
    int pix_stride;
    const double* gt_jp;        // [n][12]
    const double* seed;         // [n][6] dOuter/d(refined jp6) in place of dLossMax against gt_jp; null: dLossMax
    double f, cx, cy;
    const Cam* cams;            // [n] or null: the camera of every frame is f, cx, cy
    int H, thr, skip, fix_q4;
    double alpha, beta, grad_clamp;
    // forward state
    const double* hyp_pose;     // [n][H][6]
    const int32_t* img_idx;     // [n][H][4]
    const double* sf;           // [n][H]
    const double* avg_pose;     // [n][6]
    const double* ref_pose;     // [n][6]
    const int32_t* inlier_map;  // [n][N]
    BackwardScratch s;
    // k_dscore splits the hypotheses of a frame over `groups` CTAs; group g accumulates into part[frame][g][N*3]
    // (zeroed by the caller) and k_dscore_reduce adds the groups to s.row in order
    double* part;
    int groups;
    // score seam, adjoint side (lua_calls.h:312-341): when set, dScore/dDiffMap of every hypothesis comes from the
    // registered backward hook -- [n][H][40][40] doubles, element (y, x) as the reference's gradients[c](y, x) -- instead
    // of the closed-form derivative of the soft-inlier score
    const double* ext_g;
};

// ------------------------------------------------------------------ DSAC / RANSAC variant (train_ransac.cpp:304-381)
// dRefine of hypothesis h (cnn.h:866-990) is a list of refine() evaluations (cnn.h:787-852); each is one k_refine job.
// The jobs that perturb a minimal-set point start from the P3P pose of the PERTURBED set: this kernel computes it.
struct DsacBwParams {
    const int16_t* coords;
    const int32_t* pix;
    int pix_stride;
    double f, cx, cy;
    const Cam* cams;            // [n] or null: the camera of every frame is f, cx, cy
    int H;
    const int32_t* img_idx;     // [n][H][4]
    const double* ref_pose;     // [n*H][6] refined cv pose of every hypothesis (forward_dsac)
    const double* sf;           // [n*H]
    const double* gt_jp;        // [n][12]
    const double* seed;         // [n*H][6] dOuter/d(refined jp6) in place of sf_h dLossMax_h; null: sf_h dLossMax_h
    // jobs
    int n_jobs;
    const int32_t* job_frame;   // [n_jobs]
    const int32_t* job_p3p;     // [n_jobs][3] {global hypothesis index or -1, point*3+channel, delta}
    double* job_init;           // [n_jobs][6]
    const double* job_jp6;      // [n_jobs][6] results of k_refine
    // central-difference pairs (jobs 2p, 2p+1 = forward, backward step), sorted by frame, hypothesis
    int n_frames;
    const int32_t* frame_pair_begin;   // [n+1]
    const int32_t* pair_hyp;    // [n_pairs] global hypothesis index
    const int32_t* pair_col;    // [n_pairs] cell*3+channel
    const int32_t* pair_scale;  // [n_pairs] 1 or skip
    double* path1;              // [n][N*3]
};

__global__ void k_dsac_job_p3p(DsacBwParams p) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= p.n_jobs) return;
    const int hyp = p.job_p3p[j * 3];
    if (hyp < 0) return;
    const int frame = p.job_frame[j];
    const int16_t* coords = p.coords + (size_t)frame * DSAC_N_CONST * 3;
    const int32_t* pix = p.pix + (size_t)frame * p.pix_stride;
    const int32_t* idx = p.img_idx + (size_t)hyp * 4;
    float obj[12], img[8];
    for (int q = 0; q < 4; q++) {
        const int c = idx[q];
        img[q * 2] = (float)pix[c * 2];
        img[q * 2 + 1] = (float)pix[c * 2 + 1];
        for (int k = 0; k < 3; k++) obj[q * 3 + k] = (float)coords[c * 3 + k];
    }
    obj[p.job_p3p[j * 3 + 1]] += (float)p.job_p3p[j * 3 + 2];   // objPts[pt] +/- eps (integers in float: exact)
    double pose[6], R[9], t[3], e2;
    P3PProblem pr;
    const Cam cam = frame_cam(p, frame);
    make_problem(obj, img, cam.f, cam.cx, cam.cy, pr);
    if (p3p_best(pr, cam.f, cam.cx, cam.cy, R, t, &e2) > 0) {
        rodrigues_m2v(R, pose);
        pose[3] = t[0]; pose[4] = t[1]; pose[5] = t[2];
    } else {
        for (int k = 0; k < 6; k++) pose[k] = 0;   // safeSolvePnP leaves a zero pose (cnn.h:66-71)
    }
    for (int k = 0; k < 6; k++) p.job_init[(size_t)j * 6 + k] = pose[k];
}

// The same for an RGB-D pass: the initial pose of a job that perturbs a minimal-set point is the Kabsch fit of the
// perturbed points 0..2 to their eye points (eye [n][N][3]).  Depth is not perturbed: the gradient is the scene's.
__global__ void k_dsac_job_kabsch(DsacBwParams p, const double* __restrict__ eye) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= p.n_jobs) return;
    const int hyp = p.job_p3p[j * 3];
    if (hyp < 0) return;
    const int frame = p.job_frame[j];
    const int16_t* coords = p.coords + (size_t)frame * DSAC_N_CONST * 3;
    const double* ey = eye + (size_t)frame * DSAC_N_CONST * 3;
    const int32_t* idx = p.img_idx + (size_t)hyp * 4;
    double a[9], b[9];
    for (int q = 0; q < 3; q++)
        for (int k = 0; k < 3; k++) { a[q * 3 + k] = (double)coords[idx[q] * 3 + k]; b[q * 3 + k] = ey[idx[q] * 3 + k]; }
    const int pc = p.job_p3p[j * 3 + 1];
    if (pc < 9) a[pc] += (double)p.job_p3p[j * 3 + 2];
    double R[9], pose[6];
    kabsch_fit(3, a, b, R, pose + 3);
    rodrigues_m2v(R, pose);
    for (int k = 0; k < 6; k++) p.job_init[(size_t)j * 6 + k] = pose[k];
}

// path I: dLoss_dObj(idx, c) += sf_h * (dLossMax(refined_h, gt) . dRefine_h)(idx*3+c), hypotheses and columns in the
// reference's order (one thread per frame: the sums are reproducible)
// path I of the DSAC variant: row[col] += sf_h * dLossMax_h . (refine(+eps) - refine(-eps)) / (2 eps) * scale over the
// central-difference pairs of a frame, in pair order (pairs are sorted by hypothesis; a hypothesis touches a column at
// most once, so within one hypothesis' run the additions are independent, and the runs are applied one after the other).
// One warp per frame: first the lanes evaluate dLossMax of the frame's selected hypotheses in parallel, then the runs
// are walked in order with the lanes spread over a run's pairs.  A seeded backward takes seed_h with weight 1 in place
// of dLossMax_h with weight sf_h, and reads no ground truth.
constexpr int DSAC_COMBINE_MAX_HYPS = 1024;   // = DSAC_MAX_HYPS
__global__ void __launch_bounds__(32) k_dsac_combine(DsacBwParams p) {
    __shared__ int s_run_begin[DSAC_COMBINE_MAX_HYPS + 1];
    __shared__ double s_dl[32][7];                       // dLossMax (1x6) and sf of 32 runs' hypotheses at a time
    const int frame = blockIdx.x, lane = threadIdx.x;
    if (frame >= p.n_frames) return;
    double* row = p.path1 + (size_t)frame * DSAC_N_CONST * 3;
    const int q_begin = p.frame_pair_begin[frame], q_end = p.frame_pair_begin[frame + 1];
    // runs of equal hypothesis
    int n_runs = 0;
    for (int q0 = q_begin; q0 < q_end; q0 += 32) {
        const int q = q0 + lane;
        const bool start = q < q_end && (q == q_begin || p.pair_hyp[q] != p.pair_hyp[q - 1]);
        const unsigned m = __ballot_sync(0xffffffffu, start);
        if (start) {
            const int r = n_runs + __popc(m & ((1u << lane) - 1u));
            if (r < DSAC_COMBINE_MAX_HYPS) s_run_begin[r] = q;
        }
        n_runs += __popc(m);
    }
    n_runs = min(n_runs, DSAC_COMBINE_MAX_HYPS);
    if (lane == 0) s_run_begin[n_runs] = q_end;
    __syncwarp();
    // dLossMax of every run's hypothesis
    double gt6[6];
    if (!p.seed) {
        const double* g = p.gt_jp + (size_t)frame * 12;
        rodrigues_m2v(g, gt6);
        gt6[3] = g[9]; gt6[4] = g[10]; gt6[5] = g[11];
    }
    for (int r0 = 0; r0 < n_runs; r0 += 32) {
        if (r0 + lane < n_runs) {
            const int hyp = p.pair_hyp[s_run_begin[r0 + lane]];
            if (p.seed) {
                for (int k = 0; k < 6; k++) s_dl[lane][k] = p.seed[(size_t)hyp * 6 + k];
                s_dl[lane][6] = 1.0;
            } else {
                double ref6[6], dl[6];
                jp6_from_cv_dev(p.ref_pose + (size_t)hyp * 6, ref6);
                dloss_max_dev(ref6, gt6, dl);
                for (int k = 0; k < 6; k++) s_dl[lane][k] = dl[k];
                s_dl[lane][6] = p.sf[hyp];
            }
        }
        __syncwarp();
        for (int r = r0; r < min(n_runs, r0 + 32); r++) {
            const double sf = s_dl[r - r0][6];
            for (int q = s_run_begin[r] + lane; q < s_run_begin[r + 1]; q += 32) {
                const double* fS = p.job_jp6 + (size_t)(2 * q) * 6;
                const double* bS = fS + 6;
                const double scale = (double)p.pair_scale[q];
                double acc = 0;
                for (int k = 0; k < 6; k++) acc += s_dl[r - r0][k] * ((fS[k] - bS[k]) / 4.0 * scale);   // / (2 * eps), eps = 2; * skip
                row[p.pair_col[q]] += sf * acc;
            }
            __syncwarp();   // the next run may touch the same columns
        }
    }
}


// ---- per frame: dLossMax (or the caller's seed) and the refine job list (one warp, lane 0 does the serial scan).
// IMPLICIT (dsac_set_coord_derivatives): the 12 dRefineHyp jobs only, BW_JOBS_IMPLICIT per frame; dRefineObj is k_refine_ift's.
constexpr int BW_JOBS_IMPLICIT = 12;
template <bool IMPLICIT>
__device__ __forceinline__ void bw_prep_body(const BwParams& p, int n) {
    constexpr int BW_JOBS = IMPLICIT ? BW_JOBS_IMPLICIT : dsac::BW_JOBS;
    const int frame = blockIdx.x * blockDim.x + threadIdx.x;
    if (frame >= n) return;
    // dLoss/dRefinedPose
    if (p.seed) {
        for (int k = 0; k < 6; k++) p.s.dl[(size_t)frame * 6 + k] = p.seed[(size_t)frame * 6 + k];
    } else {
        double ref6[6], gt6[6], dl[6];
        jp6_from_cv_dev(p.ref_pose + (size_t)frame * 6, ref6);
        const double* g = p.gt_jp + (size_t)frame * 12;
        rodrigues_m2v(g, gt6);  // poseGT.getRodVecAndTrans()
        gt6[3] = g[9]; gt6[4] = g[10]; gt6[5] = g[11];
        dloss_max_dev(ref6, gt6, dl);
        for (int k = 0; k < 6; k++) p.s.dl[(size_t)frame * 6 + k] = dl[k];
    }
    // jobs 0..11: dRefineHyp (cnn_softam.h:756-833): +-eps on the cv rvec (eps = 0.001f) / cv tvec (eps*1000)
    int32_t* jf = p.s.job_frame + (size_t)frame * BW_JOBS;
    double* ji = p.s.job_init + (size_t)frame * BW_JOBS * 6;
    int32_t* jp = p.s.job_pert + (size_t)frame * BW_JOBS * 2;
    const double* avg = p.avg_pose + (size_t)frame * 6;
    const float eps = 0.001f;
    for (int i = 0; i < 6; i++) {
        double init[6];
        for (int k = 0; k < 6; k++) init[k] = avg[k];
        // the reference perturbs one shared copy in place: +eps, -2eps, +eps (the residue of earlier
        // parameters is below double rounding of these magnitudes only by luck, so replay it exactly)
        for (int q = 0; q < i; q++) {
            if (q < 3) { init[q] += eps; init[q] -= 2 * eps; init[q] += eps; }
            else { init[q] += eps * 1000; init[q] -= 2 * eps * 1000; init[q] += eps * 1000; }
        }
        double fwd = init[i], bwd;
        if (i < 3) { fwd += eps; bwd = fwd; bwd -= 2 * eps; }
        else { fwd += eps * 1000; bwd = fwd; bwd -= 2 * eps * 1000; }
        for (int sgn = 0; sgn < 2; sgn++) {
            int j = i * 2 + sgn;
            jf[j] = frame;
            for (int k = 0; k < 6; k++) ji[j * 6 + k] = init[k];
            ji[j * 6 + i] = sgn ? bwd : fwd;
            jp[j * 2] = -1; jp[j * 2 + 1] = 0;
        }
    }
    if constexpr (IMPLICIT) return;
    // jobs 12..: dRefineObj (cnn_softam.h:866-920): every skip-th ever-inlier pixel, x outer / y inner
    const int32_t* im = p.inlier_map + (size_t)frame * DSAC_N_CONST;
    int32_t* oc = p.s.obj_cells + (size_t)frame * BW_MAX_OBJ_PIX;
    int inCount = 0, npx = 0;
    for (int x = 0; x < DSAC_GRID_CONST; x++)
        for (int y = 0; y < DSAC_GRID_CONST; y++) {
            if (im[y * DSAC_GRID_CONST + x] == 0) continue;
            inCount++;
            if (inCount % p.skip != 0) continue;
            if (npx < BW_MAX_OBJ_PIX) oc[npx++] = y * DSAC_GRID_CONST + x;
        }
    for (int k = npx; k < BW_MAX_OBJ_PIX; k++) oc[k] = -1;
    for (int px = 0; px < BW_MAX_OBJ_PIX; px++)
        for (int c = 0; c < 3; c++)
            for (int sgn = 0; sgn < 2; sgn++) {
                int j = 12 + (px * 3 + c) * 2 + sgn;
                if (px < npx) {
                    jf[j] = frame;
                    for (int k = 0; k < 6; k++) ji[j * 6 + k] = avg[k];
                    jp[j * 2] = oc[px] * 3 + c;
                    jp[j * 2 + 1] = sgn ? -2 : 2;   // short += eps (2.f), then -= 2*eps  (cnn_softam.h:887,901)
                } else {
                    jf[j] = -1;
                    jp[j * 2] = -1; jp[j * 2 + 1] = 0;
                }
            }
}

__global__ void k_bw_prep(BwParams p, int n) { bw_prep_body<false>(p, n); }
__global__ void k_bw_prep_implicit(BwParams p, int n) { bw_prep_body<true>(p, n); }

// ---- per frame (one warp): dRefineHyp, dLossMax . dRefineObj into the row, scoreOutputGradients (IMPLICIT: no dRefineObj
// columns, k_refine_ift adds them)
template <bool IMPLICIT>
__device__ __forceinline__ void bw_combine_body(const BwParams& p, int n) {
    constexpr int BW_JOBS = IMPLICIT ? BW_JOBS_IMPLICIT : dsac::BW_JOBS;
    const int frame = blockIdx.x, lane = threadIdx.x;
    if (frame >= n) return;
    __shared__ double s_dref[36], s_dl[6], s_dldavg[6];
    const double* jp6 = p.s.job_jp6 + (size_t)frame * BW_JOBS * 6;
    const float eps = 0.001f;
    if (lane < 6) s_dl[lane] = p.s.dl[(size_t)frame * 6 + lane];
    if (lane < 6) {
        const int i = lane;
        const double* fS = jp6 + (i * 2) * 6;
        const double* bS = jp6 + (i * 2 + 1) * 6;
        for (int k = 0; k < 3; k++) s_dref[k * 6 + i] = (fS[k] - bS[k]) / (2 * eps);
        for (int k = 3; k < 6; k++) s_dref[k * 6 + i] = (fS[k] - bS[k]) / (2 * eps * 1000);
    }
    __syncwarp();
    if (lane < 6) {
        double s = 0;
        for (int k = 0; k < 6; k++) s += s_dl[k] * s_dref[k * 6 + lane];
        s_dldavg[lane] = s;
        p.s.dldavg[(size_t)frame * 6 + lane] = s;
    }
    for (int k = lane; k < 36; k += 32) p.s.drefhyp[(size_t)frame * 36 + k] = s_dref[k];
    __syncwarp();
    // dRefineObj columns -> row (and the optional 6 x 4800 diagnostic matrix)
    double* row = p.s.row + (size_t)frame * DSAC_N_CONST * 3;
    const int32_t* oc = p.s.obj_cells + (size_t)frame * BW_MAX_OBJ_PIX;
    for (int col = lane; !IMPLICIT && col < BW_MAX_OBJ_PIX * 3; col += 32) {
        const int px = col / 3, c = col % 3;
        if (oc[px] < 0) continue;
        const double* fS = jp6 + (12 + col * 2) * 6;
        const double* bS = jp6 + (12 + col * 2 + 1) * 6;
        const float eps2 = 2.f;
        double s = 0;
        for (int k = 0; k < 6; k++) {
            double v = (fS[k] - bS[k]) / (2 * eps2) * p.skip;   // cnn_softam.h:918
            s += s_dl[k] * v;
            if (p.s.drefobj) p.s.drefobj[((size_t)frame * 6 + k) * DSAC_N_CONST * 3 + oc[px] * 3 + c] = v;
        }
        row[oc[px] * 3 + c] += s;   // distinct cells: no conflicts
    }
    __syncwarp();
    // scoreOutputGradients (train_ransac_softam.cpp:361-376): g_j = sf_j (hf_j - sum_h sf_h hf_h)
    const double* hp = p.hyp_pose + (size_t)frame * p.H * 6;
    const double* sf = p.sf + (size_t)frame * p.H;
    double part = 0;
    for (int h = lane; h < p.H; h += 32) {
        double hf = 0;
        for (int i = 0; i < 3; i++) hf += s_dldavg[i] * hp[h * 6 + i] + s_dldavg[3 + i] * (hp[h * 6 + 3 + i] / 1000);
        part += sf[h] * hf;
    }
    for (int off = 16; off; off >>= 1) part += __shfl_xor_sync(0xffffffffu, part, off);
    for (int h = lane; h < p.H; h += 32) {
        double hf = 0;
        for (int i = 0; i < 3; i++) hf += s_dldavg[i] * hp[h * 6 + i] + s_dldavg[3 + i] * (hp[h * 6 + 3 + i] / 1000);
        p.s.sog[(size_t)frame * p.H + h] = sf[h] * hf - sf[h] * part;
    }
}
__global__ void k_bw_combine(BwParams p, int n) { bw_combine_body<false>(p, n); }
__global__ void k_bw_combine_implicit(BwParams p, int n) { bw_combine_body<true>(p, n); }

// ---- dPNP (cnn_softam.h:101-146): thread = (hypothesis, column 0..11); 2 full P3P solves each.
// Also prepares the jp pose + Rodrigues Jacobian of every hypothesis for k_dscore.
__global__ void __launch_bounds__(192) k_dpnp(BwParams p) {
    const int frame = blockIdx.y;
    const int h = blockIdx.x * 16 + threadIdx.x / 12, col = threadIdx.x % 12;
    __shared__ int s_nan[16];
    if (threadIdx.x < 16) s_nan[threadIdx.x] = 0;
    __syncthreads();
    const bool active = h < p.H;
    double colv[6] = {0, 0, 0, 0, 0, 0};
    if (active) {
        const int16_t* coords = p.coords + (size_t)frame * DSAC_N_CONST * 3;
        const int32_t* pix = p.pix + (size_t)frame * p.pix_stride;
        const int32_t* idx = p.img_idx + ((size_t)frame * p.H + h) * 4;
        float obj[12], img[8];
        bool valid = true;
        for (int j = 0; j < 4; j++) {
            int c = idx[j];
            if (c < 0) { valid = false; c = 0; }
            img[j * 2] = (float)pix[c * 2];
            img[j * 2 + 1] = (float)pix[c * 2 + 1];
            for (int k = 0; k < 3; k++) obj[j * 3 + k] = (float)coords[c * 3 + k];
        }
        const float eps = 0.1f;
        // columns before `col` were perturbed and restored in float by the reference's serial loop
        for (int q = 0; q < col; q++) {
            obj[q] += eps;
            obj[q] -= 2 * eps;
            obj[q] += eps;
        }
        double fS[6], bS[6], pose[6], R[9], t[3], e2;
        P3PProblem pr;
        const Cam cam = frame_cam(p, frame);
        obj[col] += eps;
        make_problem(obj, img, cam.f, cam.cx, cam.cy, pr);
        if (valid && p3p_best(pr, cam.f, cam.cx, cam.cy, R, t, &e2) > 0) {
            rodrigues_m2v(R, pose);
            pose[3] = t[0]; pose[4] = t[1]; pose[5] = t[2];
        } else {
            for (int k = 0; k < 6; k++) pose[k] = 0;  // safeSolvePnP, cnn_softam.h:66-71
        }
        jp6_from_cv_dev(pose, fS);
        obj[col] -= 2 * eps;
        make_problem(obj, img, cam.f, cam.cx, cam.cy, pr);
        if (valid && p3p_best(pr, cam.f, cam.cx, cam.cy, R, t, &e2) > 0) {
            rodrigues_m2v(R, pose);
            pose[3] = t[0]; pose[4] = t[1]; pose[5] = t[2];
        } else {
            for (int k = 0; k < 6; k++) pose[k] = 0;
        }
        jp6_from_cv_dev(pose, bS);
        bool nan = false;
        for (int k = 0; k < 6; k++) {
            colv[k] = (fS[k] - bS[k]) / (2 * eps);
            if (colv[k] != colv[k]) nan = true;
        }
        if (nan) s_nan[threadIdx.x / 12] = 1;
    }
    __syncthreads();
    if (active) {
        // a NaN in column c makes the reference return zeros(6,12) at that point of its serial loop
        const bool zero = s_nan[threadIdx.x / 12] != 0;
        double* out = p.s.dpnp + ((size_t)frame * p.H + h) * 72;
        for (int k = 0; k < 6; k++) out[k * 12 + col] = zero ? 0.0 : colv[k];
        if (col == 0) {  // jp pose + Rodrigues Jacobian of this hypothesis (dScore re-solves the same P3P: cnn_softam.h:597-598)
            double* hj = p.s.hypjp + ((size_t)frame * p.H + h) * 39;
            double R[9], t[3], rod[3], Rt[9], J[27];
            cv2our_dev(p.hyp_pose + ((size_t)frame * p.H + h) * 6, R, t);
            rodrigues_m2v(R, rod);
            rodrigues_jac(rod, Rt, J);
            for (int k = 0; k < 9; k++) hj[k] = R[k];
            for (int k = 0; k < 3; k++) hj[9 + k] = t[k];
            for (int k = 0; k < 27; k++) hj[12 + k] = J[k];
        }
    }
}

// ---- dPNP of an RGB-D pass: the same central differences (eps 0.1 on the float coordinates, the reference's serial
// perturb / restore) of the 3-point Kabsch hypothesis, scene to eye (eye [n][N][3]); the columns of the 4th point are
// zero, since the fit does not use it.  Also the jp pose + Rodrigues Jacobian of every hypothesis for k_dscore.
__global__ void __launch_bounds__(192) k_dkabsch(BwParams p, const double* __restrict__ eye) {
    const int frame = blockIdx.y;
    const int h = blockIdx.x * 16 + threadIdx.x / 12, col = threadIdx.x % 12;
    __shared__ int s_nan[16];
    if (threadIdx.x < 16) s_nan[threadIdx.x] = 0;
    __syncthreads();
    const bool active = h < p.H;
    double colv[6] = {0, 0, 0, 0, 0, 0};
    if (active && col < 9) {
        const int16_t* coords = p.coords + (size_t)frame * DSAC_N_CONST * 3;
        const double* ey = eye + (size_t)frame * DSAC_N_CONST * 3;
        const int32_t* idx = p.img_idx + ((size_t)frame * p.H + h) * 4;
        float obj[9];
        double b[9];
        bool valid = true;
        for (int j = 0; j < 3; j++) {
            int c = idx[j];
            if (c < 0) { valid = false; c = 0; }
            for (int k = 0; k < 3; k++) { obj[j * 3 + k] = (float)coords[c * 3 + k]; b[j * 3 + k] = ey[c * 3 + k]; }
        }
        const float eps = 0.1f;
        for (int q = 0; q < col; q++) {
            obj[q] += eps;
            obj[q] -= 2 * eps;
            obj[q] += eps;
        }
        double fS[6], bS[6];
        for (int side = 0; side < 2; side++) {
            obj[col] += side ? -2 * eps : eps;
            double a[9], R[9], pose[6] = {0, 0, 0, 0, 0, 0};
            for (int k = 0; k < 9; k++) a[k] = (double)obj[k];
            if (valid) {
                kabsch_fit(3, a, b, R, pose + 3);
                rodrigues_m2v(R, pose);
            }
            jp6_from_cv_dev(pose, side ? bS : fS);
        }
        bool nan = false;
        for (int k = 0; k < 6; k++) {
            colv[k] = (fS[k] - bS[k]) / (2 * eps);
            if (colv[k] != colv[k]) nan = true;
        }
        if (nan) s_nan[threadIdx.x / 12] = 1;
    }
    __syncthreads();
    if (active) {
        const bool zero = s_nan[threadIdx.x / 12] != 0;
        double* out = p.s.dpnp + ((size_t)frame * p.H + h) * 72;
        for (int k = 0; k < 6; k++) out[k * 12 + col] = zero ? 0.0 : colv[k];
        if (col == 0) {
            double* hj = p.s.hypjp + ((size_t)frame * p.H + h) * 39;
            double R[9], t[3], rod[3], Rt[9], J[27];
            cv2our_dev(p.hyp_pose + ((size_t)frame * p.H + h) * 6, R, t);
            rodrigues_m2v(R, rod);
            rodrigues_jac(rod, Rt, J);
            for (int k = 0; k < 9; k++) hj[k] = R[k];
            for (int k = 0; k < 3; k++) hj[9 + k] = t[k];
            for (int k = 0; k < 27; k++) hj[12 + k] = J[k];
        }
    }
}

// ---- per frame (one warp): row += dLdAvg . sum_h sf_h dPNP_h scattered to the support points
//      (train_ransac_softam.cpp:340-353); hypotheses in order, so the sums are reproducible
__global__ void k_bw_scatter_pnp(BwParams p, int n) {
    const int frame = blockIdx.x, lane = threadIdx.x;
    if (frame >= n || lane >= 12) return;
    double* row = p.s.row + (size_t)frame * DSAC_N_CONST * 3;
    const double* dld = p.s.dldavg + (size_t)frame * 6;
    double w[6];
    for (int k = 0; k < 6; k++) w[k] = dld[k];
    for (int h = 0; h < p.H; h++) {
        const int32_t* idx = p.img_idx + ((size_t)frame * p.H + h) * 4;
        const int c = idx[lane / 3];
        const double* J = p.s.dpnp + ((size_t)frame * p.H + h) * 72;
        double s = 0;
        for (int k = 0; k < 6; k++) s += w[k] * (p.sf[(size_t)frame * p.H + h] * J[k * 12 + lane]);
        if (c >= 0) row[c * 3 + lane % 3] += s;
        __syncwarp(0xfff);
    }
}

// ---- dScore (cnn_softam.h:564-646): thread = scene coordinate, loop over a group of the frame's hypotheses.
// grid (groups, frames): with one CTA per frame a training batch of 16..64 frames left most of the 132 SMs idle for the
// dominant kernel of the backward pass.  Every addition into a group's partial row is ordered (barriers of the h loop),
// and the groups are added in order, so the gradient is run-to-run reproducible.
constexpr int K5_THREADS = 320, K5_PTS = 5, K5_WARPS = K5_THREADS / 32;
constexpr int K5_MAX_GROUPS = 32;

// hypothesis groups for n frames: enough CTAs for ~4 per SM, at most K5_MAX_GROUPS, at least 8 hypotheses each
inline int dscore_groups(int n_frames, int n_hyps, int sm_count) {
    int g = (4 * sm_count + n_frames - 1) / std::max(1, n_frames);
    g = std::min(g, K5_MAX_GROUPS);
    g = std::min(g, std::max(1, n_hyps / 8));
    return std::max(1, g);
}

// scoreOutputGradients clamped to +-clamp, as the reference's score backward does before back-propagating
// (train_score_softam.lua:97) -- the copy a registered backward hook receives
__global__ void k_clamp_copy(const double* __restrict__ src, double* __restrict__ dst, size_t count, double clamp) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    double v = src[i];
    if (clamp > 0) v = fmax(-clamp, fmin(clamp, v));
    dst[i] = v;
}

__global__ void k_dscore_reduce(BwParams p) {
    const int frame = blockIdx.x;
    double* row = p.s.row + (size_t)frame * DSAC_N_CONST * 3;
    const double* part = p.part + (size_t)frame * p.groups * DSAC_N_CONST * 3;
    for (int c = threadIdx.x; c < DSAC_N_CONST * 3; c += blockDim.x) {
        double s = row[c];
        for (int g = 0; g < p.groups; g++) s += part[(size_t)g * DSAC_N_CONST * 3 + c];
        row[c] = s;
    }
}

// The rig backward's form (k_dscore_rig): frame f = r C + c scores its rig's pool, p.H = P slots with the composed poses
// T_c o T_j in hypjp [n][P][39]; the score output gradients are the rig's, sog [R][P], and the 1x6 sum over the cells goes
// to w [n][P][6] in place of the support scatter, which crosses cameras (rig.cuh, k_rig_bw_support).
struct RigDscore {
    int C;
    double* w;
};
template <bool RIG>
__device__ __forceinline__ void k_dscore_body(const BwParams& p, const RigDscore& rig) {
    __shared__ double s_h[39];
    __shared__ double s_red[K5_WARPS][6];
    __shared__ double s_w[6];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int frame = blockIdx.y, group = blockIdx.x;
    const int per_group = (p.H + p.groups - 1) / p.groups, h_begin = group * per_group, h_end = min(p.H, h_begin + per_group);
    const int16_t* coords = p.coords + (size_t)frame * DSAC_N_CONST * 3;
    const int32_t* pix = p.pix + (size_t)frame * p.pix_stride;
    double* row = p.part + ((size_t)frame * p.groups + group) * DSAC_N_CONST * 3;
    double X[K5_PTS], Y[K5_PTS], Z[K5_PTS], pu[K5_PTS], pv[K5_PTS], acc[K5_PTS][3];
#pragma unroll
    for (int j = 0; j < K5_PTS; j++) {
        int pt = tid + j * K5_THREADS;
        X[j] = (double)(float)coords[pt * 3]; Y[j] = (double)(float)coords[pt * 3 + 1]; Z[j] = (double)(float)coords[pt * 3 + 2];
        pu[j] = (double)(float)pix[pt * 2]; pv[j] = (double)(float)pix[pt * 2 + 1];
        acc[j][0] = acc[j][1] = acc[j][2] = 0;
    }
    const Cam cam = frame_cam(p, frame);
    const double f = cam.f, cx = cam.cx, cy = cam.cy;
    for (int h = h_begin; h < h_end; h++) {
        __syncthreads();
        if (tid < 39) s_h[tid] = p.s.hypjp[((size_t)frame * p.H + h) * 39 + tid];
        __syncthreads();
        double go = p.s.sog[(size_t)(RIG ? frame / rig.C : frame) * p.H + h];
        if (p.grad_clamp > 0) go = fmax(-p.grad_clamp, fmin(p.grad_clamp, go));   // train_score_softam.lua:97
        const double* R = s_h;       // jp rotation
        const double* t = s_h + 9;
        const double* J = s_h + 12;  // 3x9 Rodrigues Jacobian at rod(R)
        // cv pose of the same hypothesis for the reprojection-error image (getDiffMap on cvHyp, cnn_softam.h:601):
        // cv R = diag(1,-1,-1) R_jp, cv t = (t0,-t1,-t2)  (cv2our never flips for a proper rotation)
        double w6[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll
        for (int j = 0; j < K5_PTS; j++) {
            // --- diffmap entry with the reference's roundings (projection -> float, float diff, double norm, float store)
            double xc = dot3_plain(R[0], X[j], R[1], Y[j], R[2], Z[j], t[0]);
            double yc = dot3_plain(-R[3], X[j], -R[4], Y[j], -R[5], Z[j], -t[1]);
            double zc = dot3_plain(-R[6], X[j], -R[7], Y[j], -R[8], Z[j], -t[2]);
            double iz = zc ? __ddiv_rn(1., zc) : 1;
            float pfu = (float)__dadd_rn(__dmul_rn(__dmul_rn(xc, iz), f), cx), pfv = (float)__dadd_rn(__dmul_rn(__dmul_rn(yc, iz), f), cy);
            float du = __fsub_rn((float)pu[j], pfu), dv = __fsub_rn((float)pv[j], pfv);
            double e = (double)(float)fmin(sqrt(__dadd_rn(__dmul_rn((double)du, (double)du), __dmul_rn((double)dv, (double)dv))), 100.0);
            double g;
            if (p.ext_g) {
                g = p.ext_g[((size_t)frame * p.H + h) * DSAC_N_CONST + tid + j * K5_THREADS];   // backward hook's dDiffMaps[h](y,x)
            } else {
                double sg = 1.0 / (1.0 + exp(-p.beta * ((double)p.thr - e)));
                g = go * (-p.alpha * p.beta * sg * (1.0 - sg));   // dDiffMaps[h](y,x) under the soft-inlier score
            }
            // --- dProjectdObj / dProjectdHyp in the jp convention (cnn_softam.h:404-528)
            double ex = R[0] * X[j] + R[1] * Y[j] + R[2] * Z[j] + t[0];
            double ey = R[3] * X[j] + R[4] * Y[j] + R[5] * Z[j] + t[1];
            double ez = R[6] * X[j] + R[7] * Y[j] + R[8] * Z[j] + t[2];
            if (fabs(ez) < 1e-8) continue;
            double px = -f * ex / ez + cx, py = f * ey / ez + cy;
            double err = sqrt((pu[j] - px) * (pu[j] - px) + (pv[j] - py) * (pv[j] - py));
            if (err > 100.0) continue;
            err += 1e-8;
            double ddx = pu[j] - px, ddy = pv[j] - py;
#pragma unroll
            for (int k = 0; k < 3; k++) {
                double pxd = -f * R[0 * 3 + k] / ez + f * ex / ez / ez * R[2 * 3 + k];
                double pyd = f * R[1 * 3 + k] / ez - f * ey / ez / ez * R[2 * 3 + k];
                acc[j][k] += g * (0.5 / err * (2 * ddx * -pxd + 2 * ddy * -pyd));
            }
            double dN0 = -1 / err * ddx, dN1 = -1 / err * ddy;
            double Xv[3] = {X[j], Y[j], Z[j]};
            double v9[9];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                v9[k] = dN0 * (-f * Xv[k] / ez);
                v9[3 + k] = dN1 * (f * Xv[k] / ez);
                v9[6 + k] = dN0 * (f * ex / ez / ez * Xv[k]) + dN1 * (-f * ey / ez / ez * Xv[k]);
            }
#pragma unroll
            for (int m = 0; m < 3; m++) {
                double s = 0;
#pragma unroll
                for (int k = 0; k < 9; k++) s += v9[k] * J[m * 9 + k];
                w6[m] += g * s;
            }
            w6[3] += g * (dN0 * (-f / ez));
            w6[4] += g * (dN1 * (f / ez));
            w6[5] += g * (dN0 * (f * ex / ez / ez) + dN1 * (-f * ey / ez / ez));
        }
        // sum_i g * dProjectdHyp  (1x6) over the 1600 points
#pragma unroll
        for (int k = 0; k < 6; k++) {
            double v = w6[k];
#pragma unroll
            for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
            if (lane == 0) s_red[warp][k] = v;
        }
        __syncthreads();
        if (tid < 6) {
            double v = 0;
            for (int w = 0; w < K5_WARPS; w++) v += s_red[w][tid];
            s_w[tid] = v;
        }
        __syncthreads();
        // supportPointGradients = w . dPNP_h (1x12) onto the 4 support cells (cnn_softam.h:632-642)
        if constexpr (RIG) {
            if (tid < 6) rig.w[((size_t)frame * p.H + h) * 6 + tid] = s_w[tid];
        } else if (tid < 12) {
            const double* Jp = p.s.dpnp + ((size_t)frame * p.H + h) * 72;
            double s = 0;
            for (int k = 0; k < 6; k++) s += s_w[k] * Jp[k * 12 + tid];
            int c = p.img_idx[((size_t)frame * p.H + h) * 4 + tid / 3];
            if (c >= 0) {
                int x = c % DSAC_GRID_CONST, y = c / DSAC_GRID_CONST;
                int colb = p.fix_q4 ? (y * DSAC_GRID_CONST + x) * 3 : (x * DSAC_GRID_CONST + y) * 3;   // quirk Q4
                row[colb + tid % 3] += s;   // 12 distinct addresses; ordered by the barriers of the h loop
            }
        }
    }
    __syncthreads();
    // direct part: column of point (x,y) -- x-major in the reference (quirk Q4, cnn_softam.h:628)
#pragma unroll
    for (int j = 0; j < K5_PTS; j++) {
        int pt = tid + j * K5_THREADS;
        int x = pt % DSAC_GRID_CONST, y = pt / DSAC_GRID_CONST;
        int colb = p.fix_q4 ? pt * 3 : (x * DSAC_GRID_CONST + y) * 3;
        for (int k = 0; k < 3; k++) row[colb + k] += acc[j][k];
    }
}
__global__ void __launch_bounds__(K5_THREADS) k_dscore(BwParams p) { k_dscore_body<false>(p, RigDscore{}); }
__global__ void __launch_bounds__(K5_THREADS) k_dscore_rig(BwParams p, RigDscore rig) { k_dscore_body<true>(p, rig); }

// ------------------------------------------------------------------ implicit-function derivatives (DSAC_DERIV_IMPLICIT)
// dRefine / dObj of a refined pose: the IFT of the last accepted refinement step's fit over the cells it fitted (ift.cuh),
// one CTA per refined pose (job).  The lanes own the recorded cells; the 21 Hessian entries are reduced with the transposed
// butterfly of k_refine's normal_equations_pass, one lane factors and solves in fp64, then every lane writes its cells.
struct IftParams {
    const int16_t* coords;      // [n][N][3]
    const int32_t* pix;
    int pix_stride;
    double f, cx, cy;
    const Cam* cams;            // [n] or null
    const double* eye;          // [n][N][3] (RGB-D) or null
    const int32_t* job_frame;   // [jobs] frame, -1 unused; null: job j -> frame j
    const double* pose;         // [jobs][6] cv pose the recording replay ended with
    const uint16_t* sel;        // [jobs][K4_MAX_INLIERS] cells of its last accepted step
    const int32_t* count;       // [jobs] their number, 0: no step accepted
    const double* seed;         // [jobs][6] dOuter / d(refined jp6)
    double* row;                // [n][N*3] += seed . dRefine/dObj (distinct cells per job), or null
    double* drefobj;            // [n][6][N*3] dRefine/dObj, or null
    double* contrib;            // [jobs][K4_MAX_INLIERS][3] seed . dRefine/dObj per recorded cell, or null
};
constexpr int IFT_THREADS = 64, IFT_WARPS = IFT_THREADS / 32;

// the soft-argmax backward's recording replay (one job per frame), in dsac_engine::ift_buf
struct IftScratch {
    double* pose = nullptr;      // [n][6]
    uint16_t* sel = nullptr;     // [n][K4_MAX_INLIERS]
    int32_t* count = nullptr;    // [n]
};

// RIG (k_refine_ift_rig, the rig backward): job r is rig r of rig.C cameras, pose the rig's, sel entries cam << 11 | cell
// at a stride of C K4_MAX_INLIERS (k_refine_rig_rec).  A cell is set up in its own camera frame and mapped to the rig frame
// (ift_point_to_rig); its row is its camera frame's, and drefobj is [R][6][C N 3], camera-major.  RIG with RGBD
// (k_refine_ift_rig_rgbd, RGB-D rigs): the residual is the cell's in its own camera frame, against its eye point.
template <bool PER_FRAME, bool RGBD, bool RIG = false>
__device__ __forceinline__ void k_refine_ift_body(const IftParams& p, RigRefine rig = RigRefine{}) {
    __shared__ double s_red[IFT_WARPS][32];
    __shared__ double s_W[36], s_v[6];
    __shared__ int s_ok;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int job = blockIdx.x;
    const int frame = p.job_frame ? p.job_frame[job] : job;
    if (frame < 0) return;
    const Cam cam = frame_cam<PER_FRAME>(p, frame);
    const int cnt = p.count[job];
    const int n_cams = RIG ? rig.C : 1;
    const size_t width = (size_t)n_cams * DSAC_N_CONST * 3;   // row / drefobj columns of a job
    const uint16_t* sel = p.sel + (size_t)job * n_cams * K4_MAX_INLIERS;
    const int16_t* coords = p.coords + (size_t)frame * DSAC_N_CONST * 3;
    const int32_t* pix = p.pix + (size_t)frame * p.pix_stride;
    double pose[6], R[9];
    for (int k = 0; k < 6; k++) pose[k] = p.pose[(size_t)job * 6 + k];
    rodrigues_v2m(pose, R);
    auto point = [&](int i, IftPoint& P) {
        if constexpr (RIG) {
            const int code = sel[i], fr = frame * n_cams + (code >> 11), cell = code & 2047;
            const int16_t* co = p.coords + ((size_t)fr * DSAC_N_CONST + cell) * 3;
            const int32_t* px = p.pix + (size_t)fr * p.pix_stride + cell * 2;
            const double Y[3] = {(double)co[0], (double)co[1], (double)co[2]};
            double e[3] = {(double)px[0], (double)px[1], 0};
            if constexpr (RGBD) {
                const double* ey = p.eye + ((size_t)fr * DSAC_N_CONST + cell) * 3;
                e[0] = ey[0]; e[1] = ey[1]; e[2] = ey[2];
            }
            const double* E = rig.ext + (size_t)fr * 12;
            double Rk[9], tk[3];
            rig_compose(E, E + 9, R, pose + 3, Rk, tk);
            const Cam cm = frame_cam<PER_FRAME>(p, fr);
            ift_point_setup(Rk, tk, Y, e, cm.f, cm.cx, cm.cy, RGBD, P);
            ift_point_to_rig(E, P);
            return;
        }
        const int c = sel[i];
        const double Y[3] = {(double)coords[c * 3], (double)coords[c * 3 + 1], (double)coords[c * 3 + 2]};
        double e[3];
        if constexpr (RGBD) {
            const double* ey = p.eye + ((size_t)frame * DSAC_N_CONST + c) * 3;
            e[0] = ey[0]; e[1] = ey[1]; e[2] = ey[2];
        } else {
            e[0] = (double)pix[c * 2]; e[1] = (double)pix[c * 2 + 1]; e[2] = 0;
        }
        ift_point_setup(R, pose + 3, Y, e, cam.f, cam.cx, cam.cy, RGBD, P);
    };
    // Hessian: per-lane sums, then the transposed butterfly (lane L ends with entry L), then the warps in order
    double v[32];
#pragma unroll
    for (int k = 0; k < 32; k++) v[k] = 0;
    for (int i = tid; i < cnt; i += IFT_THREADS) {
        IftPoint P;
        point(i, P);
        ift_point_hess(P, v);
    }
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
    __syncthreads();
    if (tid == 0) {
        double U[21], M[36], Rm[9];
        for (int k = 0; k < 21; k++) {
            double t = 0;
            for (int w = 0; w < IFT_WARPS; w++) t += s_red[w][k];
            U[k] = t;
        }
        bool ok = cnt > 0 && ift_chol6(U);
        if (ok) {
            ift_jp_jacobian(pose, Rm, M);
            ift_weights(U, M, s_W);
            for (int a = 0; a < 6; a++) {
                double t = 0;
                for (int k = 0; k < 6; k++) t += s_W[a * 6 + k] * p.seed[(size_t)job * 6 + k];
                s_v[a] = t;
                ok = ok && t - t == 0.0;
            }
            for (int k = 0; k < 36; k++) ok = ok && s_W[k] - s_W[k] == 0.0;
        }
        s_ok = ok ? 1 : 0;
    }
    __syncthreads();
    const bool ok = s_ok != 0;
    double* row = p.row ? p.row + (size_t)frame * width : nullptr;
    for (int i = tid; i < cnt; i += IFT_THREADS) {
        const int c = RIG ? (sel[i] >> 11) * DSAC_N_CONST + (sel[i] & 2047) : sel[i];   // column / 3 within the job's width
        double o[3] = {0, 0, 0};
        if (ok) {
            IftPoint P;
            double B[18];
            point(i, P);
            ift_point_cross(P, R, B);
            for (int j = 0; j < 3; j++) {
                double t = 0;
                for (int a = 0; a < 6; a++) t += s_v[a] * B[a * 3 + j];
                o[j] = -t;
            }
            if (p.drefobj) {
                double D[18];
                ift_point_deriv(s_W, B, D);
                for (int k = 0; k < 6; k++)
                    for (int j = 0; j < 3; j++) p.drefobj[((size_t)frame * 6 + k) * width + c * 3 + j] = D[k * 3 + j];
            }
        }
        for (int j = 0; j < 3; j++) {
            if (row) row[c * 3 + j] += o[j];
            if (p.contrib) p.contrib[((size_t)job * K4_MAX_INLIERS + i) * 3 + j] = o[j];
        }
    }
}
__global__ void __launch_bounds__(IFT_THREADS) k_refine_ift(IftParams p) { k_refine_ift_body<false, false>(p); }
__global__ void __launch_bounds__(IFT_THREADS) k_refine_ift_cam(IftParams p) { k_refine_ift_body<true, false>(p); }
__global__ void __launch_bounds__(IFT_THREADS) k_refine_ift_rgbd(IftParams p) { k_refine_ift_body<false, true>(p); }
__global__ void __launch_bounds__(IFT_THREADS) k_refine_ift_rgbd_cam(IftParams p) { k_refine_ift_body<true, true>(p); }
__global__ void __launch_bounds__(IFT_THREADS) k_refine_ift_rig(IftParams p, RigRefine rig) { k_refine_ift_body<false, false, true>(p, rig); }
__global__ void __launch_bounds__(IFT_THREADS) k_refine_ift_rig_cam(IftParams p, RigRefine rig) { k_refine_ift_body<true, false, true>(p, rig); }
__global__ void __launch_bounds__(IFT_THREADS) k_refine_ift_rig_rgbd(IftParams p, RigRefine rig) { k_refine_ift_body<false, true, true>(p, rig); }
__global__ void __launch_bounds__(IFT_THREADS) k_refine_ift_rig_rgbd_cam(IftParams p, RigRefine rig) { k_refine_ift_body<true, true, true>(p, rig); }
// [per-frame camera][RGB-D]
constexpr void (*k_refine_ift_rig_tab[2][2])(IftParams, RigRefine) = {{k_refine_ift_rig, k_refine_ift_rig_rgbd},
                                                                     {k_refine_ift_rig_cam, k_refine_ift_rig_rgbd_cam}};

inline void launch_refine_ift(const IftParams& p, unsigned jobs, cudaStream_t stream) {
    // [per-frame camera][RGB-D]
    constexpr void (*tab[2][2])(IftParams) = {{k_refine_ift, k_refine_ift_rgbd}, {k_refine_ift_cam, k_refine_ift_rgbd_cam}};
    tab[p.cams != nullptr][p.eye != nullptr]<<<jobs, IFT_THREADS, 0, stream>>>(p);
}

// jp pose + Rodrigues Jacobian of hypothesis h for k_dscore, as k_dpnp / k_dkabsch write it
__device__ __forceinline__ void write_hypjp(const BwParams& p, int frame, int h) {
    double* hj = p.s.hypjp + ((size_t)frame * p.H + h) * 39;
    double R[9], t[3], rod[3], Rt[9], J[27];
    cv2our_dev(p.hyp_pose + ((size_t)frame * p.H + h) * 6, R, t);
    rodrigues_m2v(R, rod);
    rodrigues_jac(rod, Rt, J);
    for (int k = 0; k < 9; k++) hj[k] = R[k];
    for (int k = 0; k < 3; k++) hj[9 + k] = t[k];
    for (int k = 0; k < 27; k++) hj[12 + k] = J[k];
}

// ---- dPNP by the IFT of the P3P equations at the hypothesis' pose (ift_dpnp_p3p): thread = (hypothesis, column 0..11) as
// in k_dpnp, one 6x6 solve per column; a singular system or a non-finite column zeroes the hypothesis.
__global__ void __launch_bounds__(192) k_dpnp_ift(BwParams p) {
    const int frame = blockIdx.y;
    const int h = blockIdx.x * 16 + threadIdx.x / 12, col = threadIdx.x % 12;
    __shared__ int s_bad[16];
    if (threadIdx.x < 16) s_bad[threadIdx.x] = 0;
    __syncthreads();
    const bool active = h < p.H;
    double out[72];
    bool ok = true;
    if (active && col < 9) {
        const int16_t* coords = p.coords + (size_t)frame * DSAC_N_CONST * 3;
        const int32_t* pix = p.pix + (size_t)frame * p.pix_stride;
        const int32_t* idx = p.img_idx + ((size_t)frame * p.H + h) * 4;
        double X[9], uv[6];
        for (int j = 0; j < 3; j++) {
            int c = idx[j];
            if (c < 0) { ok = false; c = 0; }
            for (int k = 0; k < 3; k++) X[j * 3 + k] = (double)coords[c * 3 + k];
            uv[j * 2] = (double)pix[c * 2]; uv[j * 2 + 1] = (double)pix[c * 2 + 1];
        }
        const Cam cam = frame_cam(p, frame);
        ok = ok && ift_dpnp_p3p(p.hyp_pose + ((size_t)frame * p.H + h) * 6, X, uv, cam.f, cam.cx, cam.cy, out, col);
        if (!ok) s_bad[threadIdx.x / 12] = 1;
    }
    __syncthreads();
    if (active) {
        const bool zero = s_bad[threadIdx.x / 12] != 0 || col >= 9;
        double* o = p.s.dpnp + ((size_t)frame * p.H + h) * 72;
        for (int k = 0; k < 6; k++) o[k * 12 + col] = zero ? 0.0 : out[k * 12 + col];
        if (col == 0) write_hypjp(p, frame, h);
    }
}

// ---- dPNP of an RGB-D pass by the IFT of the 3-point Kabsch fit (ift_dpnp_kabsch); grid and zero rule of k_dpnp_ift
__global__ void __launch_bounds__(192) k_dkabsch_ift(BwParams p, const double* __restrict__ eye) {
    const int frame = blockIdx.y;
    const int h = blockIdx.x * 16 + threadIdx.x / 12, col = threadIdx.x % 12;
    __shared__ int s_bad[16];
    if (threadIdx.x < 16) s_bad[threadIdx.x] = 0;
    __syncthreads();
    const bool active = h < p.H;
    double out[72];
    bool ok = true;
    if (active && col < 9) {
        const int16_t* coords = p.coords + (size_t)frame * DSAC_N_CONST * 3;
        const double* ey = eye + (size_t)frame * DSAC_N_CONST * 3;
        const int32_t* idx = p.img_idx + ((size_t)frame * p.H + h) * 4;
        double a[9], b[9];
        for (int j = 0; j < 3; j++) {
            int c = idx[j];
            if (c < 0) { ok = false; c = 0; }
            for (int k = 0; k < 3; k++) { a[j * 3 + k] = (double)coords[c * 3 + k]; b[j * 3 + k] = ey[c * 3 + k]; }
        }
        ok = ok && ift_dpnp_kabsch(a, b, out);
        if (!ok) s_bad[threadIdx.x / 12] = 1;
    }
    __syncthreads();
    if (active) {
        const bool zero = s_bad[threadIdx.x / 12] != 0 || col >= 9;
        double* o = p.s.dpnp + ((size_t)frame * p.H + h) * 72;
        for (int k = 0; k < 6; k++) o[k * 12 + col] = zero ? 0.0 : out[k * 12 + col];
        if (col == 0) write_hypjp(p, frame, h);
    }
}

// ---- DSAC variant, implicit: the seed of selected hypothesis s, sf_h dLossMax(refined_h, gt) or the caller's seed_h, in
// w [n H][6]; threads past the selection exit
__global__ void k_dsac_ift_seed(DsacBwParams p, const int32_t* __restrict__ sel, const int32_t* __restrict__ sel_frame,
                                const int32_t* __restrict__ totals, double* __restrict__ w) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= totals[0]) return;
    const int g = sel[s];
    if (p.seed) {
        for (int k = 0; k < 6; k++) w[(size_t)s * 6 + k] = p.seed[(size_t)g * 6 + k];
        return;
    }
    const double* gj = p.gt_jp + (size_t)sel_frame[s] * 12;
    double gt6[6], ref6[6], dl[6];
    rodrigues_m2v(gj, gt6);
    gt6[3] = gj[9]; gt6[4] = gj[10]; gt6[5] = gj[11];
    jp6_from_cv_dev(p.ref_pose + (size_t)g * 6, ref6);
    dloss_max_dev(ref6, gt6, dl);
    for (int k = 0; k < 6; k++) w[(size_t)s * 6 + k] = p.sf[g] * dl[k];
}

// ---- DSAC variant, implicit: path1 += the selected hypotheses' recorded-cell contributions (k_refine_ift's contrib), one
// warp per frame, hypotheses in selection order (a hypothesis' cells are distinct, so its lanes add independently); the
// support cells are skipped, as job_cell skips them in central mode.  No atomics: the same call gives the same bits.
__global__ void __launch_bounds__(32) k_dsac_ift_combine(DsacBwParams p, const int32_t* __restrict__ sel, const int32_t* __restrict__ sel_begin,
                                                         const uint16_t* __restrict__ rec_sel, const int32_t* __restrict__ rec_count,
                                                         const double* __restrict__ contrib) {
    const int frame = blockIdx.x, lane = threadIdx.x;
    if (frame >= p.n_frames) return;
    double* row = p.path1 + (size_t)frame * DSAC_N_CONST * 3;
    for (int s = sel_begin[frame]; s < sel_begin[frame + 1]; s++) {
        const int32_t* cells = p.img_idx + (size_t)sel[s] * 4;
        const int cnt = rec_count[s];
        for (int i = lane; i < cnt; i += 32) {
            const int c = rec_sel[(size_t)s * K4_MAX_INLIERS + i];
            if (c == cells[0] || c == cells[1] || c == cells[2] || c == cells[3]) continue;
            for (int j = 0; j < 3; j++) row[c * 3 + j] += contrib[((size_t)s * K4_MAX_INLIERS + i) * 3 + j];
        }
        __syncwarp();
    }
}

// ---- batched Kabsch (Hypothesis::calcRigidBodyTransform, Hypothesis.cpp:145-200): thread = problem (kabsch_fit, rigid.cuh).
__global__ void k_kabsch(int n, int m, const double* __restrict__ a, const double* __restrict__ b, double* R, double* t) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double Ro[9], to[3];
    kabsch_fit(m, a + (size_t)i * m * 3, b + (size_t)i * m * 3, Ro, to);
    for (int k = 0; k < 9; k++) R[(size_t)i * 9 + k] = Ro[k];
    for (int r = 0; r < 3; r++) t[(size_t)i * 3 + r] = to[r];
}

}  // namespace dsac

int backward_run(dsac_engine* e, int32_t n, const int16_t* coords, const int32_t* pix, int32_t pix_shared,
                 const double* gt_jp, dsac_backward_out* out);
// d_seed: [n][6] dOuter/d(refined jp6) in place of dLossMax (the ground truth is then not needed); null: dLossMax
int backward_device_run(dsac_engine* e, int32_t n, const double* d_loss_grad, double* d_dloss_dobj, float* d_dloss_dpred,
                        float clamp, cudaStream_t stream, const double* d_seed = nullptr);
int kabsch_run(dsac_engine* e, int32_t n, int32_t m, const double* a, const double* b, double* R, double* t);
struct dsac_backward_dsac_out;
// seeded: path I from d_seed [n][H][6] in place of sf_h dLossMax_h, path II from d_grad_sf [n][H] in place of the
// losses; a null seed skips its path, and the ground truth is not needed
int backward_dsac_run(dsac_engine* e, int32_t n, const double* d_loss_grad, const dsac_backward_dsac_out* out, bool out_on_host,
                      float* d_dloss_dpred, float clamp, cudaStream_t stream, bool seeded = false,
                      const double* d_seed = nullptr, const double* d_grad_sf = nullptr);
