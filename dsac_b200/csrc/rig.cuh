// rig.cuh -- multi-camera rigs (dsac_forward_rig_device): the pool of rig poses lifted from every camera's hypotheses,
// its projection rows in every camera, and the per-rig score sum and softmax tail.
//
// A rig pass covers n frames as R = n / C rigs of C cameras; frame f = r C + c is camera c of rig r, with the extrinsic
// X_cam = Rc X_rig + tc.  The sampler runs on the frames as in an ordinary pass.  Then:
//   k_rig_lift   the extrinsics (Rc, tc), the rig status, the pool -- slot j = c H + h of rig r is camera c's hypothesis h
//                lifted to the rig frame -- and the fp32 rows of every pool pose in every camera of its rig;
//   k_score_rig  (k_score without its softmax tail) every camera frame against its rig's pool of P = C H poses;
//   k_rig_tail   the rig's score of slot j is the sum of its cameras' scores in camera order, then softargmax_tail;
//   k_refine_rig the refinement of the soft-argmax rig pose over all cameras' cells (refine.cuh).
#pragma once
#include <cuda_runtime.h>

#include "camera.cuh"
#include "kernels.cuh"
#include "pose_math.cuh"
#include "refine.cuh"

namespace dsac {

constexpr int RIG_LIFT_THREADS = 256;

struct RigLiftParams {
    int C, H;                       // cameras per rig, hypotheses per frame; the pool holds P = C H
    const double* cam_from_rig;     // [n][6] cv poses (rvec, tvec mm)
    const double* hyp_pose;         // [n][H][6] the frames' hypotheses
    const uint32_t* frame_status;   // [n] the sampler's status bits
    double f;                       // the config's focal length
    const Cam* cams;                // [n] or null
    double* ext;                    // [n][12] Rc (row-major), tc
    double* rig_hyp;                // [R][P][6] the pool's rig poses
    float* rig_P;                   // [n][P][12] rows of pool pose j in camera frame f
    uint32_t* status;               // [R]
};

// Grid (ceil(P / 256), R): thread j of rig r lifts pool slot j and writes its rows in each camera of the rig.  A rig with a
// non-finite extrinsic gets DSAC_ST_BAD_RIG and zero pool poses (its rows stay finite; k_rig_tail zeroes its scores).  An
// extrinsic whose rvec is exactly zero has Rc = I exactly (rodrigues_v2m), so the lift is exact and the hypothesis keeps
// its rvec bits rather than a round trip through the matrix.
__global__ void __launch_bounds__(RIG_LIFT_THREADS) k_rig_lift(RigLiftParams p) {
    __shared__ double s_ext[RIG_MAX_CAMERAS][12];
    __shared__ int s_ident[RIG_MAX_CAMERAS];
    __shared__ int s_bad;
    const int tid = threadIdx.x, r = blockIdx.y, C = p.C, P = C * p.H;
    if (tid == 0) s_bad = 0;
    __syncthreads();
    if (tid < C) {
        const double* e = p.cam_from_rig + (size_t)(r * C + tid) * 6;
        double v[6];
        bool ok = true;
        for (int k = 0; k < 6; k++) {
            v[k] = e[k];
            ok = ok && isfinite(v[k]);
        }
        if (!ok) s_bad = 1;
        if (!ok)
            for (int k = 0; k < 6; k++) v[k] = 0.0;
        double R[9];
        rodrigues_v2m(v, R);
        for (int k = 0; k < 9; k++) s_ext[tid][k] = R[k];
        for (int k = 0; k < 3; k++) s_ext[tid][9 + k] = v[3 + k];
        s_ident[tid] = v[0] == 0.0 && v[1] == 0.0 && v[2] == 0.0;
    }
    __syncthreads();
    const bool bad = s_bad != 0;
    if (blockIdx.x == 0) {
        if (tid < C)
            for (int k = 0; k < 12; k++) p.ext[(size_t)(r * C + tid) * 12 + k] = s_ext[tid][k];
        if (tid == 0) {
            uint32_t st = bad ? RIG_ST_BAD : 0u;
            for (int c = 0; c < C; c++) st |= p.frame_status[r * C + c];
            p.status[r] = st;
        }
    }
    const int j = blockIdx.x * RIG_LIFT_THREADS + tid;
    if (j >= P) return;
    const int c = j / p.H, h = j - c * p.H;
    double hp[6] = {0, 0, 0, 0, 0, 0};
    if (!bad)
        for (int k = 0; k < 6; k++) hp[k] = p.hyp_pose[((size_t)(r * C + c) * p.H + h) * 6 + k];
    double Rh[9], Rr[9], tr[3], rr[3];
    rodrigues_v2m(hp, Rh);
    rig_lift(s_ext[c], s_ext[c] + 9, Rh, hp + 3, Rr, tr);
    if (s_ident[c]) {
        rr[0] = hp[0]; rr[1] = hp[1]; rr[2] = hp[2];
    } else {
        rodrigues_m2v(Rr, rr);
    }
    double* o = p.rig_hyp + ((size_t)r * P + j) * 6;
    if (bad)
        for (int k = 0; k < 6; k++) o[k] = 0.0;
    else {
        o[0] = rr[0]; o[1] = rr[1]; o[2] = rr[2]; o[3] = tr[0]; o[4] = tr[1]; o[5] = tr[2];
    }
    for (int c2 = 0; c2 < C; c2++) {
        const int fr = r * C + c2;
        double Rk[9], tk[3];
        rig_compose(s_ext[c2], s_ext[c2] + 9, Rr, tr, Rk, tk);
        pose_rows(p.cams ? p.cams[fr].f : p.f, Rk, tk, p.rig_P + ((size_t)fr * P + j) * 12);
    }
}

struct RigTailParams {
    ScoreParams sp;                 // scores, sf, hyp_pose (the pool), entropy, avg_pose per rig; H = P
    const double* cam_scores;       // [n][P] k_score's scores of each camera frame
    int C;
    const uint32_t* status;         // [R]
};

// One CTA per rig: scores[r][j] = sum over cameras c = 0 .. C-1, left to right in fp64, of cam_scores[r C + c][j], then the
// softmax / entropy / soft-argmax tail of an ordinary pass over the pool.  A bad rig gets zeros.
__global__ void __launch_bounds__(K2_THREADS) k_rig_tail(RigTailParams p) {
    __shared__ double s_red[8 * K2_WARPS];
    const int r = blockIdx.x, tid = threadIdx.x, P = p.sp.H, C = p.C;
    const bool bad = (p.status[r] & RIG_ST_BAD) != 0;
    for (int j = tid; j < P; j += K2_THREADS) {
        const double* cs = p.cam_scores + (size_t)r * C * P + j;
        double s = cs[0];
        for (int c = 1; c < C; c++) s += cs[(size_t)c * P];
        p.sp.scores[(size_t)r * P + j] = bad ? 0.0 : s;
        if (bad) p.sp.sf[(size_t)r * P + j] = 0.0;
    }
    if (bad) {
        if (tid == 0) p.sp.entropy[r] = 0.0;
        if (tid < 6) p.sp.avg_pose[(size_t)r * 6 + tid] = 0.0;
        return;
    }
    __syncthreads();
    softargmax_tail(p.sp, r, s_red);
}

}  // namespace dsac
