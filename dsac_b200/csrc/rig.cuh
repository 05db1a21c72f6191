// rig.cuh -- multi-camera rigs (dsac_forward_rig_device): the pool of rig poses lifted from every camera's hypotheses,
// its projection rows in every camera, and the per-rig score sum and softmax tail.
//
// A rig pass covers n frames as R = n / C rigs of C cameras; frame f = r C + c is camera c of rig r, with the extrinsic
// X_cam = Rc X_rig + tc.  The sampler runs on the frames as in an ordinary pass.  Then:
//   k_rig_lift   the extrinsics (Rc, tc), the rig status, the pool -- slot j = c H + h of rig r is camera c's hypothesis h
//                lifted to the rig frame -- and the fp32 rows of every pool pose in every camera of its rig;
//   k_score_rig  (k_score without its softmax tail) every camera frame against its rig's pool of P = C H poses; with the
//                rig score hooks it writes the error images [n][P][N] too and the forward hook replaces its scores;
//   k_rig_tail   the rig's score of slot j is the sum of its cameras' scores in camera order, then softargmax_tail;
//   k_refine_rig the refinement of the soft-argmax rig pose over all cameras' cells (refine.cuh).
// The rig backward (dsac_backward_rig_device, rig_backward_host.inc) is the soft-argmax backward's implicit chain over the
// pool: k_bw_prep_implicit, k_refine_rig_rec and the 12 dRefineHyp jobs of k_refine_rig, k_bw_combine_implicit and
// k_refine_ift_rig per rig; k_dpnp_ift per frame; then
//   k_rig_bw_hypjp    the composed pose T_c o T_j of every (frame, slot) in jp with its Rodrigues Jacobian;
//   k_dscore_rig      every camera frame against its rig's pool: the direct part into the frame's row, w per (frame, slot)
//                     (after a hooked pass k_rig_clamp_broadcast and the backward hook first, whose dScore/dDiffMap it reads);
//   k_rig_bw_support  per (frame, hypothesis) the 1x6 of path I (dLdAvg L_j) and of path II (sum_c w K_c,j);
//   k_rig_bw_scatter  per frame, hypotheses in order: both through dPNP onto the minimal set's cells.
#pragma once
#include <cuda_runtime.h>

#include "backward.cuh"
#include "camera.cuh"
#include "ift.cuh"
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
    const double* prior_pose;       // [R][prior_k][6] the rig pose priors (dsac_set_rig_pose_priors_device), or null
    int prior_k;                    // 0: none
};

// Grid (ceil(P / 256), R): thread j of rig r lifts pool slot j and writes its rows in each camera of the rig.  A rig with a
// non-finite extrinsic gets DSAC_ST_BAD_RIG and zero pool poses (its rows stay finite; k_rig_tail zeroes its scores), and so
// does a rig whose frames carry DSAC_ST_BAD_PRIOR (a bad rig prior, k_rig_prior_prep).  An extrinsic whose rvec is exactly
// zero has Rc = I exactly (rodrigues_v2m), so the lift is exact and the hypothesis keeps its rvec bits rather than a round
// trip through the matrix.  With rig priors, camera c's prior slot H - k + j is pool slot c H + H - k + j and takes rig
// prior j's own bits, so the pool holds C copies of each prior.
__global__ void __launch_bounds__(RIG_LIFT_THREADS) k_rig_lift(RigLiftParams p) {
    __shared__ double s_ext[RIG_MAX_CAMERAS][12];
    __shared__ int s_ident[RIG_MAX_CAMERAS];
    __shared__ int s_bad;
    __shared__ uint32_t s_st;
    const int tid = threadIdx.x, r = blockIdx.y, C = p.C, P = C * p.H;
    if (tid == 0) {
        s_bad = 0;
        uint32_t st = 0;
        for (int c = 0; c < C; c++) st |= p.frame_status[r * C + c];
        s_st = st;
    }
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
    const bool bad = s_bad != 0 || (s_st & RIG_ST_SPOILED) != 0;
    if (blockIdx.x == 0) {
        if (tid < C)
            for (int k = 0; k < 12; k++) p.ext[(size_t)(r * C + tid) * 12 + k] = s_ext[tid][k];
        if (tid == 0) p.status[r] = s_st | (s_bad ? RIG_ST_BAD : 0u);
    }
    const int j = blockIdx.x * RIG_LIFT_THREADS + tid;
    if (j >= P) return;
    const int c = j / p.H, h = j - c * p.H, hk = h - (p.H - p.prior_k);
    double Rr[9], tr[3], rr[3];
    if (hk >= 0 && !bad) {   // a prior slot: the rig prior itself
        const double* pp = p.prior_pose + ((size_t)r * p.prior_k + hk) * 6;
        for (int k = 0; k < 3; k++) { rr[k] = pp[k]; tr[k] = pp[3 + k]; }
        rodrigues_v2m(rr, Rr);
    } else {
        double hp[6] = {0, 0, 0, 0, 0, 0};
        if (!bad)
            for (int k = 0; k < 6; k++) hp[k] = p.hyp_pose[((size_t)(r * C + c) * p.H + h) * 6 + k];
        double Rh[9];
        rodrigues_v2m(hp, Rh);
        rig_lift(s_ext[c], s_ext[c] + 9, Rh, hp + 3, Rr, tr);
        if (s_ident[c]) {
            rr[0] = hp[0]; rr[1] = hp[1]; rr[2] = hp[2];
        } else {
            rodrigues_m2v(Rr, rr);
        }
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
    const bool bad = (p.status[r] & RIG_ST_SPOILED) != 0;
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

struct RigBwParams {
    int C, H, P, fix_q4;
    const double* ext;          // [n][12] Rc (row-major), tc (k_rig_lift)
    const double* rig_hyp;      // [R][P][6] the pool (cv)
    const double* hyp_pose;     // [n][H][6] the frames' hypotheses (cv)
    const int32_t* img_idx;     // [n][H][4]
    const double* sf;           // [R][P]
    const uint32_t* status;     // [R]
    const double* dldavg;       // [R][6] dLoss/dAvg (k_bw_combine_implicit)
    const double* dpnp;         // [n][H][72] (k_dpnp_ift)
    const double* w;            // [n][P][6] (k_dscore_rig)
    double* hypjp;              // [n][P][39]
    double* u;                  // [n][H][12] the two 1x6 of each hypothesis' support scatter
    double* row;                // [n][N * 3]
};
constexpr int RIG_BW_THREADS = 128;

// Grid (ceil(P / 128), n): camera frame f's pose of pool slot j, T_c o T_j, as k_dscore reads a hypothesis (write_hypjp):
// R, t of cv2our and the Rodrigues Jacobian at its rotation vector.  An identity extrinsic changes no bit (rig_compose),
// so with C = 1 this is write_hypjp's output.
__global__ void __launch_bounds__(RIG_BW_THREADS) k_rig_bw_hypjp(RigBwParams p) {
    const int j = blockIdx.x * RIG_BW_THREADS + threadIdx.x, f = blockIdx.y;
    if (j >= p.P) return;
    const double* hp = p.rig_hyp + ((size_t)(f / p.C) * p.P + j) * 6;
    const double* E = p.ext + (size_t)f * 12;
    double Rr[9], R[9], t[3], rod[3], Rt[9], J[27];
    rodrigues_v2m(hp, Rr);
    rig_compose(E, E + 9, Rr, hp + 3, R, t);
    // cv2our_dev on the composed pose
    t[1] = -t[1]; t[2] = -t[2];
    for (int k = 3; k < 9; k++) R[k] = -R[k];
    const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) + R[2] * (R[3] * R[7] - R[4] * R[6]);
    if (det < 0) {
        for (int k = 0; k < 9; k++) R[k] = -R[k];
        for (int k = 0; k < 3; k++) t[k] = -t[k];
    }
    if (t[0] != t[0] || t[1] != t[1] || t[2] != t[2]) t[0] = t[1] = t[2] = 0;
    rodrigues_m2v(R, rod);
    rodrigues_jac(rod, Rt, J);
    double* hj = p.hypjp + ((size_t)f * p.P + j) * 39;
    for (int k = 0; k < 9; k++) hj[k] = R[k];
    for (int k = 0; k < 3; k++) hj[9 + k] = t[k];
    for (int k = 0; k < 27; k++) hj[12 + k] = J[k];
}

// Grid (ceil(H / 128), n): hypothesis h of frame f' = r C + c' (pool slot j = c' H + h) moves, through its minimal set, the
// pool pose j.  Path I's 1x6 is dLdAvg_r L_j (the slot's sf_j is applied in the scatter, as k_bw_scatter_pnp applies it),
// path II's sum over the rig's cameras c of w[r C + c][j] K_c,j (rig_lift_jac, rig_cross_jac in ift.cuh).  A bad rig's are
// zero.
__global__ void __launch_bounds__(RIG_BW_THREADS) k_rig_bw_support(RigBwParams p) {
    const int h = blockIdx.x * RIG_BW_THREADS + threadIdx.x, f = blockIdx.y;
    if (h >= p.H) return;
    const int C = p.C, r = f / C, c2 = f - r * C, j = c2 * p.H + h;
    double* u = p.u + ((size_t)f * p.H + h) * 12;
    if (p.status[r] & RIG_ST_SPOILED) {
        for (int k = 0; k < 12; k++) u[k] = 0.0;
        return;
    }
    const double* hp = p.hyp_pose + ((size_t)f * p.H + h) * 6;
    const double* E2 = p.ext + (size_t)f * 12;
    double M[36], Rh[9], o[12];
    rig_lift_jac(E2, hp, M);
    const double* dld = p.dldavg + (size_t)r * 6;
    for (int m = 0; m < 6; m++) {
        double s = 0;
        for (int k = 0; k < 6; k++) s += dld[k] * M[k * 6 + m];
        o[m] = s;
        o[6 + m] = 0;
    }
    rodrigues_v2m(hp, Rh);
    for (int c = 0; c < C; c++) {
        rig_cross_jac(p.ext + (size_t)(r * C + c) * 12, E2, Rh, c == c2, M);
        const double* w = p.w + ((size_t)(r * C + c) * p.P + j) * 6;
        for (int m = 0; m < 6; m++) {
            double s = 0;
            for (int k = 0; k < 6; k++) s += w[k] * M[k * 6 + m];
            o[6 + m] += s;
        }
    }
    for (int k = 0; k < 12; k++) u[k] = o[k];
}

// One warp per frame f': its hypotheses in order, lanes 0..11 = (point, channel) of the minimal set, dPNP applied to
// both 1x6 of k_rig_bw_support -- path I onto the cells as k_bw_scatter_pnp puts them, path II in the layout of quirk
// Q4 as k_dscore's support scatter (fix_q4) -- with no atomics, so the rows are run-to-run identical.  Last in the chain:
// it zeroes the rows of a bad rig's frames.
__global__ void __launch_bounds__(32) k_rig_bw_scatter(RigBwParams p) {
    const int f = blockIdx.x, lane = threadIdx.x, r = f / p.C, c2 = f - r * p.C;
    double* row = p.row + (size_t)f * DSAC_N_CONST * 3;
    if (p.status[r] & RIG_ST_SPOILED) {
        for (int i = lane; i < DSAC_N_CONST * 3; i += 32) row[i] = 0.0;
        return;
    }
    if (lane >= 12) return;
    for (int h = 0; h < p.H; h++) {
        const size_t fh = (size_t)f * p.H + h;
        const int c = p.img_idx[fh * 4 + lane / 3];
        const double* J = p.dpnp + fh * 72;
        const double* u = p.u + fh * 12;
        const double sf = p.sf[(size_t)r * p.P + c2 * p.H + h];
        double s1 = 0, s2 = 0;
        for (int k = 0; k < 6; k++) s1 += u[k] * (sf * J[k * 12 + lane]);
        for (int k = 0; k < 6; k++) s2 += u[6 + k] * J[k * 12 + lane];
        if (c >= 0) row[c * 3 + lane % 3] += s1;
        __syncwarp(0xfff);
        if (c >= 0) {
            const int x = c % DSAC_GRID_CONST, y = c / DSAC_GRID_CONST;
            row[(p.fix_q4 ? c : x * DSAC_GRID_CONST + y) * 3 + lane % 3] += s2;   // quirk Q4
        }
        __syncwarp(0xfff);
    }
}

// A hooked rig pass (dsac_set_rig_score_hooks): the rig's score output gradients sog [R][P] clamped to +-clamp, as
// k_clamp_copy clamps an ordinary pass's, and given to every camera frame of the rig [n][P] -- the rig score is the sum of
// its cameras' scores, so d(rig score) / d(camera score) = 1 -- the input of the rig score backward hook
__global__ void k_rig_clamp_broadcast(const double* __restrict__ sog, int C, int P, size_t count, double clamp, double* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const size_t f = i / P, j = i - f * P;
    double v = sog[(f / C) * P + j];
    if (clamp > 0) v = fmax(-clamp, fmin(clamp, v));
    out[i] = v;
}

// the per-rig loss gradient [R] read per frame [n], as k_e2e_grad indexes it
__global__ void k_rig_frame_grad(const double* __restrict__ g, int C, int n, double* __restrict__ out) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < n) out[f] = g[f / C];
}

}  // namespace dsac
