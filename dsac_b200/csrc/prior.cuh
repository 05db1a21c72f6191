// prior.cuh -- pose priors (dsac_set_pose_priors_device): caller poses that take the last k hypothesis slots of a frame, and
// the optional covariance gate on the sampled hypotheses.
//
//   PriorGate        one prior as the gate reads it: its rotation, translation and the Cholesky factor of its information
//   prior_cholesky   the factor from the lower triangle of a 6x6 information matrix, with the refusal of DSAC_ST_BAD_PRIOR
//   so3_angle        the angle of a rotation, atan2(|skew part|, (tr - 1) / 2)
//   so3_log          the principal log of a rotation, accurate up to and at pi
//   prior_d2         xi^T Lambda xi of a pose against one prior, xi = (log(R_h R_j^T), t_h - t_j)
//   k_prior_prep     once per setting: validates every prior of a frame, writes the gate table and the frame's bad flag
//   k_prior_inject   once per pass, after the sampler: the prior slots, or the empty frame of a bad setting
//
// The math compiles for the host as well (DSAC_HOST_ONLY): tests/host_shim/prior_shim.cpp checks it against scipy.
#pragma once
#include <math.h>
#include <stdint.h>

#include "pose_math.cuh"

namespace dsac {

constexpr int PRIOR_MAX = 16;                 // DSAC_MAX_PRIORS
constexpr uint32_t PRIOR_ST_BAD = 128u;       // DSAC_ST_BAD_PRIOR
constexpr double PRIOR_PIVOT_REL = 1e-12;     // a Cholesky pivot below this fraction of its diagonal entry is refused

struct PriorGate {
    double R[9];    // rotation of the prior (row-major, from its rvec)
    double t[3];    // translation (mm)
    double L[21];   // lower Cholesky factor of the information, by rows: L(i, j) = L[i (i + 1) / 2 + j], j <= i
};

// Lambda = L L^T from the lower triangle of info (row-major 6x6; entries above the diagonal are not read).  False when an
// entry is not finite, a diagonal entry is not > 0, or a pivot falls below PRIOR_PIVOT_REL of its diagonal entry
// (singular or indefinite).
DSAC_HD bool prior_cholesky(const double* info, double L[21]) {
    for (int i = 0; i < 6; i++) {
        for (int j = 0; j <= i; j++) {
            double s = info[i * 6 + j];
            if (!isfinite(s)) return false;
            for (int k = 0; k < j; k++) s -= L[i * (i + 1) / 2 + k] * L[j * (j + 1) / 2 + k];
            if (i == j) {
                const double a = info[i * 6 + i];
                if (!(a > 0) || !(s > PRIOR_PIVOT_REL * a)) return false;
                L[i * (i + 1) / 2 + i] = sqrt(s);
            } else {
                L[i * (i + 1) / 2 + j] = s / L[j * (j + 1) / 2 + j];
            }
        }
    }
    return true;
}

// M = A B^T of two row-major 3x3 matrices.
DSAC_HD void rot_mul_bt(const double A[9], const double B[9], double M[9]) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) M[i * 3 + j] = A[i * 3] * B[j * 3] + A[i * 3 + 1] * B[j * 3 + 1] + A[i * 3 + 2] * B[j * 3 + 2];
}

// The rotation angle th in [0, pi] of a rotation M (row-major): atan2(|v|, c), accurate everywhere, from the skew part
// v = sin(th) n and c = cos(th) = (tr - 1) / 2; also returns v, s = |v| and c.  so3_log and the pose modes' nearness test
// (modes.cuh) share it.
DSAC_HD double so3_angle(const double M[9], double v[3], double* s, double* c) {
    v[0] = 0.5 * (M[7] - M[5]); v[1] = 0.5 * (M[2] - M[6]); v[2] = 0.5 * (M[3] - M[1]);
    *s = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    *c = 0.5 * (M[0] + M[4] + M[8] - 1.0);
    return atan2(*s, *c);
}

// w = log(M), |w| <= pi, for a rotation M (row-major).  The angle is so3_angle's; the axis comes from the skew part below
// pi / 2 and from the symmetric part M + M^T = 2 c I + 2 (1 - c) n n^T above, where the skew part vanishes (its sign picks n
// against -n; at exactly pi both are the principal log).
DSAC_HD void so3_log(const double M[9], double w[3]) {
    double v[3], s, c;
    const double th = so3_angle(M, v, &s, &c);
    if (c > 0) {
        const double k = s > 0 ? th / s : 1.0;
        for (int i = 0; i < 3; i++) w[i] = k * v[i];
        return;
    }
    int i = 0;
    for (int j = 1; j < 3; j++)
        if (M[j * 4] > M[i * 4]) i = j;
    const double bii = M[i * 4] - c;   // (1 - c) n_i^2, the largest of the three
    const double sc = 1.0 / sqrt(bii * (1.0 - c));
    double n[3];
    for (int j = 0; j < 3; j++) n[j] = (j == i ? bii : 0.5 * (M[i * 3 + j] + M[j * 3 + i])) * sc;
    const double sg = (n[0] * v[0] + n[1] * v[1] + n[2] * v[2]) < 0 ? -th : th;
    for (int j = 0; j < 3; j++) w[j] = sg * n[j];
}

// d^2 = xi^T Lambda xi = |L^T xi|^2 of the pose (Rh, th) against prior g, xi = (log(Rh Rj^T) rad, th - tj mm), fp64.
DSAC_HD double prior_d2(const double Rh[9], const double th[3], const PriorGate& g) {
    double M[9];
    rot_mul_bt(Rh, g.R, M);
    double xi[6];
    so3_log(M, xi);
    for (int i = 0; i < 3; i++) xi[3 + i] = th[i] - g.t[i];
    double d2 = 0;
    for (int j = 0; j < 6; j++) {
        double y = 0;
        for (int i = j; i < 6; i++) y += g.L[i * (i + 1) / 2 + j] * xi[i];
        d2 += y * y;
    }
    return d2;
}

// The gate: the cv pose (rvec, tvec) passes iff min_j d^2_j <= chi2 over the frame's k priors.
DSAC_HD bool prior_gate_pass(const PriorGate* tab, int k, double chi2, const double rvec[3], const double tvec[3]) {
    double R[9];
    rodrigues_v2m(rvec, R);
    for (int j = 0; j < k; j++)
        if (prior_d2(R, tvec, tab[j]) <= chi2) return true;
    return false;
}

// One prior's gate entry from its cv pose and (nullable) information; false: DSAC_ST_BAD_PRIOR.
DSAC_HD bool prior_entry(const double pose[6], const double* info, PriorGate& g) {
    bool ok = true;
    for (int m = 0; m < 6; m++) ok = ok && isfinite(pose[m]);
    const double zero[6] = {0, 0, 0, 0, 0, 0};
    const double* po = ok ? pose : zero;
    rodrigues_v2m(po, g.R);
    for (int m = 0; m < 3; m++) g.t[m] = po[3 + m];
    for (int m = 0; m < 21; m++) g.L[m] = 0;
    if (info) ok = prior_cholesky(info, g.L) && ok;
    return ok;
}

// A rig prior (R_j, t_j) seen from camera frame f of its rig, whose extrinsic is the cv pose ext (X_cam = R_c X_rig + t_c):
// the pose T_c o T_j = (R_c R_j, R_c t_j + t_c) and, for a non-null info, Lambda_f = B Lambda_j B^T with B = blockdiag(R_c,
// R_c).  A camera hypothesis lifted to the rig, (R_r, t_r), has xi_cam = B xi_rig against these, so the camera-frame gate is
// the rig-frame gate of the lifted hypothesis.  An extrinsic whose rvec is exactly zero (R_c = I exactly) keeps the prior's
// rvec and information bits, as k_rig_lift keeps a hypothesis' rvec.  False when an entry of ext is not finite.
DSAC_HD bool rig_prior_compose(const double ext[6], const double pose[6], const double* info, double out_pose[6], double* out_info) {
    bool ok = true;
    for (int m = 0; m < 6; m++) ok = ok && isfinite(ext[m]);
    double Rc[9], Rj[9], R[9];
    rodrigues_v2m(ext, Rc);
    rodrigues_v2m(pose, Rj);
    rig_compose(Rc, ext + 3, Rj, pose + 3, R, out_pose + 3);
    const bool ident = ext[0] == 0.0 && ext[1] == 0.0 && ext[2] == 0.0;
    if (ident) {
        for (int m = 0; m < 3; m++) out_pose[m] = pose[m];
    } else {
        rodrigues_m2v(R, out_pose);
    }
    if (!info) return ok;
    if (ident) {
        for (int m = 0; m < 36; m++) out_info[m] = info[m];
        return ok;
    }
    double T[36];   // B Lambda_j, then (B Lambda_j) B^T: B's two blocks are R_c
    for (int i = 0; i < 6; i++)
        for (int j = 0; j < 6; j++) {
            const int bi = i / 3 * 3, ri = i % 3;
            T[i * 6 + j] = Rc[ri * 3] * info[bi * 6 + j] + Rc[ri * 3 + 1] * info[(bi + 1) * 6 + j] + Rc[ri * 3 + 2] * info[(bi + 2) * 6 + j];
        }
    for (int i = 0; i < 6; i++)
        for (int j = 0; j < 6; j++) {
            const int bj = j / 3 * 3, rj = j % 3;
            out_info[i * 6 + j] = T[i * 6 + bj] * Rc[rj * 3] + T[i * 6 + bj + 1] * Rc[rj * 3 + 1] + T[i * 6 + bj + 2] * Rc[rj * 3 + 2];
        }
    return ok;
}

#if defined(__CUDACC__) && !defined(DSAC_HOST_ONLY)
}  // namespace dsac
#include "camera.cuh"
namespace dsac {

// One warp per frame, lane j < k for prior j: the gate table [n][k] and bad [n] (0 or DSAC_ST_BAD_PRIOR).
__global__ void __launch_bounds__(32) k_prior_prep(const double* __restrict__ poses, const double* __restrict__ info, int k,
                                                   PriorGate* __restrict__ tab, uint32_t* __restrict__ bad) {
    const int f = blockIdx.x, j = threadIdx.x;
    bool ok = true;
    if (j < k) {
        const size_t i = (size_t)f * k + j;
        PriorGate g;
        ok = prior_entry(poses + i * 6, info ? info + i * 36 : nullptr, g);
        tab[i] = g;
    }
    const unsigned any_bad = __ballot_sync(0xffffffffu, !ok);
    if (j == 0) bad[f] = any_bad ? PRIOR_ST_BAD : 0u;
}

struct PriorInjectParams {
    const double* poses;       // [n][k][6]
    const uint32_t* bad;       // [n]
    int k, H, T;               // priors per frame, hypothesis slots per frame, sampler streams
    uint32_t skip;             // stream_skip: where stream 0 stands after a frame that sampled nothing
    double f;                  // the config's focal length
    const Cam* cams;           // [n] or null
    double* hyp_pose;          // [n][H][6]
    float* hyp_P;              // [n][H][12]
    int32_t* img_idx;          // [n][H][4]
    int32_t* cand_idx;         // [n][H]
    long long* stream_ncand;   // [n][T]
    unsigned long long* stream_endpos;   // [n][T]
    uint32_t* status;          // [n]
};

// One CTA per frame, after the sampler.  Prior j goes to slot H - k + j: its pose bits, hyp_P as the sampler writes it
// (k1_write_hyp, with the frame's focal length), img_idx and cand_idx -1.  A bad frame instead gets the empty hypotheses
// of an exhausted stream in all H slots, no candidates, stream 0 right after stream_skip, and DSAC_ST_BAD_PRIOR in place
// of DSAC_ST_SAMPLER_EXHAUSTED, as if it had sampled nothing.  With k == H nothing was sampled either: stream 0 stands right
// after stream_skip, where the DSAC variant's draw continues it.
__global__ void __launch_bounds__(128) k_prior_inject(PriorInjectParams p) {
    const int f = blockIdx.x, tid = threadIdx.x;
    const double fc = p.cams ? p.cams[f].f : p.f;
    const bool bad = p.bad[f] != 0;
    const int h0 = bad ? 0 : p.H - p.k;
    for (int h = h0 + tid; h < p.H; h += blockDim.x) {
        const size_t hi = (size_t)f * p.H + h;
        double po[6] = {0, 0, 0, 0, 0, 0};
        if (!bad)
            for (int m = 0; m < 6; m++) po[m] = p.poses[((size_t)f * p.k + (h - h0)) * 6 + m];
        for (int m = 0; m < 6; m++) p.hyp_pose[hi * 6 + m] = po[m];
        double Rm[9];
        rodrigues_v2m(po, Rm);
        pose_rows(fc, Rm, po + 3, p.hyp_P + hi * 12);
        *reinterpret_cast<int4*>(p.img_idx + hi * 4) = make_int4(-1, -1, -1, -1);
        p.cand_idx[hi] = -1;
    }
    if (!bad && p.k < p.H) return;
    // nothing sampled (a bad frame, or k == H: every stream had a quota of 0)
    for (int s = tid; s < p.T; s += blockDim.x) {
        p.stream_ncand[(size_t)f * p.T + s] = 0;
        p.stream_endpos[(size_t)f * p.T + s] = (s == 0) ? p.skip : 0u;
    }
    if (tid == 0 && bad) p.status[f] = (p.status[f] & ~1u) | PRIOR_ST_BAD;
}

// dsac_set_rig_pose_priors_device, at each rig pass: the per-frame tables k_prior_inject and the gate read, composed with the
// pass's extrinsics.  Frame f = r C + c of a rig of C cameras gets prior j of rig r as T_c o T_j (rig_prior_compose).
struct RigPriorParams {
    int C, k;                   // cameras per rig, priors per rig
    const double* cam_from_rig; // [n][6] the pass's extrinsics
    const double* poses;        // [R][k][6] rig priors (cv)
    const double* info;         // [R][k][36] or null
    double* out_pose;           // [n][k][6]
    PriorGate* tab;             // [n][k]
    uint32_t* bad;              // [n] DSAC_ST_BAD_PRIOR or 0
};
constexpr int RIG_PRIOR_THREADS = 128;   // >= RIG_MAX_CAMERAS x PRIOR_MAX
static_assert(RIG_PRIOR_THREADS >= 8 * PRIOR_MAX, "one thread per (camera, prior) of a rig");

// One CTA per rig, thread c k + j for camera c's prior j.  A rig whose composed entries prior_entry refuses, or one of whose
// extrinsics is not finite, is bad in all its frames.
__global__ void __launch_bounds__(RIG_PRIOR_THREADS) k_rig_prior_prep(RigPriorParams p) {
    const int r = blockIdx.x, t = threadIdx.x, C = p.C, k = p.k;
    bool ok = true;
    if (t < C * k) {
        const int c = t / k, j = t - c * k;
        const size_t f = (size_t)r * C + c, src = (size_t)r * k + j, dst = f * k + j;
        double pose[6], info[36];
        ok = rig_prior_compose(p.cam_from_rig + f * 6, p.poses + src * 6, p.info ? p.info + src * 36 : nullptr, pose, info);
        PriorGate g;
        ok = prior_entry(pose, p.info ? info : nullptr, g) && ok;
        p.tab[dst] = g;
        for (int m = 0; m < 6; m++) p.out_pose[dst * 6 + m] = pose[m];
    }
    const int any_bad = __syncthreads_or(!ok);
    if (t < C) p.bad[(size_t)r * C + t] = any_bad ? PRIOR_ST_BAD : 0u;
}

#endif

}  // namespace dsac
