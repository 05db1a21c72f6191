// pose_math.cuh -- fp64 pose arithmetic of the hypothesis engine (device + host-testable).
//
// Everything here is written from the published algorithms (Rodrigues formula; Gao et al.
// P3P, PAMI 2003; absolute orientation of congruent triangles) for one-thread-per-problem
// execution in registers.  It replaces, for the hot path, what the reference obtains from
// OpenCV: cv::solvePnP(CV_P3P) via safeSolvePnP (cnn_softam.h:56-73, call site :1042),
// cv::Rodrigues (types.h:190) and cv::projectPoints (cnn_softam.h:351,1046).
//
// The header compiles both under nvcc (device code) and under a plain C++ compiler with
// DSAC_HOST_ONLY defined; tests/test_host_math.py uses the latter to check the product
// arithmetic against the oracle on the CPU box (the product itself never runs on the CPU).
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__) && !defined(DSAC_HOST_ONLY)
#define DSAC_HD __host__ __device__ __forceinline__
#define DSAC_HDN __host__ __device__
#else
#define DSAC_HD inline
#define DSAC_HDN inline
#endif

#define DSAC_GRID_CONST 40  /* CNN_OBJ_PATCHSIZE, lua_calls.h:33 */
#define DSAC_N_CONST 1600
#define DSAC_MAXINPUT_F 100.0f  /* CNN_OBJ_MAXINPUT, lua_calls.h:36 */
// Width (px) of the conservative filter's band above the acceptance threshold: a candidate is "certainly
// rejected" only if every P3P root puts the 4th point farther than thr + band.  The filter and the exact check
// differ by fp64 noise (amplified at most 1e4x by the conditioning guards) plus the reference's float rounding
// of pixels and projections (6e-5 px at 640 px), so 0.05 px leaves a margin of ~10^3.
#ifndef DSAC_FILTER_BAND_PX
#define DSAC_FILTER_BAND_PX 0.05
#endif

namespace dsac {

constexpr double kPi = 3.14159265358979323846;

// ----------------------------------------------------------------------------- Rodrigues
// rvec -> R (row-major).  Same formula as cv::Rodrigues: R = c I + (1-c) r r^T + s [r]x.
DSAC_HD void rodrigues_v2m(const double r[3], double R[9]) {
    double th2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    double theta = sqrt(th2);
    if (theta < 2.220446049250313e-16) {
        R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
        return;
    }
    double s, c;
#if defined(__CUDA_ARCH__)
    sincos(theta, &s, &c);
#else
    s = sin(theta); c = cos(theta);
#endif
    double c1 = 1.0 - c, it = 1.0 / theta;
    double x = r[0] * it, y = r[1] * it, z = r[2] * it;
    R[0] = c + c1 * x * x;     R[1] = c1 * x * y - s * z; R[2] = c1 * x * z + s * y;
    R[3] = c1 * x * y + s * z; R[4] = c + c1 * y * y;     R[5] = c1 * y * z - s * x;
    R[6] = c1 * x * z - s * y; R[7] = c1 * y * z + s * x; R[8] = c + c1 * z * z;
}

// R -> rvec for an orthonormal R (cv::Rodrigues' matrix branch without its SVD projection,
// which is the identity for the rotation matrices produced here).
DSAC_HD void rodrigues_m2v(const double R[9], double r[3]) {
    double rx = R[7] - R[5], ry = R[2] - R[6], rz = R[3] - R[1];
    double s = sqrt((rx * rx + ry * ry + rz * rz) * 0.25);
    double c = (R[0] + R[4] + R[8] - 1) * 0.5;
    c = c > 1. ? 1. : c < -1. ? -1. : c;
    double theta = acos(c);
    if (s < 1e-5) {
        if (c > 0) {
            r[0] = r[1] = r[2] = 0;
        } else {
            double t;
            t = (R[0] + 1) * 0.5; rx = sqrt(t > 0 ? t : 0.);
            t = (R[4] + 1) * 0.5; ry = sqrt(t > 0 ? t : 0.) * (R[1] < 0 ? -1. : 1.);
            t = (R[8] + 1) * 0.5; rz = sqrt(t > 0 ? t : 0.) * (R[2] < 0 ? -1. : 1.);
            if (fabs(rx) < fabs(ry) && fabs(rx) < fabs(rz) && (R[5] > 0) != (ry * rz > 0)) rz = -rz;
            theta /= sqrt(rx * rx + ry * ry + rz * rz);
            r[0] = rx * theta; r[1] = ry * theta; r[2] = rz * theta;
        }
    } else {
        double vth = theta / (2 * s);
        r[0] = rx * vth; r[1] = ry * vth; r[2] = rz * vth;
    }
}

// Multi-camera rigs: a camera's fixed extrinsic (Rc, tc) maps rig coordinates to camera coordinates, X_cam = Rc X_rig + tc.
// The camera pose of rig pose (R, t): Rc R, Rc t + tc.  Rc = I and tc = 0 give (R, t) exactly.
DSAC_HD void rig_compose(const double Rc[9], const double tc[3], const double R[9], const double t[3], double Ro[9], double to[3]) {
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) Ro[i * 3 + j] = Rc[i * 3] * R[j] + Rc[i * 3 + 1] * R[3 + j] + Rc[i * 3 + 2] * R[6 + j];
        to[i] = Rc[i * 3] * t[0] + Rc[i * 3 + 1] * t[1] + Rc[i * 3 + 2] * t[2] + tc[i];
    }
}
// The rig pose of camera pose (R, t): Rc^T R, Rc^T (t - tc), the inverse of rig_compose.
DSAC_HD void rig_lift(const double Rc[9], const double tc[3], const double R[9], const double t[3], double Ro[9], double to[3]) {
    const double d[3] = {t[0] - tc[0], t[1] - tc[1], t[2] - tc[2]};
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) Ro[i * 3 + j] = Rc[i] * R[j] + Rc[3 + i] * R[3 + j] + Rc[6 + i] * R[6 + j];
        to[i] = Rc[i] * d[0] + Rc[3 + i] * d[1] + Rc[6 + i] * d[2];
    }
}
// The rig-frame point of camera-frame point e: Rc^T (e - tc), so that |Rc (R Y + t) + tc - e| = |R Y + t - Rc^T (e - tc)|.
// An extrinsic rotation that is exactly I (a zero rvec) gives e - tc exactly, and with tc = 0 e itself.
DSAC_HD void rig_point(const double Rc[9], const double tc[3], const double e[3], double o[3]) {
    const double d[3] = {e[0] - tc[0], e[1] - tc[1], e[2] - tc[2]};
    bool ident = true;
    for (int k = 0; k < 9; k++) ident = ident && Rc[k] == (k % 4 == 0 ? 1.0 : 0.0);
    for (int i = 0; i < 3; i++) o[i] = ident ? d[i] : Rc[i] * d[0] + Rc[3 + i] * d[1] + Rc[6 + i] * d[2];
}

// The angle (degrees) of a relative rotation from its trace, as maxloss.h and Hypothesis::calcAngularDistance compute
// it: the trace clamped to [-1, 3], then 180 acos((trace - 1) / 2) / pi.
DSAC_HD double rot_err_deg(double trace) {
    trace = fmin(3.0, fmax(-1.0, trace));
    return 180 * acos((trace - 1.0) / 2.0) / kPi;
}

// cv::projectPoints for one point, zero distortion (double arithmetic, z==0 -> 1).
DSAC_HD void project_point(const double R[9], const double t[3], double X, double Y, double Z, double f, double cx,
                           double cy, double* u, double* v) {
    double x = R[0] * X + R[1] * Y + R[2] * Z + t[0];
    double y = R[3] * X + R[4] * Y + R[5] * Z + t[1];
    double z = R[6] * X + R[7] * Y + R[8] * Z + t[2];
    z = z ? 1. / z : 1;
    x *= z;
    y *= z;
    *u = x * f + cx;
    *v = y * f + cy;
}

// ----------------------------------------------------------------------------- reprojection error of one cell
// Separately rounded double operations (no FMA contraction), as the scalar code of cv::projectPoints.
#if defined(__CUDA_ARCH__)
#define DSAC_DMUL(a, b) __dmul_rn((a), (b))
#define DSAC_DADD(a, b) __dadd_rn((a), (b))
#define DSAC_DDIV(a, b) __ddiv_rn((a), (b))
#define DSAC_FSUB(a, b) __fsub_rn((a), (b))
#else
#define DSAC_DMUL(a, b) ((a) * (b))
#define DSAC_DADD(a, b) ((a) + (b))
#define DSAC_DDIV(a, b) ((a) / (b))
#define DSAC_FSUB(a, b) ((a) - (b))
#endif

// One entry of getDiffMap (cnn_softam.h:319-362) with the reference's roundings: projection in double, rounded
// to a float Point2f, float difference to the float pixel, norm in double, clamp at 100, stored as float.
DSAC_HD float reproj_error_exact(const double R[9], const double t[3], double X, double Y, double Z, double f, double cx,
                                 double cy, float pix_u, float pix_v) {
    double x = DSAC_DADD(DSAC_DADD(DSAC_DADD(DSAC_DMUL(R[0], X), DSAC_DMUL(R[1], Y)), DSAC_DMUL(R[2], Z)), t[0]);
    double y = DSAC_DADD(DSAC_DADD(DSAC_DADD(DSAC_DMUL(R[3], X), DSAC_DMUL(R[4], Y)), DSAC_DMUL(R[5], Z)), t[1]);
    double z = DSAC_DADD(DSAC_DADD(DSAC_DADD(DSAC_DMUL(R[6], X), DSAC_DMUL(R[7], Y)), DSAC_DMUL(R[8], Z)), t[2]);
    z = z ? DSAC_DDIV(1., z) : 1;
    x = DSAC_DMUL(x, z);
    y = DSAC_DMUL(y, z);
    const float pu = (float)DSAC_DADD(DSAC_DMUL(x, f), cx), pv = (float)DSAC_DADD(DSAC_DMUL(y, f), cy);
    const float du = DSAC_FSUB(pix_u, pu), dv = DSAC_FSUB(pix_v, pv);
    const double nrm = sqrt(DSAC_DADD(DSAC_DMUL((double)du, (double)du), DSAC_DMUL((double)dv, (double)dv)));
    return (float)fmin(nrm, 100.0);
}

// Conservative fp32 version of "reproj_error_exact(...) < thr" for the refinement's inlier test (the only use the
// refinement makes of its error maps, cnn_softam.h:1125-1133).  P = rows (f R0 | f t0), (f R1 | f t1), (R2 | t2)
// rounded to float; pu, pv = pixel - principal point; c_abs = |cx| + |cy|.  Returns 1 / 0 when the decision is
// certain, -1 when the fp32 error e = |(pu z - x, pv z - y)| / |z| is within its own error bound B of the threshold
// (the caller then evaluates reproj_error_exact).
//   Bound: every fp32 sum s = sum_k P_k X_k carries at most 4 roundings of 2^-24 relative to S = sum_k |P_k X_k|
//   (2.4e-7 S; 1e-6 S is used), which propagate to e as [dx + dy + (|pu| + |pv| + e) dz] / |z|; the reference's own
//   float rounding of the projected pixel adds 6e-8 (|u| + |v|); e is replaced by T = 2 thr inside B (for e > T the
//   decision "not below" only needs B < thr, which is required).
//   The test is made on squares, multiplied through by |z| (no sqrt, no division):
//       sqrt(A) < thr |z| - B |z|  ->  below,     sqrt(A) > thr |z| + B |z|  ->  not below.
// NaN / a bound that is not small against the threshold (z ~ 0) return -1.
DSAC_HD int reproj_below_thr_fast(const float* P, float X, float Y, float Z, float pu, float pv, float c_abs, float thr) {
    const float xs = fmaf(P[0], X, fmaf(P[1], Y, fmaf(P[2], Z, P[3])));
    const float ys = fmaf(P[4], X, fmaf(P[5], Y, fmaf(P[6], Z, P[7])));
    const float zs = fmaf(P[8], X, fmaf(P[9], Y, fmaf(P[10], Z, P[11])));
    const float aX = fabsf(X), aY = fabsf(Y), aZ = fabsf(Z);
    const float Sx = fmaf(fabsf(P[0]), aX, fmaf(fabsf(P[1]), aY, fmaf(fabsf(P[2]), aZ, fabsf(P[3]))));
    const float Sy = fmaf(fabsf(P[4]), aX, fmaf(fabsf(P[5]), aY, fmaf(fabsf(P[6]), aZ, fabsf(P[7]))));
    const float Sz = fmaf(fabsf(P[8]), aX, fmaf(fabsf(P[9]), aY, fmaf(fabsf(P[10]), aZ, fabsf(P[11]))));
    const float az = fabsf(zs), apuv = fabsf(pu) + fabsf(pv), T = 2.f * thr;
    const float du = fmaf(pu, zs, -xs), dv = fmaf(pv, zs, -ys);
    const float A = fmaf(du, du, dv * dv);
    const float c1 = 1e-6f * (Sx + Sy + (apuv + T) * Sz);
    const float k3 = fmaf(2.4e-7f, apuv + c_abs, fmaf(1.05e-5f, T, 2e-4f));
#ifdef DSAC_REPROJ_BOUND_SCALE   /* test aid: how far can the bound shrink before a decision goes wrong */
    const float Bz = (float)(DSAC_REPROJ_BOUND_SCALE) * fmaf(k3, az, c1);
#else
    const float Bz = fmaf(k3, az, c1);                  // B |z|
#endif
    const float taz = thr * az;
    if (!(Bz < 0.5f * taz)) return -1;
    const float lo = taz - Bz, hi = taz + Bz;
    if (A < lo * lo) return 1;
    if (A > hi * hi) return 0;
    return -1;
}

// ----------------------------------------------------------------------------- k_score's fp32 arithmetic
// MUFU approximations on the device, plain libm on the host (the host build only serves the CPU-side checks)
#if defined(__CUDA_ARCH__)
DSAC_HD float approx_rsqrt(float x) { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
DSAC_HD float approx_rcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
DSAC_HD float approx_ex2(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
#else
DSAC_HD float approx_rsqrt(float x) { return 1.0f / sqrtf(x); }
DSAC_HD float approx_rcp(float x) { return 1.0f / x; }
DSAC_HD float approx_ex2(float x) { return exp2f(x); }
#endif

// One entry of the H x N reprojection-error matrix as k_score computes it: rows r0 = (f R0 | f t0), r1 = (f R1 | f t1),
// r2 = (R2 | t2) of the hypothesis in float, scene coordinate (X, Y, Z), pixel minus principal point (pu, pv).
//   e = |pix - proj| = sqrt(A) / |z|,  A = (pu z - xs)^2 + (pv z - ys)^2   ->   e = A * rsqrt(max(A z^2, floor)),
// clamped at 100 (CNN_OBJ_MAXINPUT, cnn_softam.h:357).  A = 0 (the float projection lands exactly on the pixel -- it does
// happen for the three points a P3P pose fits exactly) gives 0 * rsqrt(floor) = 0; A > 0 implies A >= ulp^2 and z != 0
// implies z^2 far above the floor.  GUARDED adds cv::projectPoints' z ? 1/z : 1; *az returns |z| before that substitution
// (the unguarded caller uses it to detect z == 0 and repeat with GUARDED).
#ifndef DSAC_K2_FLOOR_FMA
#define DSAC_K2_FLOOR_FMA 1   /* floor under k_score's rsqrt as an FMA addend (1) or as a separate max (0) */
#endif
template <bool GUARDED>
DSAC_HD float score_pair_error(float r0x, float r0y, float r0z, float r0w, float r1x, float r1y, float r1z, float r1w, float r2x,
                               float r2y, float r2z, float r2w, float X, float Y, float Z, float pu, float pv, float* az) {
    const float xs = fmaf(r0x, X, fmaf(r0y, Y, fmaf(r0z, Z, r0w)));
    const float ys = fmaf(r1x, X, fmaf(r1y, Y, fmaf(r1z, Z, r1w)));
    float zs = fmaf(r2x, X, fmaf(r2y, Y, fmaf(r2z, Z, r2w)));
    *az = fabsf(zs);
    if (GUARDED) zs = (zs != 0.f) ? zs : 1.f;  // z ? 1/z : 1 (cv::projectPoints)
    const float du = fmaf(pu, zs, -xs);
    const float dv = fmaf(pv, zs, -ys);
    const float A = fmaf(du, du, dv * dv);
    // floor under the rsqrt (A = 0: a point exactly on its pixel) as the addend of an FMA instead of a separate max: for
    // every A z^2 that is not (sub)normal-small the sum rounds to A z^2 itself, i.e. the same bits as before
#if DSAC_K2_FLOOR_FMA
    return fminf(A * approx_rsqrt(fmaf(A, zs * zs, 1e-30f)), DSAC_MAXINPUT_F);
#else
    return fminf(A * approx_rsqrt(fmaxf(A * (zs * zs), 1e-30f)), DSAC_MAXINPUT_F);
#endif
}

// Sum of the soft-inlier sigmoids sigma(beta (tau - e_j)) = 1 / (1 + 2^(kbeta e_j - tau_k)) of five errors over ONE
// reciprocal, sum_j 1/w_j = N / D: w_j clamped to 2^25 + 1 so that D < 2^126 (a sigmoid below 2^-25 is rounded up to
// 2^-25: <= 5e-6 absolute on a score).  The XU / MIO queue is k_score's scarcest resource, so one MUFU per five points
// beats one per two.
DSAC_HD float score_sigmoid_sum5(const float e[5], float kbeta, float tau_k) {
    float w[5];
    for (int j = 0; j < 5; j++) w[j] = 1.f + approx_ex2(fmaf(kbeta, e[j], -tau_k));
    const float u0 = fminf(w[0], 33554433.f), u1 = fminf(w[1], 33554433.f), u2 = fminf(w[2], 33554433.f),
                u3 = fminf(w[3], 33554433.f), u4 = fminf(w[4], 33554433.f);
    const float p01 = u0 * u1, p23 = u2 * u3, qq = p23 * u4;
    const float Nn = fmaf(u0 + u1, qq, p01 * fmaf(u2 + u3, u4, p23));
    return Nn * approx_rcp(p01 * qq);
}

// ----------------------------------------------------------------------------- P3P
// Products of the exact P3P solve's closed forms (cubic_first_root, quartic_roots) that are never contracted into a
// fused multiply-add.  Those closed forms take exact sign decisions (D <= 0, R2 >= 0, D2 >= 0, E2 >= 0) that sit on a
// near-double root for some minimal sets; nvcc's default contraction rounds such a discriminant differently from the
// reference's (uncontracted) arithmetic and can flip it, and the sampler then drops a minimal set the reference accepts
// (seen at f = 1500: tests/test_gpu_params.py).  __dmul_rn is never fused; on the host the product goes through a volatile,
// which no -ffp-contract setting can fuse into the following sum (tests/test_host_params.py builds it with -mfma to check).
DSAC_HD double p3p_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    volatile double r = a * b;
    return r;
#endif
}

// Largest real root of y^3 + a2 y^2 + a1 y + a0 (the resolvent cubic of Ferrari's method).
#if defined(__CUDA_ARCH__)
#define DSAC_RSQRTF_EARLY(x) rsqrtf(x)
#else
#define DSAC_RSQRTF_EARLY(x) (1.0f / sqrtf(x))
#endif

DSAC_HD double cubic_first_root(double a2, double a1, double a0) {
    const double a22 = p3p_mul(a2, a2);
    double Q = (p3p_mul(3, a1) - a22) / 9;
    double R = (p3p_mul(p3p_mul(9, a2), a1) - p3p_mul(27, a0) - p3p_mul(p3p_mul(2, a22), a2)) / 54;
    double Q3 = p3p_mul(p3p_mul(Q, Q), Q), D = Q3 + p3p_mul(R, R), sh = a2 / 3;
    if (Q == 0) return (R == 0) ? -sh : cbrt(2 * R) - sh;
    if (D <= 0) {
        double theta = acos(R / sqrt(-Q3));
        return p3p_mul(2 * sqrt(-Q), cos(theta / 3.0)) - sh;
    }
    double AD = cbrt(fabs(R) + sqrt(D)) * (R > 0 ? 1 : (R < 0 ? -1 : 0));
    double BD = (AD == 0) ? 0 : -Q / AD;
    return AD + BD - sh;
}

// Real roots of the quartic (closed form; accuracy is restored afterwards by Newton steps
// on the two-quadric system, see p3p_best).  Every product that feeds a sum is p3p_mul (see above).
DSAC_HD int quartic_roots(double a, double b, double c, double d, double e, double x[4]) {
    if (a == 0) return 0;
    double ia = 1.0 / a;
    b *= ia; c *= ia; d *= ia; e *= ia;
    const double bb = p3p_mul(b, b);
    double y1 = cubic_first_root(-c, p3p_mul(d, b) - p3p_mul(4, e), p3p_mul(p3p_mul(4, c), e) - p3p_mul(d, d) - p3p_mul(bb, e));
    double R2 = p3p_mul(0.25, bb) - c + y1;
    if (!(R2 >= 0)) return 0;
    double R = sqrt(R2), D2, E2;
    if (R < 10e-12) {
        double t = p3p_mul(y1, y1) - p3p_mul(4, e);
        if (t < 0) {
            D2 = E2 = -1;
        } else {
            double st = sqrt(t);
            D2 = p3p_mul(p3p_mul(0.75, b), b) - p3p_mul(2, c) + p3p_mul(2, st);
            E2 = D2 - p3p_mul(4, st);
        }
    } else {
        double u = p3p_mul(p3p_mul(0.75, b), b) - p3p_mul(2, c) - R2;
        double v = p3p_mul(0.25, p3p_mul(p3p_mul(4, b), c) - p3p_mul(8, d) - p3p_mul(bb, b)) / R;
        D2 = u + v;
        E2 = u - v;
    }
    int n = 0;
    if (D2 >= 0) {
        double Dq = sqrt(D2);
        x[0] = p3p_mul(0.5, R) + p3p_mul(0.5, Dq) - p3p_mul(0.25, b);
        x[1] = x[0] - Dq;
        n = 2;
    }
    if (E2 >= 0) {
        double Eq = sqrt(E2);
        x[n] = p3p_mul(-0.5, R) + p3p_mul(0.5, Eq) - p3p_mul(0.25, b);
        x[n + 1] = x[n] - Eq;
        n += 2;
    }
    return n;
}

DSAC_HD double rsqrt_or(double x) {
#if defined(__CUDA_ARCH__)
    return rsqrt(x);
#else
    return 1.0 / sqrt(x);
#endif
}

// Reciprocal / reciprocal square root / square root for the CONSERVATIVE FILTER only (p3p_lambda_core):
// the hardware's 20-bit approximation refined by two Newton steps -- a few ulp, five to nine instructions instead of the
// IEEE division / square root sequences (which were ~30 % of the filter's instructions).  The filter's decisions are
// protected by bands >= 1e-9 relative (and 0.05 px), nine orders of magnitude above that error; zero, subnormal, infinite
// or NaN arguments give inf / NaN, which every test of the filter sends to "needs the full solve".  The full solve and
// everything that produces results keeps IEEE arithmetic.  On the host these are the exact operations.
DSAC_HD double filt_rcp(double x) {
#if defined(__CUDA_ARCH__)
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
    double e = fma(-x, r, 1.0);
    r = fma(r, e, r);
    e = fma(-x, r, 1.0);
    return fma(r, e, r);
#else
    return 1.0 / x;
#endif
}
DSAC_HD double filt_rsqrt(double x) {
#if defined(__CUDA_ARCH__)
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
    const double h = 0.5 * x;
    double e = fma(-h, y * y, 0.5);
    y = fma(y, e, y);
    e = fma(-h, y * y, 0.5);
    return fma(y, e, y);
#else
    return 1.0 / sqrt(x);
#endif
}
DSAC_HD double filt_sqrt(double x) {   // x > 0
#if defined(__CUDA_ARCH__)
    return x * filt_rsqrt(x);
#else
    return sqrt(x);
#endif
}

// A real root of y^3 + a2 y^2 + a1 y + a0 (the largest one when there are three), for the conservative filter only
// (p3p_lambda_core's cubic): an fp32 closed-form seed (a handful of MUFU operations instead of fp64 acos/cos/cbrt/sqrt,
// ~300 instructions) restored to fp64 accuracy by three Newton steps (quadratic convergence from the seed's ~1e-6 relative
// error).  *ok is false
// when the last step has not collapsed below 1e-13 of the problem's scale (near-multiple root: there Newton converges only
// linearly and the root is no better than a few steps' size; overflow, NaN) and
// the caller must then treat the candidate as uncertain.
DSAC_HD double cubic_first_root_seeded(double a2, double a1, double a0, bool* ok) {
    // Branch-free: the lanes of a warp hold different candidates, and a divergent branch here costs every lane the
    // instructions of both sides anyway.  Both closed forms are evaluated in fp32 (the fp32 pipe is idle in the filter)
    // on arguments clamped into their domains, and the one that applies is selected.
    const double Q = (3 * a1 - a2 * a2) * (1.0 / 9), R = (9 * a2 * a1 - 27 * a0 - 2 * a2 * a2 * a2) * (1.0 / 54);
    const double Q3 = Q * Q * Q, D = Q3 + R * R, sh = a2 * (1.0 / 3);
    const float Qf = (float)Q, Rf = (float)R;
    // D <= 0: three real roots, the largest one is 2 sqrt(-Q) cos(acos(R / sqrt(-Q^3)) / 3)
    float cs = Rf * DSAC_RSQRTF_EARLY(fmaxf(-(float)Q3, 1e-37f));
    cs = fminf(1.f, fmaxf(-1.f, cs));
#if defined(__CUDA_ARCH__)
    const float s_trig = 2.f * sqrtf(fmaxf(-Qf, 0.f)) * __cosf(acosf(cs) * (1.f / 3));
#else
    const float s_trig = 2.f * sqrtf(fmaxf(-Qf, 0.f)) * cosf(acosf(cs) * (1.f / 3));
#endif
    // D > 0: one real root, Cardano
    float AD = cbrtf(fabsf(Rf) + sqrtf(fmaxf((float)D, 0.f)));
    AD = (Rf >= 0) ? AD : -AD;
    const float s_card = AD + ((AD == 0) ? 0.f : -Qf / AD);
    const float s = (D <= 0) ? s_trig : s_card;
    double y = (double)s - sh, dy = 0;
#pragma unroll
    for (int it = 0; it < 3; it++) {
        const double g = ((y + a2) * y + a1) * y + a0, gp = (3 * y + 2 * a2) * y + a1;
        dy = g * filt_rcp(gp);
        y -= dy;
    }
    *ok = fabs(dy) <= 1e-13 * (fabs(y) + fabs(sh));
    return y;
}

struct P3PProblem {
    double mu[4], mv[4];  // pixel positions as P3P sees them (float-rounded normalised coords mapped back through K)
    double X[4][3];       // scene coordinates (mm)
};

// Orthonormal frame of a triangle: e1 along P1-P0, e3 along the normal, e2 = e3 x e1.
DSAC_HD void triangle_frame(const double P0[3], const double P1[3], const double P2[3], double E[9]) {
    double ax = P1[0] - P0[0], ay = P1[1] - P0[1], az = P1[2] - P0[2];
    double bx = P2[0] - P0[0], by = P2[1] - P0[1], bz = P2[2] - P0[2];
    double ia = 1.0 / sqrt(ax * ax + ay * ay + az * az);
    ax *= ia; ay *= ia; az *= ia;
    double nx = ay * bz - az * by, ny = az * bx - ax * bz, nz = ax * by - ay * bx;
    double in = 1.0 / sqrt(nx * nx + ny * ny + nz * nz);
    nx *= in; ny *= in; nz *= in;
    E[0] = ax; E[1] = ay; E[2] = az;
    E[3] = ny * az - nz * ay; E[4] = nz * ax - nx * az; E[5] = nx * ay - ny * ax;
    E[6] = nx; E[7] = ny; E[8] = nz;
}

// Pose from one P3P solution: camera-frame points L_i * bearing_i aligned with the world
// triangle (congruent after the Newton polish, so the frame-to-frame rotation equals the
// least-squares absolute orientation to rounding).
DSAC_HD void pose_from_lengths(const double Lx, const double Ly, const double Lz, const double bear[3][3],
                               const double Ew[9], const double Cw[3], double R[9], double t[3]) {
    double M0[3] = {Lx * bear[0][0], Lx * bear[0][1], Lx * bear[0][2]};
    double M1[3] = {Ly * bear[1][0], Ly * bear[1][1], Ly * bear[1][2]};
    double M2[3] = {Lz * bear[2][0], Lz * bear[2][1], Lz * bear[2][2]};
    double Ec[9];
    triangle_frame(M0, M1, M2, Ec);
    // R = Ec^T * Ew  (rows of E are the frame axes)
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) R[i * 3 + j] = Ec[0 + i] * Ew[0 + j] + Ec[3 + i] * Ew[3 + j] + Ec[6 + i] * Ew[6 + j];
    double Cc[3] = {(M0[0] + M1[0] + M2[0]) / 3, (M0[1] + M1[1] + M2[1]) / 3, (M0[2] + M1[2] + M2[2]) / 3};
    for (int i = 0; i < 3; i++) t[i] = Cc[i] - (R[i * 3] * Cw[0] + R[i * 3 + 1] * Cw[1] + R[i * 3 + 2] * Cw[2]);
}

// Front end shared by the quick filter and the full solve: bearings, the two quadrics'
// coefficients and the closed-form roots of the quartic in x = |PA|/|PC|.
struct P3PFront {
    double bear[3][3];
    double p, q, r, a, b;       // quadrics: f1 = (1-a)y^2 - a x^2 - p y + a r x y + 1, f2 = (1-b)x^2 - b y^2 - q x + b r x y + 1
    double N2, N1, N0, D1, D0;  // y * (D1 x + D0) = -(N2 x^2 + N1 x + N0)
    double d01;
    double xr[4];
    int nroots;
};

#if defined(__CUDACC__) && !defined(DSAC_HOST_ONLY)
#define DSAC_NOINLINE __noinline__
#else
#define DSAC_NOINLINE
#endif

// Not inlined on the device so that the quick filter and the full solve see bit-identical
// roots (one compiled instance, one FMA-contraction pattern).
DSAC_HDN DSAC_NOINLINE void p3p_front(const P3PProblem& pr, double f, double cx, double cy, P3PFront& fr) {
    double inv_f = 1.0 / f, cx_f = cx * inv_f, cy_f = cy * inv_f;
    for (int i = 0; i < 3; i++) {
        double u = inv_f * pr.mu[i] - cx_f, v = inv_f * pr.mv[i] - cy_f;
#if defined(__CUDA_ARCH__)
        double k = rsqrt(u * u + v * v + 1);
#else
        double k = 1. / sqrt(u * u + v * v + 1);
#endif
        fr.bear[i][0] = u * k; fr.bear[i][1] = v * k; fr.bear[i][2] = k;
    }
    // only ratios of squared distances enter the quadrics; |AB| itself fixes the scale
    double s12, s02, s01;
    {
        double dx = pr.X[1][0] - pr.X[2][0], dy = pr.X[1][1] - pr.X[2][1], dz = pr.X[1][2] - pr.X[2][2];
        s12 = dx * dx + dy * dy + dz * dz;
        dx = pr.X[0][0] - pr.X[2][0]; dy = pr.X[0][1] - pr.X[2][1]; dz = pr.X[0][2] - pr.X[2][2];
        s02 = dx * dx + dy * dy + dz * dz;
        dx = pr.X[0][0] - pr.X[1][0]; dy = pr.X[0][1] - pr.X[1][1]; dz = pr.X[0][2] - pr.X[1][2];
        s01 = dx * dx + dy * dy + dz * dz;
    }
    fr.d01 = sqrt(s01);
    const double (*bear)[3] = fr.bear;
    double p = 2 * (bear[1][0] * bear[2][0] + bear[1][1] * bear[2][1] + bear[1][2] * bear[2][2]);
    double q = 2 * (bear[0][0] * bear[2][0] + bear[0][1] * bear[2][1] + bear[0][2] * bear[2][2]);
    double r = 2 * (bear[0][0] * bear[1][0] + bear[0][1] * bear[1][1] + bear[0][2] * bear[1][2]);
    double inv_c2 = 1.0 / s01;
    double a = inv_c2 * s12, b = inv_c2 * s02;
    fr.p = p; fr.q = q; fr.r = r; fr.a = a; fr.b = b;
    fr.nroots = 0;
    if (p * p + q * q + r * r - p * q * r - 1 == 0) return;
    double N2 = 1 - a - b, N1 = q * (a - 1), N0 = 1 - a + b;
    double D1 = b * r, D0 = -b * p;
    fr.N2 = N2; fr.N1 = N1; fr.N0 = N0; fr.D1 = D1; fr.D0 = D0;
    double c4, c3, c2, c1, c0;
    {
        double F2 = 1 - b, F1 = -q;
        double DD2 = D1 * D1, DD1 = 2 * D1 * D0, DD0 = D0 * D0;
        double br = b * r;
        c4 = F2 * DD2 - b * (N2 * N2) - br * (N2 * D1);
        c3 = F2 * DD1 + F1 * DD2 - b * (2 * N2 * N1) - br * (N2 * D0 + N1 * D1);
        c2 = F2 * DD0 + F1 * DD1 + DD2 - b * (2 * N2 * N0 + N1 * N1) - br * (N1 * D0 + N0 * D1);
        c1 = F1 * DD0 + DD1 - b * (2 * N1 * N0) - br * (N0 * D0);
        c0 = DD0 - b * (N0 * N0);
    }
    if (c4 == 0) return;
    fr.nroots = quartic_roots(c4, c3, c2, c1, c0, fr.xr);
}

// y candidates for a quartic root x0: the linear relation, or (where it degenerates) both
// roots of the first quadric.
DSAC_HD int p3p_y_candidates(const P3PFront& fr, double x0, double* ya, double* yb) {
    double Dn = fr.D1 * x0 + fr.D0;
    if (fabs(Dn) > 1e-3 * (fabs(fr.D1 * x0) + fabs(fr.D0))) {
        *ya = *yb = -((fr.N2 * x0 + fr.N1) * x0 + fr.N0) / Dn;
        return 1;
    }
    double qa = 1 - fr.a, qb = fr.a * fr.r * x0 - fr.p, qc = 1 - fr.a * x0 * x0;
    double disc = qb * qb - 4 * qa * qc;
    if (disc < 0) disc = 0;
    double sq = sqrt(disc);
    if (qa != 0) {
        *ya = (-qb + sq) / (2 * qa);
        *yb = (-qb - sq) / (2 * qa);
        return 2;
    }
    if (qb != 0) {
        *ya = *yb = -qc / qb;
        return 1;
    }
    *ya = *yb = 0;
    return 0;
}

// All P3P solutions from points 0..2 (given the front end), the one with the smallest squared
// reprojection error of point 3 is returned (cv::solvePnP CV_P3P semantics).  Returns the
// number of solutions; *best_err2 is that smallest squared error (pixels^2).
// Only quartic roots with index in [root_lo, root_hi) are processed (the sampler's full-solve phase spreads
// the roots of one candidate over a group of lanes and takes the minimum across them).
DSAC_HDN int p3p_full(const P3PProblem& pr, const P3PFront& fr, double f, double cx, double cy, double Rbest[9],
                      double tbest[3], double* best_err2, int root_lo = 0, int root_hi = 4) {
    if (fr.nroots == 0) return 0;
    const double a = fr.a, b = fr.b, p = fr.p, q = fr.q, r = fr.r;
    double Ew[9], Cw[3];
    triangle_frame(pr.X[0], pr.X[1], pr.X[2], Ew);
    for (int k = 0; k < 3; k++) Cw[k] = (pr.X[0][k] + pr.X[1][k] + pr.X[2][k]) / 3;

    double sx[4], sy[4];
    int ns = 0, nsol = 0;
    double best = 0;
    for (int i = root_lo; i < fr.nroots && i < root_hi; i++) {
        double x0 = fr.xr[i];
        if (!(x0 == x0)) continue;
        double y0a, y0b;
        int nc = p3p_y_candidates(fr, x0, &y0a, &y0b);
        for (int c = 0; c < nc; c++) {
            double x = x0, y = c ? y0b : y0a;
            bool good = false;
            for (int it = 0; it < 8; it++) {
                double f1 = (1 - a) * y * y - a * x * x - p * y + a * r * x * y + 1;
                double f2 = (1 - b) * x * x - b * y * y - q * x + b * r * x * y + 1;
                double j11 = -2 * a * x + a * r * y, j12 = 2 * (1 - a) * y - p + a * r * x;
                double j21 = 2 * (1 - b) * x - q + b * r * y, j22 = -2 * b * y + b * r * x;
                double det = j11 * j22 - j12 * j21;
                if (det == 0 || !(det == det)) break;
                double idet = 1.0 / det;
                double dx = (f1 * j22 - f2 * j12) * idet, dy = (j11 * f2 - j21 * f1) * idet;
                x -= dx;
                y -= dy;
                if (fabs(dx) + fabs(dy) <= 1e-15 * (fabs(x) + fabs(y))) {
                    good = true;
                    break;
                }
            }
            if (!good) {
                double f1 = (1 - a) * y * y - a * x * x - p * y + a * r * x * y + 1;
                double f2 = (1 - b) * x * x - b * y * y - q * x + b * r * x * y + 1;
                good = fabs(f1) + fabs(f2) < 1e-12 * (1 + x * x + y * y);
            }
            if (!good || !(x > 0) || !(y > 0)) continue;
            bool dup = false;
            for (int k = 0; k < 4; k++)
                if (k < ns && fabs(sx[k] - x) + fabs(sy[k] - y) < 1e-9 * (fabs(x) + fabs(y))) dup = true;
            if (dup || ns >= 4) continue;
            sx[ns] = x;
            sy[ns] = y;
            ns++;
            double v = x * x + y * y - x * y * r;
            if (!(v > 0)) continue;
            double Z = fr.d01 / sqrt(v);
            double R[9], t[3];
            pose_from_lengths(x * Z, y * Z, Z, fr.bear, Ew, Cw, R, t);
            double X3 = R[0] * pr.X[3][0] + R[1] * pr.X[3][1] + R[2] * pr.X[3][2] + t[0];
            double Y3 = R[3] * pr.X[3][0] + R[4] * pr.X[3][1] + R[5] * pr.X[3][2] + t[1];
            double Z3 = R[6] * pr.X[3][0] + R[7] * pr.X[3][1] + R[8] * pr.X[3][2] + t[2];
            double u3 = cx + f * X3 / Z3, v3 = cy + f * Y3 / Z3;
            double e2 = (u3 - pr.mu[3]) * (u3 - pr.mu[3]) + (v3 - pr.mv[3]) * (v3 - pr.mv[3]);
            if (nsol == 0 || best > e2) {
                best = e2;
                for (int k = 0; k < 9; k++) Rbest[k] = R[k];
                tbest[0] = t[0]; tbest[1] = t[1]; tbest[2] = t[2];
            }
            nsol++;
        }
    }
    *best_err2 = best;
    return nsol;
}

DSAC_HDN int p3p_best(const P3PProblem& pr, double f, double cx, double cy, double Rbest[9], double tbest[3],
                      double* best_err2) {
    P3PFront fr;
    p3p_front(pr, f, cx, cy, fr);
    return p3p_full(pr, fr, f, cx, cy, Rbest, tbest, best_err2);
}

// Conservative filter: returns false only if the full solve certainly cannot produce a pose
// whose 4th-point error is below `thr` (so the candidate is certainly rejected by the
// sampling loop, cnn_softam.h:1049-1057); returns true ("needs the full solve") otherwise,
// including every numerically delicate situation.  Per root it takes ONE Newton step on the
// two quadrics; if that step is tiny and well conditioned the stepped (x, y) is within ~1e-12
// of the true solution, and the 4th point's camera position follows from the congruence of
// the camera and world triangles without building the pose:
//   M3 = M0 + alpha e1 + beta e2 + gamma e3,  e1 = (M1-M0)/d01, e3 = (M1-M0)x(M2-M0)/|n_w|, e2 = e3 x e1.
DSAC_HDN bool p3p_quick_needs_full(const P3PProblem& pr, const P3PFront& fr, double f, double cx, double cy, double thr) {
    if (fr.nroots == 0) return false;  // same front end as the full solve: it finds nothing either
    const double a = fr.a, b = fr.b, p = fr.p, q = fr.q, r = fr.r;
    // world triangle frame and the 4th point's coordinates in it
    double ax = pr.X[1][0] - pr.X[0][0], ay = pr.X[1][1] - pr.X[0][1], az = pr.X[1][2] - pr.X[0][2];
    double bx = pr.X[2][0] - pr.X[0][0], by = pr.X[2][1] - pr.X[0][1], bz = pr.X[2][2] - pr.X[0][2];
    double nx = ay * bz - az * by, ny = az * bx - ax * bz, nz = ax * by - ay * bx;
    double nn = nx * nx + ny * ny + nz * nz;
    if (!(fr.d01 > 0) || !(nn > 0)) return true;
    double inv_d = 1.0 / fr.d01, inv_n = 1.0 / sqrt(nn);
    double e1x = ax * inv_d, e1y = ay * inv_d, e1z = az * inv_d;
    double e3x = nx * inv_n, e3y = ny * inv_n, e3z = nz * inv_n;
    double e2x = e3y * e1z - e3z * e1y, e2y = e3z * e1x - e3x * e1z, e2z = e3x * e1y - e3y * e1x;
    double wx = pr.X[3][0] - pr.X[0][0], wy = pr.X[3][1] - pr.X[0][1], wz = pr.X[3][2] - pr.X[0][2];
    double al = wx * e1x + wy * e1y + wz * e1z, be = wx * e2x + wy * e2y + wz * e2z, ga = wx * e3x + wy * e3y + wz * e3z;
    const double lim2 = (thr + DSAC_FILTER_BAND_PX) * (thr + DSAC_FILTER_BAND_PX);
    for (int i = 0; i < fr.nroots; i++) {
        double x0 = fr.xr[i];
        if (!(x0 == x0)) return true;
        double y0a, y0b;
        int nc = p3p_y_candidates(fr, x0, &y0a, &y0b);
        if (nc != 1) return true;  // degenerate linear relation: let the full solve handle it
        double x = x0, y = y0a;
        double f1 = (1 - a) * y * y - a * x * x - p * y + a * r * x * y + 1;
        double f2 = (1 - b) * x * x - b * y * y - q * x + b * r * x * y + 1;
        double j11 = -2 * a * x + a * r * y, j12 = 2 * (1 - a) * y - p + a * r * x;
        double j21 = 2 * (1 - b) * x - q + b * r * y, j22 = -2 * b * y + b * r * x;
        double det = j11 * j22 - j12 * j21;
        double jn = j11 * j11 + j12 * j12 + j21 * j21 + j22 * j22;
        if (!(fabs(det) > 1e-4 * jn)) return true;  // (near-)singular Jacobian, NaN
        double idet = 1.0 / det;
        double dx = (f1 * j22 - f2 * j12) * idet, dy = (j11 * f2 - j21 * f1) * idet;
        x -= dx;
        y -= dy;
        if (!(fabs(dx) + fabs(dy) <= 1e-6 * (fabs(x) + fabs(y)))) return true;  // not yet in the quadratic regime
        if (x < -1e-6 || y < -1e-6) continue;       // certainly a non-physical solution
        if (x < 1e-6 || y < 1e-6) return true;      // borderline positivity
        double v = x * x + y * y - x * y * r;
        if (!(v > 1e-12)) return true;
        double Z = fr.d01 / sqrt(v);
        double L0 = x * Z, L1 = y * Z;
        double M0x = L0 * fr.bear[0][0], M0y = L0 * fr.bear[0][1], M0z = L0 * fr.bear[0][2];
        double ux = L1 * fr.bear[1][0] - M0x, uy = L1 * fr.bear[1][1] - M0y, uz = L1 * fr.bear[1][2] - M0z;
        double vx = Z * fr.bear[2][0] - M0x, vy = Z * fr.bear[2][1] - M0y, vz = Z * fr.bear[2][2] - M0z;
        double cxn = uy * vz - uz * vy, cyn = uz * vx - ux * vz, czn = ux * vy - uy * vx;
        double c1x = ux * inv_d, c1y = uy * inv_d, c1z = uz * inv_d;
        double c3x = cxn * inv_n, c3y = cyn * inv_n, c3z = czn * inv_n;
        double c2x = c3y * c1z - c3z * c1y, c2y = c3z * c1x - c3x * c1z, c2z = c3x * c1y - c3y * c1x;
        double X3 = M0x + al * c1x + be * c2x + ga * c3x;
        double Y3 = M0y + al * c1y + be * c2y + ga * c3y;
        double Z3 = M0z + al * c1z + be * c2z + ga * c3z;
        double iz = 1.0 / Z3;
        double du = cx + f * X3 * iz - pr.mu[3], dv = cy + f * Y3 * iz - pr.mv[3];
        double e2 = du * du + dv * dv;
        if (!(e2 > lim2)) return true;  // possibly below the threshold (or NaN): full solve decides
    }
    return false;
}

// The pixel a P3P solve actually sees: cv::undistortPoints rounds the normalised
// coordinate to float, p3p maps it back through K.
DSAC_HD double p3p_pixel(float pix, double c, double f) {
    float n = (float)(((double)pix - c) * (1. / f));
    return n * f + c;
}

// Minimal-set hypothesis exactly as the sampling loop evaluates it (cnn_softam.h:1041-1059):
// P3P on the 4 correspondences, then all 4 reprojection errors (projection rounded to
// float, float difference, double norm) must be below the integer threshold.
// Returns true if accepted; rvec/tvec are the cv pose.  *fragile is set when a decision
// was within 1e-6 px of the threshold.  pr: the P3P problem (see make_problem); obj/img: the
// float correspondences the reprojection check uses.
// Second half of the sampling loop's test, given the P3P winner (R, t, e2 = its squared 4th-point error):
// Rodrigues vector, then all 4 reprojection errors exactly as the reference measures them.
DSAC_HDN bool minimal_set_accept(const float obj[12], const float img[8], double f, double cx, double cy, int thr,
                                 const double R[9], const double t[3], double e2, double rvec[3], double tvec[3],
                                 bool* fragile) {
    *fragile = false;
    // cheap exact-safe pre-check: the 4th point's error as P3P measured it differs from the
    // reference's float-rounded check by < 1e-4 px
    if (!(e2 < ((double)thr + 1e-3) * ((double)thr + 1e-3))) return false;
    rodrigues_m2v(R, rvec);
    tvec[0] = t[0]; tvec[1] = t[1]; tvec[2] = t[2];
    double Rp[9];
    rodrigues_v2m(rvec, Rp);  // cv::projectPoints rebuilds R from rvec
    bool ok = true;
    for (int j = 0; j < 4; j++) {
        double u, v;
        project_point(Rp, tvec, obj[j * 3], obj[j * 3 + 1], obj[j * 3 + 2], f, cx, cy, &u, &v);
        float du = img[j * 2] - (float)u, dv = img[j * 2 + 1] - (float)v;
        double nrm = sqrt((double)du * du + (double)dv * dv);
        if (fabs(nrm - thr) < 1e-6) *fragile = true;
        if (!(nrm < thr)) ok = false;
    }
    return ok;
}

DSAC_HDN bool minimal_set_hypothesis_pr(const P3PProblem& pr, const float obj[12], const float img[8], double f, double cx,
                                        double cy, int thr, double rvec[3], double tvec[3], bool* fragile) {
    double R[9], t[3], e2;
    *fragile = false;
    P3PFront fr;
    p3p_front(pr, f, cx, cy, fr);
    if (p3p_full(pr, fr, f, cx, cy, R, t, &e2) == 0) return false;
    return minimal_set_accept(obj, img, f, cx, cy, thr, R, t, e2, rvec, tvec, fragile);
}

DSAC_HD void make_problem(const float obj[12], const float img[8], double f, double cx, double cy, P3PProblem& pr) {
    for (int i = 0; i < 4; i++) {
        pr.mu[i] = p3p_pixel(img[i * 2], cx, f);
        pr.mv[i] = p3p_pixel(img[i * 2 + 1], cy, f);
        pr.X[i][0] = obj[i * 3]; pr.X[i][1] = obj[i * 3 + 1]; pr.X[i][2] = obj[i * 3 + 2];
    }
}

DSAC_HDN bool minimal_set_hypothesis(const float obj[12], const float img[8], double f, double cx, double cy, int thr,
                                     double rvec[3], double tvec[3], bool* fragile) {
    P3PProblem pr;
    make_problem(obj, img, f, cx, cy, pr);
    return minimal_set_hypothesis_pr(pr, obj, img, f, cx, cy, thr, rvec, tvec, fragile);
}

// Self-contained (fully inlined, register-resident) version of the conservative filter: same contract as
// p3p_quick_needs_full, but it does not share the front end with the full solve, so every decision the
// front end takes (degeneracy tests, existence of real roots) is protected by a tolerance band instead.
// DSAC_FLAG(k): "needs the full solve", k = which guard fired (counted only in the host statistics build)
#if defined(DSAC_FILTER_STATS) && !defined(__CUDA_ARCH__)
static long long g_filter_reason[24];
static double g_filter_fp32_maxdev = 0;
#define DSAC_FLAG(k) (g_filter_reason[k]++, true)
#else
#define DSAC_FLAG(k) true
#endif
#ifndef DSAC_FILTER_FP32_TAIL
#define DSAC_FILTER_FP32_TAIL 1        /* 4th-point stage of the conservative filter in fp32 with a widened band (else fp64) */
#endif
#ifndef DSAC_FILTER_FP32_BAND
#define DSAC_FILTER_FP32_BAND 0.25     /* px: candidates whose 4th point lands within thr + 0.25 px go to the full solve */
#endif
#define DSAC_U32 5.9604645e-8f         /* 2^-24: unit roundoff of fp32 */
#define DSAC_TAIL_EPS 4.6e-7f          /* 1e-7 (depth accuracy, f7) + 6 u: relative error of a camera point the tail forms */
#define DSAC_TAIL_MARGIN 0.05          /* px: headroom beyond thr + the fp32 tail's error bound (not derived: see the tail) */
// Core of the filter on prepared inputs: unit bearings of points 0..2, the four scene coordinates and the pixel
// (mu3, mv3) of the 4th point as P3P sees it (k_sample keeps 1/|(u, v, 1)| per cell in shared memory).
//
// Lambda Twist (Persson & Nordberg, ECCV 2018), written from the published algorithm.  With a_ij = |X_i - X_j|^2 and
// b_ij = bear_i . bear_j the depths lambda of points 0..2 solve E_ij: l_i^2 + l_j^2 - 2 b_ij l_i l_j = a_ij.
//   a12 E01 - a01 E12 and a12 E02 - a02 E12 cancel the right-hand sides: two homogeneous conics l^T D1 l = l^T D2 l = 0
//   (below divided by a12: A01 = a01 / a12, A02 = a02 / a12).
//   A real root g of the cubic det(D1 + g D2) makes D0 = D1 + g D2 singular, and every solution lies on D0.  Its
//   2 x 2 minors decide what D0 is: two real planes through its null vector (P = d01^2 - d00 d11 >= 0, Q = d02^2 - d00 d22
//   >= 0, P Q = m^2), or a single real direction, the null vector (P, Q <= 0).
//   Two planes: d00 l0 = (-d01 +- alpha) l1 + (-d02 +- beta) l2 with (alpha l1 + beta l2)^2 = P l1^2 + 2 m l1 l2 + Q l2^2.
//   Each plane substituted into a second conic of the pencil (D2, or D1 where |g| > 1 makes D0 close to g D2) gives a
//   quadratic in tau = l1 / l2; then l2 = sqrt(a12 / (tau^2 - 2 b12 tau + 1)), l1 = tau l2, l0 from the plane.
// So one cubic, one 2 x 2 split and one quadratic per plane: no quartic and no y-from-x division.  The exact solve (Gao's
// quartic, p3p_front / p3p_full) finds the same real solutions x = l0 / l2, y = l1 / l2 with x, y > 0.
//
// BRANCH-FREE on purpose.  One thread filters one candidate, and the candidates of a warp differ in everything that a
// branch could test (number of real solutions, their signs, degeneracy): with early exits the warp ran at 16 of 32 lanes
// (profiled with Nsight Compute).  Every test below therefore only sets a flag; root slots 0 and 1 are evaluated by all
// lanes (slots >= nroots are masked) and the verdict is the OR of the flags.  A NaN or infinity anywhere makes the
// comparison it reaches fail, and every comparison is written so that failing means "needs the full solve".
// Flag k: the guard DSAC_FLAG(k) of the statistics build (tools/filter_stats.py).
DSAC_HD bool p3p_lambda_core(const double bear[3][3], const double X[4][3], double mu3, double mv3, double f, double cx,
                             double cy, double thr) {
    const double ax = X[1][0] - X[0][0], ay = X[1][1] - X[0][1], az = X[1][2] - X[0][2];
    const double bx = X[2][0] - X[0][0], by = X[2][1] - X[0][1], bz = X[2][2] - X[0][2];
    const double gx = X[2][0] - X[1][0], gy = X[2][1] - X[1][1], gz = X[2][2] - X[1][2];
    const double s01 = ax * ax + ay * ay + az * az, s02 = bx * bx + by * by + bz * bz, s12 = gx * gx + gy * gy + gz * gz;
    const double nx = ay * bz - az * by, ny = az * bx - ax * bz, nz = ax * by - ay * bx;
    const double nn = nx * nx + ny * ny + nz * nz;
    const bool g1 = (!(s01 > 0)) | (!(s12 > 0)) | (!(nn > 0));                          // (1) degenerate triangle
    // world triangle frame and the 4th point's coordinates in it (first, so that the scene coordinates are dead early)
    const double inv_d = filt_rsqrt(s01), inv_n = filt_rsqrt(nn);
    const double e1x = ax * inv_d, e1y = ay * inv_d, e1z = az * inv_d;
    const double e3x = nx * inv_n, e3y = ny * inv_n, e3z = nz * inv_n;
    const double e2x = e3y * e1z - e3z * e1y, e2y = e3z * e1x - e3x * e1z, e2z = e3x * e1y - e3y * e1x;
    const double wx = X[3][0] - X[0][0], wy = X[3][1] - X[0][1], wz = X[3][2] - X[0][2];
    const double alw = wx * e1x + wy * e1y + wz * e1z, bew = wx * e2x + wy * e2y + wz * e2z, gaw = wx * e3x + wy * e3y + wz * e3z;
#if !DSAC_FILTER_FP32_TAIL
    const double lim2 = (thr + DSAC_FILTER_BAND_PX) * (thr + DSAC_FILTER_BAND_PX);
#else
    const float b0x = (float)bear[0][0], b0y = (float)bear[0][1], b0z = (float)bear[0][2];
    const float b1x = (float)bear[1][0], b1y = (float)bear[1][1], b1z = (float)bear[1][2];
    const float b2x = (float)bear[2][0], b2y = (float)bear[2][1], b2z = (float)bear[2][2];
    const float inv_df = (float)inv_d, inv_nf = (float)inv_n, sa12f = (float)filt_sqrt(s12);
    const float alf = (float)alw, bef = (float)bew, gaf = (float)gaw, ff = (float)f, du3f = (float)(mu3 - cx), dv3f = (float)(mv3 - cy);
    const float lim2f = (float)((thr + DSAC_FILTER_FP32_BAND) * (thr + DSAC_FILTER_FP32_BAND));
    const bool illcond = !(nn > 1e-3 * s01 * s02);   // sin^2 of the world triangle's angle at point 0: cross products lose 1 / sin of their digits
    // Per-candidate factors of the bound dP3 = errA * Lam + errB on the fp32 tail's camera coordinates of the 4th point
    // (derived at the tail below): errA = eps (1 + 2 W (1 / d01 + (d01 + d02) / |n|)) + 5 u,
    // errB = u W (7.2 d01 d02 / |n| + 15.2), with W = |alpha| + |beta| + |gamma|.
    const float d01f = (float)s01 * inv_df, s02f = (float)s02, d02f = s02f * DSAC_RSQRTF_EARLY(s02f), Wf = fabsf(alf) + fabsf(bef) + fabsf(gaf);
    const float errA = DSAC_TAIL_EPS * (1.f + 2.f * Wf * (inv_df + (d01f + d02f) * inv_nf)) + 5.f * DSAC_U32;
    const float errB = DSAC_U32 * Wf * (7.2f * d01f * d02f * inv_nf + 15.2f), errL = errA * sa12f;
    // 1.25 de_zz = kf dP3 (2 |Z3| + |X3| + |Y3|) + |Z3| (kuf (|X3| + |Y3|) + kud |Z3|)
    const float kf = 1.25f * ff, kuf = 10.f * DSAC_U32 * ff, kud = 10.f * DSAC_U32 * (fabsf(du3f) + fabsf(dv3f));
    const float thrm = (float)(thr + DSAC_TAIL_MARGIN);
#endif
    const double b01 = bear[0][0] * bear[1][0] + bear[0][1] * bear[1][1] + bear[0][2] * bear[1][2];
    const double b02 = bear[0][0] * bear[2][0] + bear[0][1] * bear[2][1] + bear[0][2] * bear[2][2];
    const double b12 = bear[1][0] * bear[2][0] + bear[1][1] * bear[2][1] + bear[1][2] * bear[2][2];
    const double i12 = filt_rcp(s12), A01 = s01 * i12, A02 = s02 * i12;
    // det(D1 + g D2) = c3 g^3 + c2 g^2 + c1 g + c0
    const double sn = 1 - b12 * b12, u01 = 1 - b01 * b01, u02 = 1 - b02 * b02, k2 = 2 - 2 * b01 * b02 * b12;
    const double c3 = A02 * (A02 * sn - u02), c0 = A01 * (A01 * sn - u01), cr = 2 * A01 * A02 * sn;
    const double c2 = A02 * (A02 * sn - k2) + cr - A01 * u02 + u02;
    const double c1 = A01 * (A01 * sn - k2) + cr - A02 * u01 + u01;
    const double i3 = filt_rcp(c3);
    bool cubic_ok;
    const double g = cubic_first_root_seeded(c2 * i3, c1 * i3, c0 * i3, &cubic_ok);
    const bool g2 = (!(fabs(c3) > 1e-12 * (fabs(c2) + fabs(c1) + fabs(c0)))) | (!cubic_ok);   // (2) cubic not settled
    // D0 = D1 + g D2 (symmetric) and its 2 x 2 minors
    const double d00 = 1 + g, d01 = -b01, d02 = -g * b02, d11 = 1 - A01 - g * A02, d12 = b12 * (A01 + g * A02),
                 d22 = g * (1 - A02) - A01;
    const double P = d01 * d01 - d00 * d11, Q = d02 * d02 - d00 * d22, m = d01 * d02 - d00 * d12;
    // P, Q and the planes move by ~eps |D0|^2 / |S| under a relative error eps of D0's entries (|D0| = Frobenius norm): the
    // sign of S and every quadratic discriminant below are decided only outside bands scaled by kappa = |D0|^2 / |S|
    const double S = P + Q, F2 = d00 * d00 + d11 * d11 + d22 * d22 + 2 * (d01 * d01 + d02 * d02 + d12 * d12);
    const bool g3 = !(fabs(S) > 1e-9 * F2);                                              // (3) planes or none
    const bool planes = S > 0;
    const bool pP = fabs(P) >= fabs(Q);
    const double pv = fabs(pP ? P : Q), ir = filt_rsqrt(pv), sq = pv * ir, mr = m * ir;
    const double al = pP ? sq : mr, be = pP ? mr : sq;
    const bool g4 = planes & !(fabs(d00) > 1e-4 * (fabs(d01) + fabs(d02) + sq + fabs(mr)));   // (4) small pivot d00
    const double id0 = filt_rcp(d00);
    const double wA0 = (al - d01) * id0, wA1 = (be - d02) * id0, wB0 = (-al - d01) * id0, wB1 = (-be - d02) * id0;
    // the second conic, e00 = 1
    const bool big = fabs(g) > 1;
    const double e01 = big ? -b01 : 0., e02 = big ? 0. : -b02, e11 = big ? 1 - A01 : -A02, e12 = b12 * (big ? A01 : A02),
                 e22 = big ? -A01 : 1 - A02;
    // per plane: qa tau^2 + 2 hb tau + qc = 0
    auto plane_quadratic = [&](double w0, double w1, double q[3], bool* real, bool* unc) {
        q[0] = w0 * (w0 + 2 * e01) + e11;
        q[1] = w0 * (w1 + e02) + e01 * w1 + e12;
        q[2] = w1 * (w1 + 2 * e02) + e22;
        const double disc = q[1] * q[1] - q[0] * q[2];
        *unc = !(fabs(disc) * fabs(S) > 1e-9 * F2 * (q[1] * q[1] + fabs(q[0] * q[2])));   // |disc| > 1e-9 kappa (scale)
        *real = disc > 0;
    };
    // its roots as t / qa and qc / t with t = -hb - sign(hb) sqrt(disc)
    auto plane_roots = [&](const double q[3], double* t1, double* t2) {
        const double ad = fabs(q[1] * q[1] - q[0] * q[2]), sd = ad * filt_rsqrt(ad);
        const double t = -q[1] - copysign(sd, q[1]), r = filt_rcp(q[0] * t);
        *t1 = t * t * r;
        *t2 = q[2] * q[0] * r;
    };
    double qA[3], qB[3];
    bool realA, realB, uncA, uncB;
    plane_quadratic(wA0, wA1, qA, &realA, &uncA);
    plane_quadratic(wB0, wB1, qB, &realB, &uncB);
    const bool g5 = planes & (uncA | uncB);                                               // (5) tau discriminant ~ 0
    const bool hasA = planes & realA, hasB = planes & realB;
    const int nroots = (hasA ? 2 : 0) + (hasB ? 2 : 0);
    // no planes: the null vector of D0 is the only real direction left; it is a solution only if it lies on the second
    // conic as well (a tangency, i.e. a double root: flagged)
    const double v0 = pP ? d01 * d12 - d02 * d11 : d01 * d22 - d02 * d12, v1 = pP ? m : Q, v2 = pP ? -P : -m;
    const double vev = v0 * v0 + e11 * v1 * v1 + e22 * v2 * v2 + 2 * (e01 * v0 * v1 + e02 * v0 * v2 + e12 * v1 * v2);
    const double vsc = (v0 * v0 + v1 * v1 + v2 * v2) * (1 + fabs(e11) + fabs(e22) + fabs(e01) + fabs(e02) + fabs(e12));
    const bool g9 = (!planes) & !(fabs(vev) > 1e-7 * vsc);                                // (9) null vector on the conic
    bool flag = g1 | g2 | g3 | g4 | g5 | g9;
#if defined(DSAC_FILTER_STATS) && !defined(__CUDA_ARCH__)
    g_filter_reason[20 + nroots / 2]++;   // statistics build: candidates with 0 / 2 / 4 real solutions (the roofline's flop model)
    if (flag) g_filter_reason[g1 ? 1 : g2 ? 2 : g3 ? 3 : g4 ? 4 : g5 ? 5 : 9]++;
#endif
    // Two real solutions are the common case (one plane holds both, the other a complex pair), four are rare: slots 0 and 1
    // (plane A if it is real, else plane B) are evaluated by every lane, slots 2 and 3 (plane B) only by the lanes that
    // have them (a divergent branch few warps take).
    // slots 0, 1: plane A if it is real, else plane B; slots 2, 3: plane B
    const double wS0 = hasA ? wA0 : wB0, wS1 = hasA ? wA1 : wB1;
    const double qS[3] = {hasA ? qA[0] : qB[0], hasA ? qA[1] : qB[1], hasA ? qA[2] : qB[2]};
    double tau_s[4];
    plane_roots(qS, &tau_s[0], &tau_s[1]);
    auto root_slot = [&](int i) {
        const double tau = (i == 0) ? tau_s[0] : (i == 1) ? tau_s[1] : (i == 2) ? tau_s[2] : tau_s[3];
        const double w0 = (i < 2) ? wS0 : wB0, w1 = (i < 2) ? wS1 : wB1;
        // depths in units of sqrt(a12) (the E_ij divided by a12)
        const double L2 = filt_rsqrt(tau * (tau - 2 * b12) + 1), L1 = tau * L2, L0 = w0 * L1 + w1 * L2;
        // Accuracy of lambda without taking the Gauss-Newton step on the E_ij: with J / 2 = [[A, B, 0], [C, 0, D], [0, E, F]]
        // and residuals r, the step J^-1 r is at most 1.5 (n1 n2 + n1 n3 + n2 n3) |r|_1 / |det| in each coordinate (every
        // cofactor is a product of entries of two different rows, n_k = row sums of |entries|).
        const double A = L0 - b01 * L1, B = L1 - b01 * L0, C = L0 - b02 * L2, D = L2 - b02 * L0, E = L1 - b12 * L2,
                     F = L2 - b12 * L1;
        const double r01 = L0 * A + L1 * B - A01, r02 = L0 * C + L2 * D - A02, r12 = L1 * E + L2 * F - 1;
        const double n1 = fabs(A) + fabs(B), n2 = fabs(C) + fabs(D), n3 = fabs(E) + fabs(F);
        const double det = A * D * E + B * C * F;                      // -det(J / 2)
        const double Ls = fabs(L0) + fabs(L1) + fabs(L2);
        const bool f6 = !(fabs(det) > 1e-4 * n1 * n2 * n3);            // ill-conditioned Jacobian (NaN)
        const bool f7 = !(1.5 * (n1 * (n2 + n3) + n2 * n3) * (fabs(r01) + fabs(r02) + fabs(r12)) <= 1e-7 * fabs(det) * Ls);
        const bool neg = (L0 < -1e-6 * Ls) | (L1 < -1e-6 * Ls);       // certainly a non-physical solution: it decides nothing
        const bool f8 = (L0 < 1e-6 * Ls) | (L1 < 1e-6 * Ls);          // borderline positivity
#if DSAC_FILTER_FP32_TAIL
        // The 4th point's camera position and pixel error in fp32 (FMA pipe, idle in this kernel) instead of fp64.  The result
        // decides only where the pixel error exceeds thr by more than its error bound, derived here.  u = 2^-24, |.| are
        // 2-norms, lengths in mm, and "true" means the exact solve's pose for the same root.
        //  (a) Camera points P_i = l_i b_i.  The depths are within 1e-7 Lam of the root (Lam = l0 + l1 + l2): f7 bounds the
        //      Gauss-Newton step on the distance equations, a first-order estimate of the depth error, not an enclosure of
        //      the root (its remainder is quadratic in a step below 1e-7).  The fp32 roundings of L_i, sqrt(a12), the bearing
        //      and two products add 5 u l_i: |dP_i| <= eps Lam, eps = 1e-7 + 6 u.
        //  (b) u = P1 - P0, v = P2 - P0 (|u| = d01, |v| = d02): |du| <= 2 eps Lam + u d01, |dv| <= 2 eps Lam + u d02.
        //  (c) c1 = u / d01: |dc1| <= 2 eps Lam / d01 + 3 u (the roundings of inv_d and of the product add 2 u).
        //  (d) n = u x v, |n| = d01 d02 sin(theta): |dn| <= |du| d02 + d01 |dv| + 3 sqrt(3) u d01 d02
        //      <= 2 eps Lam (d01 + d02) + 7.2 u d01 d02, so c3 = n / |n|: |dc3| <= (2 eps Lam (d01 + d02) + 7.2 u d01 d02) / |n| + 2 u.
        //  (e) c2 = c3 x c1 (unit vectors): |dc2| <= |dc3| + |dc1| + 3 sqrt(3) u.
        //  (f) X3 = M0x + alpha c1x + beta c2x + gamma c3x, the same for Y3 and Z3, W = |alpha| + |beta| + |gamma|:
        //      |dX3| <= |dM0| + W max|dc_k| + u W (alpha .. gamma rounded to fp32) + 4 u (Lam + W) (three products, three sums)
        //      <= Lam (eps (1 + 2 W (1 / d01 + (d01 + d02) / |n|)) + 5 u) + u W (7.2 d01 d02 / |n| + 15.2) = errA Lam + errB = dP3.
        //      This is the term the triangle's size enters: a 5 mm triangle metres away from the camera and from its 4th point
        //      gives W / d01 ~ 10^3, and |dc_k| ~ 10^3 eps.
        //  (g) Pixel error e = |(f X3 / Z3 - du3, f Y3 / Z3 - dv3)|: |d(f X3 / Z3)| <= f (|dX3| + |X3 / Z3| |dZ3|) / |Z3|.
        //      gu = f X3 - du3 Z3 rounds ff, du3f, two products and a difference: 3 u (f |X3| + |du3| |Z3|); the norm
        //      sqrt(gu^2 + gv^2) adds 4 u of itself, which is <= 4 u (f (|X3| + |Y3|) + (|du3| + |dv3|) |Z3|).  Together
        //      |de| Z3^2 <= de_zz = f dP3 (2 |Z3| + |X3| + |Y3|) + 8 u |Z3| (f (|X3| + |Y3|) + (|du3| + |dv3|) |Z3|).
        //      Beyond first order in dP3: X'/Z' - X/Z = (Z dX - X dZ) / (Z Z'), so, given (a), the bound holds without a
        //      remainder once multiplied by |Z3| / (|Z3| - dP3) (dP3 < |Z3| / 2 required).
        // A 4th point counts as certainly off only if e - 1.25 |de| |Z3| / (|Z3| - dP3) > thr + DSAC_TAIL_MARGIN (multiplied
        // through by |Z3| (|Z3| - dP3) and squared: no division, no square root), on top of the band test
        // e > thr + DSAC_FILTER_FP32_BAND.  The factor 1.25 covers the rounding of the bound itself (sums and products of
        // positive terms: a few u relative).  DSAC_TAIL_MARGIN (0.05 px, the fp64 tail's DSAC_FILTER_BAND_PX) is not derived:
        // it is headroom for what the bound leaves out, the quadratic remainder of f7's estimate in (a) and the exact
        // solve's own fp64 error on its 4th-point error (~1e-12 px).  Otherwise the candidate is flagged.
        // The bound grows with f, with the 4th pixel's distance from the principal point (|X3|, |Y3| against |Z3|), and
        // with Lam and W against |Z3|: a 4th point close to the camera of a distant triangle is the dangerous case.
        const float Zf = (float)L2 * sa12f, L0f = (float)L0 * sa12f, L1f = (float)L1 * sa12f;
        const float M0x = L0f * b0x, M0y = L0f * b0y, M0z = L0f * b0z;
        const float ux = L1f * b1x - M0x, uy = L1f * b1y - M0y, uz = L1f * b1z - M0z;
        const float vx = Zf * b2x - M0x, vy = Zf * b2y - M0y, vz = Zf * b2z - M0z;
        const float cxn = uy * vz - uz * vy, cyn = uz * vx - ux * vz, czn = ux * vy - uy * vx;
        const float c1x = ux * inv_df, c1y = uy * inv_df, c1z = uz * inv_df;
        const float c3x = cxn * inv_nf, c3y = cyn * inv_nf, c3z = czn * inv_nf;
        const float c2x = c3y * c1z - c3z * c1y, c2y = c3z * c1x - c3x * c1z, c2z = c3x * c1y - c3y * c1x;
        const float X3 = M0x + alf * c1x + bef * c2x + gaf * c3x;
        const float Y3 = M0y + alf * c1y + bef * c2y + gaf * c3y;
        const float Z3 = M0z + alf * c1z + bef * c2z + gaf * c3z;
        const float gu = ff * X3 - du3f * Z3, gv = ff * Y3 - dv3f * Z3, zz = Z3 * Z3;
        const float aX = fabsf(X3) + fabsf(Y3), aZ = fabsf(Z3), dP3 = errL * (float)Ls + errB;
        const float de125 = kf * dP3 * (2.f * aZ + aX) + aZ * (kuf * aX + kud * aZ), tz = aZ - dP3;
        const float rin = thrm * aZ * tz + de125;
        // (g): |(gu, gv)| tz > (thr + margin) |Z3| tz + 1.25 de_zz, squared (both sides positive), and dP3 < |Z3| / 2
        const bool shallow = !(dP3 < tz) | !((gu * gu + gv * gv) * (tz * tz) > rin * rin);
        const bool f10 = (!(gu * gu + gv * gv > lim2f * zz)) | (!(zz > 0.f)) | shallow | illcond;
#if defined(DSAC_FILTER_STATS) && !defined(__CUDA_ARCH__)
        {   // statistics build: the same quantity in fp64, to record the largest deviation of the fp32 pixel error
            const double sa12 = sqrt(s12), l0 = L0 * sa12, l1 = L1 * sa12, l2 = L2 * sa12;
            const double m0x = l0 * bear[0][0], m0y = l0 * bear[0][1], m0z = l0 * bear[0][2];
            const double Ux = l1 * bear[1][0] - m0x, Uy = l1 * bear[1][1] - m0y, Uz = l1 * bear[1][2] - m0z;
            const double Vx = l2 * bear[2][0] - m0x, Vy = l2 * bear[2][1] - m0y, Vz = l2 * bear[2][2] - m0z;
            const double Cx = Uy * Vz - Uz * Vy, Cy = Uz * Vx - Ux * Vz, Cz = Ux * Vy - Uy * Vx;
            const double k1x = Ux * inv_d, k1y = Uy * inv_d, k1z = Uz * inv_d, k3x = Cx * inv_n, k3y = Cy * inv_n, k3z = Cz * inv_n;
            const double k2x = k3y * k1z - k3z * k1y, k2y = k3z * k1x - k3x * k1z, k2z = k3x * k1y - k3y * k1x;
            const double X3d = m0x + alw * k1x + bew * k2x + gaw * k3x, Y3d = m0y + alw * k1y + bew * k2y + gaw * k3y,
                         Z3d = m0z + alw * k1z + bew * k2z + gaw * k3z;
            const double e64 = sqrt((f * X3d / Z3d - (mu3 - cx)) * (f * X3d / Z3d - (mu3 - cx)) + (f * Y3d / Z3d - (mv3 - cy)) * (f * Y3d / Z3d - (mv3 - cy)));
            const double e32 = sqrt((double)(gu * gu + gv * gv)) / fabs((double)Z3);
            if (i < nroots && !neg && !(f6 | f7 | f8) && !shallow && !illcond && e64 < 200.0) {
                const double dev = fabs(e32 - e64);
                if (dev > g_filter_fp32_maxdev) g_filter_fp32_maxdev = dev;
            }
        }
#endif
#else
        const double sa12 = filt_sqrt(s12), l0 = L0 * sa12, l1 = L1 * sa12, l2 = L2 * sa12;
        const double M0x = l0 * bear[0][0], M0y = l0 * bear[0][1], M0z = l0 * bear[0][2];
        const double ux = l1 * bear[1][0] - M0x, uy = l1 * bear[1][1] - M0y, uz = l1 * bear[1][2] - M0z;
        const double vx = l2 * bear[2][0] - M0x, vy = l2 * bear[2][1] - M0y, vz = l2 * bear[2][2] - M0z;
        const double cxn = uy * vz - uz * vy, cyn = uz * vx - ux * vz, czn = ux * vy - uy * vx;
        const double c1x = ux * inv_d, c1y = uy * inv_d, c1z = uz * inv_d;
        const double c3x = cxn * inv_n, c3y = cyn * inv_n, c3z = czn * inv_n;
        const double c2x = c3y * c1z - c3z * c1y, c2y = c3z * c1x - c3x * c1z, c2z = c3x * c1y - c3y * c1x;
        const double X3 = M0x + alw * c1x + bew * c2x + gaw * c3x;
        const double Y3 = M0y + alw * c1y + bew * c2y + gaw * c3y;
        const double Z3 = M0z + alw * c1z + bew * c2z + gaw * c3z;
        // |(cx + f X3 / Z3 - mu3, cy + f Y3 / Z3 - mv3)|^2 > lim2, multiplied through by Z3^2 (no division)
        const double gu = f * X3 - (mu3 - cx) * Z3, gv = f * Y3 - (mv3 - cy) * Z3, zz = Z3 * Z3;
        const bool f10 = (!(gu * gu + gv * gv > lim2 * zz)) | (!(zz > 0));
#endif
        const bool root_flag = f6 | f7 | ((!neg) & (f8 | f10));
#if defined(DSAC_FILTER_STATS) && !defined(__CUDA_ARCH__)
        if (!flag && i < nroots && root_flag) g_filter_reason[f6 ? 6 : f7 ? 7 : f8 ? 8 : 10]++;
#endif
        flag |= (i < nroots) & root_flag;
    };
    root_slot(0);
    root_slot(1);
    if (nroots > 2) {
        plane_roots(qB, &tau_s[2], &tau_s[3]);
        root_slot(2);
        root_slot(3);
    }
    return flag;
}

DSAC_HD bool p3p_quick_inline(const P3PProblem& pr, double f, double cx, double cy, double inv_f, double thr) {
    const double cx_f = cx * inv_f, cy_f = cy * inv_f;
    double bear[3][3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        double u = inv_f * pr.mu[i] - cx_f, v = inv_f * pr.mv[i] - cy_f;
#if defined(__CUDA_ARCH__)
        double k = rsqrt(u * u + v * v + 1);
#else
        double k = 1. / sqrt(u * u + v * v + 1);
#endif
        bear[i][0] = u * k; bear[i][1] = v * k; bear[i][2] = k;
    }
    return p3p_lambda_core(bear, pr.X, pr.mu[3], pr.mv[3], f, cx, cy, thr);
}

// ---------------------------------------------------------------------------------------
// fp32 version of the conservative filter.  Same decision contract as p3p_quick_needs_full
// ("false" only if the candidate is certainly rejected), but every quantity whose rounding
// could matter is guarded by a tolerance band three or more orders of magnitude wider than
// fp32 rounding, and anything inside a band is handed to the fp64 full solve:
//   * existence of real quartic roots (R^2, D^2, E^2 of Ferrari's method near zero),
//   * the linear relation for y (denominator near zero),
//   * Newton convergence / conditioning of the two-quadric system,
//   * positivity of x, y, v,
//   * the 4th point's error within 10 px of the threshold.
// The quartic's coefficients are formed in double from the fp32 geometry (60 flops) so the
// roots are those of a nearby well-posed problem; root finding and the per-root work are fp32.
#if defined(__CUDA_ARCH__)
#define DSAC_RSQRTF(x) rsqrtf(x)
#else
#define DSAC_RSQRTF(x) (1.0f / sqrtf(x))
#endif

DSAC_HD float cubic_first_root_f32(float a2, float a1, float a0) {
    float Q = (3 * a1 - a2 * a2) * (1.f / 9);
    float R = (9 * a2 * a1 - 27 * a0 - 2 * a2 * a2 * a2) * (1.f / 54);
    float Q3 = Q * Q * Q, D = Q3 + R * R, sh = a2 * (1.f / 3);
    float y;
    if (D <= 0 && Q < 0) {
        float c = R * DSAC_RSQRTF(-Q3);
        c = fminf(1.f, fmaxf(-1.f, c));
        y = 2 * sqrtf(-Q) * cosf(acosf(c) * (1.f / 3)) - sh;
    } else {
        float AD = cbrtf(fabsf(R) + sqrtf(fmaxf(D, 0.f)));
        AD = (R >= 0) ? AD : -AD;
        float BD = (AD == 0) ? 0 : -Q / AD;
        y = AD + BD - sh;
    }
    // one Newton step on the cubic removes most of the closed form's rounding
    float g = ((y + a2) * y + a1) * y + a0, gp = (3 * y + 2 * a2) * y + a1;
    if (gp != 0) y -= g / gp;
    return y;
}

// returns true if the candidate needs the fp64 full solve
#define DSAC_F32_FLAG(code) { if (reason) *reason = (code); return true; }
DSAC_HDN bool minimal_set_needs_full_f32(const float obj[12], const float img[8], double fd, double cxd, double cyd, int thr,
                                        int* reason = nullptr) {
    const float f = (float)fd, cx = (float)cxd, cy = (float)cyd, inv_f = 1.f / f;
    float bear[3][3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        float u = (img[i * 2] - cx) * inv_f, v = (img[i * 2 + 1] - cy) * inv_f;
        float k = DSAC_RSQRTF(u * u + v * v + 1);
        bear[i][0] = u * k; bear[i][1] = v * k; bear[i][2] = k;
    }
    const float u3 = img[6], v3 = img[7];
    float ax = obj[3] - obj[0], ay = obj[4] - obj[1], az = obj[5] - obj[2];      // X1 - X0
    float bx = obj[6] - obj[0], by = obj[7] - obj[1], bz = obj[8] - obj[2];      // X2 - X0
    float cxx = obj[6] - obj[3], cyy = obj[7] - obj[4], czz = obj[8] - obj[5];   // X2 - X1
    float s01 = ax * ax + ay * ay + az * az, s02 = bx * bx + by * by + bz * bz, s12 = cxx * cxx + cyy * cyy + czz * czz;
    float nx = ay * bz - az * by, ny = az * bx - ax * bz, nz = ax * by - ay * bx;
    float nn = nx * nx + ny * ny + nz * nz;
    if (!(s01 > 0) || !(nn > 1e-6f * s01 * s02)) DSAC_F32_FLAG(1)   // degenerate / nearly collinear triangle
    float inv01 = 1.f / s01;
    float af = s12 * inv01, bf = s02 * inv01;
    float pf = 2 * (bear[1][0] * bear[2][0] + bear[1][1] * bear[2][1] + bear[1][2] * bear[2][2]);
    float qf = 2 * (bear[0][0] * bear[2][0] + bear[0][1] * bear[2][1] + bear[0][2] * bear[2][2]);
    float rf = 2 * (bear[0][0] * bear[1][0] + bear[0][1] * bear[1][1] + bear[0][2] * bear[1][2]);
    float N2f, N1f, N0f, D1f, D0f, shift, P, Q, Rr;
    {
        double a = af, b = bf, p = pf, q = qf, r = rf;
        double N2 = 1 - a - b, N1 = q * (a - 1), N0 = 1 - a + b, D1 = b * r, D0 = -b * p;
        double F2 = 1 - b, F1 = -q;
        double DD2 = D1 * D1, DD1 = 2 * D1 * D0, DD0 = D0 * D0, br = b * r;
        double c4 = F2 * DD2 - b * (N2 * N2) - br * (N2 * D1);
        double c3 = F2 * DD1 + F1 * DD2 - b * (2 * N2 * N1) - br * (N2 * D0 + N1 * D1);
        double c2 = F2 * DD0 + F1 * DD1 + DD2 - b * (2 * N2 * N0 + N1 * N1) - br * (N1 * D0 + N0 * D1);
        double c1 = F1 * DD0 + DD1 - b * (2 * N1 * N0) - br * (N0 * D0);
        double c0 = DD0 - b * (N0 * N0);
        double sc = fabs(c4) + fabs(c3) + fabs(c2) + fabs(c1) + fabs(c0);
        if (!(fabs(c4) > 1e-6 * sc)) DSAC_F32_FLAG(2)   // leading coefficient (nearly) vanishes
        double i4 = 1.0 / c4;
        double B = c3 * i4, C = c2 * i4, D = c1 * i4, E = c0 * i4;
        // depressed quartic z^4 + P z^2 + Q z + Rr = 0, x = z - B/4: the roots cluster (x ~ 1), so the
        // shift is done in double and the fp32 root finder only sees the spread
        double B2 = B * B;
        shift = (float)(0.25 * B);
        P = (float)(C - 0.375 * B2);
        Q = (float)(D - 0.5 * B * C + 0.125 * B2 * B);
        Rr = (float)(E - 0.25 * B * D + 0.0625 * B2 * C - (3.0 / 256.0) * B2 * B2);
        N2f = (float)N2; N1f = (float)N1; N0f = (float)N0; D1f = (float)D1; D0f = (float)D0;
    }
    // ---- Ferrari on the depressed quartic in fp32, with a tolerance band on every sign decision.
    // scale of z: the bands are relative to it
    const float TOL = 4e-3f;
    float y1 = cubic_first_root_f32(-P, -4 * Rr, 4 * P * Rr - Q * Q);
    if (!(y1 == y1)) DSAC_F32_FLAG(3)
    float R2 = y1 - P, mR = fabsf(y1) + fabsf(P);
    if (R2 < -TOL * mR) return false;               // certainly no real roots
    if (!(R2 > TOL * mR)) DSAC_F32_FLAG(4)              // too close to call (includes the R ~ 0 branch)
    float R = sqrtf(R2);
    float uu = -2 * P - R2, vv = -2 * Q / R;
    float mD = 2 * fabsf(P) + R2 + fabsf(vv);
    float D2 = uu + vv, E2 = uu - vv;
    float xr[4];
    int n = 0;
    if (D2 > TOL * mD) {
        float Dq = sqrtf(D2);
        xr[0] = 0.5f * R + 0.5f * Dq - shift;
        xr[1] = xr[0] - Dq;
        n = 2;
    } else if (!(D2 < -TOL * mD)) DSAC_F32_FLAG(5)
    if (E2 > TOL * mD) {
        float Eq = sqrtf(E2);
        xr[n] = -0.5f * R + 0.5f * Eq - shift;
        xr[n + 1] = xr[n] - Eq;
        n += 2;
    } else if (!(E2 < -TOL * mD)) DSAC_F32_FLAG(6)
    if (n == 0) return false;

    // world frame and the 4th point's coordinates in it
    float inv_d = DSAC_RSQRTF(s01), inv_n = DSAC_RSQRTF(nn), d01 = s01 * inv_d;
    float e1x = ax * inv_d, e1y = ay * inv_d, e1z = az * inv_d;
    float e3x = nx * inv_n, e3y = ny * inv_n, e3z = nz * inv_n;
    float e2x = e3y * e1z - e3z * e1y, e2y = e3z * e1x - e3x * e1z, e2z = e3x * e1y - e3y * e1x;
    float wx = obj[9] - obj[0], wy = obj[10] - obj[1], wz = obj[11] - obj[2];
    float al = wx * e1x + wy * e1y + wz * e1z, be = wx * e2x + wy * e2y + wz * e2z, ga = wx * e3x + wy * e3y + wz * e3z;
    const float lim2 = ((float)thr + 10.f) * ((float)thr + 10.f);
    for (int i = 0; i < 4; i++) {
        if (i >= n) break;
        float x = xr[i];
        float Dn = D1f * x + D0f;
        if (!(fabsf(Dn) > 3e-2f * (fabsf(D1f * x) + fabsf(D0f)))) DSAC_F32_FLAG(7)
        float y = -((N2f * x + N1f) * x + N0f) / Dn;
        float dlast = 0;
#pragma unroll
        for (int it = 0; it < 2; it++) {
            float f1 = (1 - af) * y * y - af * x * x - pf * y + af * rf * x * y + 1;
            float f2 = (1 - bf) * x * x - bf * y * y - qf * x + bf * rf * x * y + 1;
            float j11 = -2 * af * x + af * rf * y, j12 = 2 * (1 - af) * y - pf + af * rf * x;
            float j21 = 2 * (1 - bf) * x - qf + bf * rf * y, j22 = -2 * bf * y + bf * rf * x;
            float det = j11 * j22 - j12 * j21;
            float jn = j11 * j11 + j12 * j12 + j21 * j21 + j22 * j22;
            if (!(fabsf(det) > 1e-2f * jn)) DSAC_F32_FLAG(8)
            float idet = 1.f / det;
            float dx = (f1 * j22 - f2 * j12) * idet, dy = (j11 * f2 - j21 * f1) * idet;
            x -= dx;
            y -= dy;
            dlast = fabsf(dx) + fabsf(dy);
        }
        if (!(dlast <= 1e-3f * (fabsf(x) + fabsf(y)))) DSAC_F32_FLAG(9)
        if (x < -1e-2f || y < -1e-2f) continue;     // certainly non-physical
        if (x < 1e-2f || y < 1e-2f) DSAC_F32_FLAG(10)
        float v = x * x + y * y - x * y * rf;
        if (!(v > 1e-4f * (x * x + y * y))) DSAC_F32_FLAG(11)
        float Z = d01 * DSAC_RSQRTF(v);
        float L0 = x * Z, L1 = y * Z;
        float M0x = L0 * bear[0][0], M0y = L0 * bear[0][1], M0z = L0 * bear[0][2];
        float ux = L1 * bear[1][0] - M0x, uy = L1 * bear[1][1] - M0y, uz = L1 * bear[1][2] - M0z;
        float vx = Z * bear[2][0] - M0x, vy = Z * bear[2][1] - M0y, vz = Z * bear[2][2] - M0z;
        float cxn = uy * vz - uz * vy, cyn = uz * vx - ux * vz, czn = ux * vy - uy * vx;
        float c1x = ux * inv_d, c1y = uy * inv_d, c1z = uz * inv_d;
        float c3x = cxn * inv_n, c3y = cyn * inv_n, c3z = czn * inv_n;
        float c2x = c3y * c1z - c3z * c1y, c2y = c3z * c1x - c3x * c1z, c2z = c3x * c1y - c3y * c1x;
        float X3 = M0x + al * c1x + be * c2x + ga * c3x;
        float Y3 = M0y + al * c1y + be * c2y + ga * c3y;
        float Z3 = M0z + al * c1z + be * c2z + ga * c3z;
        if (!(fabsf(Z3) > 1e-3f * (fabsf(X3) + fabsf(Y3) + 1.f))) DSAC_F32_FLAG(12)  // grazing projection
        float iz = 1.f / Z3;
        float du = cx + f * X3 * iz - u3, dv = cy + f * Y3 * iz - v3;
        float e2 = du * du + dv * dv;
        if (!(e2 > lim2)) DSAC_F32_FLAG(13)
    }
    return false;
}

// Quick conservative pre-test of a minimal set (see p3p_quick_needs_full).
DSAC_HD bool minimal_set_needs_full_pr(const P3PProblem& pr, double f, double cx, double cy, int thr) {
    return p3p_quick_inline(pr, f, cx, cy, 1.0 / f, (double)thr);
}
DSAC_HDN bool minimal_set_needs_full(const float obj[12], const float img[8], double f, double cx, double cy, int thr) {
    P3PProblem pr;
    make_problem(obj, img, f, cx, cy, pr);
    return minimal_set_needs_full_pr(pr, f, cx, cy, thr);
}

}  // namespace dsac
