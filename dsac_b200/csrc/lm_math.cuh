// lm_math.cuh -- the arithmetic of the refinement's Levenberg-Marquardt loop (cv::solvePnP CV_ITERATIVE with
// useExtrinsicGuess = CvLevMarq on the 6 pose parameters; call sites cnn_softam.h:708, :1144), written so that it
// compiles both as device code for k_refine (refine.cuh) and, with DSAC_HOST_ONLY, for the CPU-side checks in
// tests/test_host_math.py (the product itself never runs on the CPU).
#pragma once
#include "pose_math.cuh"

namespace dsac {

// Rodrigues Jacobian, 3x9 (row i = d vec(R)/d r_i), as cv::Rodrigues returns it.
DSAC_HDN void rodrigues_jac(const double r[3], double R[9], double J[27]) {
    double theta = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    if (theta < 2.220446049250313e-16) {
        for (int i = 0; i < 9; i++) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
        for (int i = 0; i < 27; i++) J[i] = 0;
        J[5] = J[15] = J[19] = -1;
        J[7] = J[11] = J[21] = 1;
        return;
    }
    double s, c;
#if defined(__CUDA_ARCH__)
    sincos(theta, &s, &c);
#else
    s = sin(theta); c = cos(theta);
#endif
    double c1 = 1.0 - c, itheta = 1.0 / theta;
    double rx = r[0] * itheta, ry = r[1] * itheta, rz = r[2] * itheta;
    double rrt[9] = {rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz};
    double r_x[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
    for (int k = 0; k < 9; k++) R[k] = c * ((k % 4 == 0) ? 1.0 : 0.0) + c1 * rrt[k] + s * r_x[k];
    const double drrt[27] = {rx + rx, ry, rz, ry, 0, 0, rz, 0, 0, 0, rx, 0, rx, ry + ry, rz, 0, rz, 0,
                             0, 0, rx, 0, 0, ry, rx, ry, rz + rz};
    const double d_r_x[27] = {0, 0, 0, 0, 0, -1, 0, 1, 0, 0, 0, 1, 0, 0, 0, -1, 0, 0, 0, -1, 0, 1, 0, 0, 0, 0, 0};
    for (int i = 0; i < 3; i++) {
        double ri = (i == 0) ? rx : (i == 1) ? ry : rz;
        double a0 = -s * ri, a1 = (s - 2 * c1 * itheta) * ri, a2 = c1 * itheta;
        double a3 = (c - s * itheta) * ri, a4 = s * itheta;
        for (int k = 0; k < 9; k++)
            J[i * 9 + k] = a0 * ((k % 4 == 0) ? 1.0 : 0.0) + a1 * rrt[k] + a2 * drrt[i * 9 + k] + a3 * r_x[k] +
                           a4 * d_r_x[i * 9 + k];
    }
}

// Solve (JtJ with diagonal * (1+lambda)) x = JtErr.  Cholesky when positive definite (the
// normal case), else minimum-norm solution through a Jacobi eigen-decomposition with
// cv::SVBkSb's threshold (CvLevMarq::step solves with an SVD).
DSAC_HDN void lm_solve6(const double* JtJ, const double* JtErr, double lambda, double x[6]) {
    double A[36];
    for (int i = 0; i < 36; i++) A[i] = JtJ[i];
    for (int i = 0; i < 6; i++) A[i * 7] *= 1. + lambda;
    double L[36];
    bool pd = true;
    for (int i = 0; i < 6 && pd; i++) {
        for (int j = 0; j <= i; j++) {
            double s = A[i * 6 + j];
            for (int k = 0; k < j; k++) s -= L[i * 6 + k] * L[j * 6 + k];
            if (i == j) {
                if (!(s > 1e-300)) { pd = false; break; }
                L[i * 6 + i] = sqrt(s);
            } else {
                L[i * 6 + j] = s / L[j * 6 + j];
            }
        }
    }
    if (pd) {
        double y[6];
        for (int i = 0; i < 6; i++) {
            double s = JtErr[i];
            for (int k = 0; k < i; k++) s -= L[i * 6 + k] * y[k];
            y[i] = s / L[i * 6 + i];
        }
        for (int i = 5; i >= 0; i--) {
            double s = y[i];
            for (int k = i + 1; k < 6; k++) s -= L[k * 6 + i] * x[k];
            x[i] = s / L[i * 6 + i];
        }
        // guard against a numerically singular factorisation
        bool finite = true;
        for (int i = 0; i < 6; i++)
            if (!(fabs(x[i]) < 1.7e308)) finite = false;
        if (finite) return;
    }
    // symmetric eigen-decomposition (cyclic Jacobi), pseudo-inverse
    double V[36];
    for (int i = 0; i < 6; i++)
        for (int j = 0; j < 6; j++) V[i * 6 + j] = (i == j) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 60; sweep++) {
        double off = 0;
        for (int p = 0; p < 5; p++)
            for (int q = p + 1; q < 6; q++) off += fabs(A[p * 6 + q]);
        if (off == 0.0) break;
        for (int p = 0; p < 5; p++)
            for (int q = p + 1; q < 6; q++) {
                double apq = A[p * 6 + q];
                if (apq == 0.0) continue;
                double theta = (A[q * 6 + q] - A[p * 6 + p]) / (2.0 * apq);
                double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 6; k++) {
                    double akp = A[k * 6 + p], akq = A[k * 6 + q];
                    A[k * 6 + p] = c * akp - s * akq;
                    A[k * 6 + q] = s * akp + c * akq;
                }
                for (int k = 0; k < 6; k++) {
                    double apk = A[p * 6 + k], aqk = A[q * 6 + k];
                    A[p * 6 + k] = c * apk - s * aqk;
                    A[q * 6 + k] = s * apk + c * aqk;
                }
                A[p * 6 + q] = A[q * 6 + p] = 0.0;
                for (int k = 0; k < 6; k++) {
                    double vkp = V[k * 6 + p], vkq = V[k * 6 + q];
                    V[k * 6 + p] = c * vkp - s * vkq;
                    V[k * 6 + q] = s * vkp + c * vkq;
                }
            }
    }
    double thr = 0;
    for (int i = 0; i < 6; i++) thr += fabs(A[i * 7]);
    thr *= 2.220446049250313e-16 * 2;
    for (int i = 0; i < 6; i++) x[i] = 0;
    for (int k = 0; k < 6; k++) {
        double w = A[k * 7];
        if (!(fabs(w) > thr)) continue;
        double d = 0;
        for (int i = 0; i < 6; i++) d += V[i * 6 + k] * JtErr[i];
        d /= w;
        for (int i = 0; i < 6; i++) x[i] += d * V[i * 6 + k];
    }
}

// CvLevMarq's damping factors exp(lambdaLg10 * log(10)), lambdaLg10 = -16..17, as glibc's exp() rounds them
// (the reference evaluates exactly this expression on the host); index lambdaLg10 + 16.
#define DSAC_LM_LAMBDA_TABLE                                                                                              \
    {9.999999999999965e-17, 9.999999999999942e-16, 9.999999999999987e-15, 9.999999999999962e-14, 9.999999999999974e-13,  \
     9.999999999999985e-12, 9.99999999999996e-11,  9.999999999999972e-10, 9.999999999999982e-09, 9.999999999999994e-08,  \
     9.999999999999987e-07, 9.99999999999998e-06,  9.999999999999991e-05, 0.0009999999999999994, 0.009999999999999995,   \
     0.09999999999999998,   1.0,                   10.000000000000002,    100.00000000000004,    1000.0000000000007,     \
     10000.00000000001,     100000.0000000002,     1000000.0000000013,    10000000.000000006,    100000000.00000018,     \
     1000000000.0000029,    10000000000.00004,     100000000000.00015,    1000000000000.0026,    10000000000000.037,     \
     100000000000000.12,    1000000000000005.9,    1.0000000000000034e+16, 1.000000000000001e+17}
#if defined(__CUDACC__) && !defined(DSAC_HOST_ONLY)
__constant__ double c_lm_lambda[34] = DSAC_LM_LAMBDA_TABLE;
#else
static const double c_lm_lambda[34] = DSAC_LM_LAMBDA_TABLE;
#endif

// Rare path of the damped solve (normal matrix not positive definite): kept out of line so that its local
// arrays do not cost the common path registers.  S = [21 upper-triangle JtJ | 6 JtErr].
DSAC_HDN DSAC_NOINLINE void lm_solve6_general(const double* S, double lambda, double x[6]) {
    double JtJ[36], JtErr[6];
    int k = 0;
    for (int a = 0; a < 6; a++)
        for (int b = a; b < 6; b++) {
            JtJ[a * 6 + b] = JtJ[b * 6 + a] = S[k];
            k++;
        }
    for (int a = 0; a < 6; a++) JtErr[a] = S[21 + a];
    lm_solve6(JtJ, JtErr, lambda, x);
}

// (JtJ with its diagonal scaled by 1 + lambda) x = JtErr, all in registers: Cholesky with one rsqrt per column
// (no division on the dependency chain); falls back to lm_solve6_general when a pivot is not positive or the
// solution is not finite.  S = [21 upper-triangle JtJ | 6 JtErr] in shared memory.
DSAC_HD void lm_solve6_fast(const double* S, double lambda, double x[6]) {
    double A[6][6];   // lower triangle used
    {
        int k = 0;
#pragma unroll
        for (int a = 0; a < 6; a++)
#pragma unroll
            for (int b = a; b < 6; b++) {
                A[b][a] = S[k];
                k++;
            }
    }
    const double damp = 1. + lambda;
    double inv[6];
    bool pd = true;
#pragma unroll
    for (int j = 0; j < 6; j++) {
        double s = A[j][j] * damp;
#pragma unroll
        for (int k = 0; k < j; k++) s -= A[j][k] * A[j][k];
        pd = pd && (s > 1e-300);
        inv[j] = rsqrt_or(s);
#pragma unroll
        for (int i = j + 1; i < 6; i++) {
            double v = A[i][j];
#pragma unroll
            for (int k = 0; k < j; k++) v -= A[i][k] * A[j][k];
            A[i][j] = v * inv[j];
        }
    }
    double y[6];
#pragma unroll
    for (int i = 0; i < 6; i++) {
        double s = S[21 + i];
#pragma unroll
        for (int k = 0; k < i; k++) s -= A[i][k] * y[k];
        y[i] = s * inv[i];
    }
#pragma unroll
    for (int i = 5; i >= 0; i--) {
        double s = y[i];
#pragma unroll
        for (int k = i + 1; k < 6; k++) s -= A[k][i] * x[k];
        x[i] = s * inv[i];
    }
    bool finite = pd;
#pragma unroll
    for (int i = 0; i < 6; i++) finite = finite && (fabs(x[i]) < 1.7e308);
    if (!finite) lm_solve6_general(S, lambda, x);
}

// cv::Rodrigues (vector -> matrix with Jacobian) spread over the lanes of one warp: lane L < 27 produces
// J[L] (row i = L / 9 = d/dr_i, column k = L % 9 = element of R), lanes < 9 also R[L].  Same formulas and
// operation order as the sequential rodrigues_jac above.
DSAC_HD void rodrigues_jac_warp(const double r[3], int lane, double* sR, double* sJ) {
    const int L = lane < 27 ? lane : 26;
    const int i = L / 9, k = L - 9 * i, a = k / 3, b = k - 3 * a;
    const double theta = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    const double eye = (a == b) ? 1.0 : 0.0;
    // [r]x element (a, b) = sgn * r_c with c = 3 - a - b:  (b - a) mod 3 == 1 -> -1, == 2 -> +1
    const int c = 3 - a - b, m = (b - a + 3) % 3;
    const double sgn = (a == b) ? 0.0 : (m == 1 ? -1.0 : 1.0);
    if (theta < 2.220446049250313e-16) {
        if (lane < 9) sR[lane] = eye;
        if (lane < 27) sJ[lane] = (a != b && c == i) ? sgn : 0.0;
        return;
    }
    double s, co;
#if defined(__CUDA_ARCH__)
    sincos(theta, &s, &co);
#else
    s = sin(theta); co = cos(theta);
#endif
    const double c1 = 1.0 - co, itheta = 1.0 / theta;
    const double rx = r[0] * itheta, ry = r[1] * itheta, rz = r[2] * itheta;
    const double ra = (a == 0) ? rx : (a == 1) ? ry : rz, rb = (b == 0) ? rx : (b == 1) ? ry : rz;
    const double rc = (c == 0) ? rx : (c == 1) ? ry : rz, ri = (i == 0) ? rx : (i == 1) ? ry : rz;
    const double rrt = ra * rb, r_x = (a == b) ? 0.0 : sgn * rc;
    const double drrt = ((a == i) ? rb : 0.0) + ((b == i) ? ra : 0.0);
    const double d_r_x = (a != b && c == i) ? sgn : 0.0;
    if (lane < 9) sR[lane] = co * eye + c1 * rrt + s * r_x;
    const double a0 = -s * ri, a1 = (s - 2 * c1 * itheta) * ri, a2 = c1 * itheta, a3 = (co - s * itheta) * ri, a4 = s * itheta;
    if (lane < 27) sJ[lane] = a0 * eye + a1 * rrt + a2 * drrt + a3 * r_x + a4 * d_r_x;
}

// CvLevMarq's state machine (modules/calib3d/src/compat_ptsetreg.cpp: STARTED -> CALC_J -> CHECK_ERR -> ...) for a
// caller that evaluates, per trial parameter vector, the squared error norm AND the normal equations in one pass:
//   sums of pass k go to buffer `next_buf()`; lm_advance() then decides.
// LM_SOLVE_NEWBASE: the trial (or, first, the initial vector) becomes the base: prev := param, buffer `cur` holds its
// normal equations; solve with the current damping and try base - x.  LM_SOLVE_KEEP: the trial was worse: same base
// and normal equations, more damping.  LM_DONE: param (the last trial) is the result.
struct LMState {
    int lambdaLg10 = -3, iters = 0, cur = 0;
    bool have_cur = false;
    double prevErr2 = 0;   // squared error norm at the base vector (CvLevMarq keeps prevErrNorm = its square root)
};
enum { LM_DONE = 0, LM_SOLVE_KEEP = 1, LM_SOLVE_NEWBASE = 2 };

DSAC_HD int lm_next_buf(const LMState& st) { return st.have_cur ? (st.cur ^ 1) : 0; }

// err2: squared error norm of the pass just made (at `param`); prev: the base vector.
// The reference compares square roots (errNorm > prevErrNorm, |param - prev| / |prev| < FLT_EPSILON); both tests are
// decided on the squares whenever those differ from equality by more than a few ulps (sqrt is monotone, the three
// roundings of the quotient are bounded by 2 ulps) and evaluated literally otherwise, so the decisions are identical
// while the sqrt / divide latency leaves the common path.
DSAC_HD int lm_advance(LMState& st, int buf, double err2, const double* param, const double* prev) {
    if (!st.have_cur) {   // CALC_J at the initial parameters
        st.have_cur = true;
        st.cur = buf;
        st.prevErr2 = err2;
        return LM_SOLVE_NEWBASE;
    }
    // CHECK_ERR at the trial parameters
    bool worse;
    if (err2 > st.prevErr2 * (1 + 4e-15)) worse = true;
    else if (!(err2 > st.prevErr2)) worse = false;          // a <= b (or NaN)  =>  !(sqrt(a) > sqrt(b))
    else worse = sqrt(err2) > sqrt(st.prevErr2);
    if (worse && ++st.lambdaLg10 <= 16) return LM_SOLVE_KEEP;
    st.lambdaLg10 = st.lambdaLg10 - 1 > -16 ? st.lambdaLg10 - 1 : -16;
    double dn = 0, pn = 0;
    for (int k = 0; k < 6; k++) {
        const double d = param[k] - prev[k];
        dn += d * d;
        pn += prev[k] * prev[k];
    }
    const double eps2pn = 1.4210854715202004e-14 * pn;      // FLT_EPSILON^2 = 2^-46, exact
    bool small;
    if (dn < eps2pn * (1 - 1e-14)) small = true;
    else if (dn > eps2pn * (1 + 1e-14)) small = false;
    else small = sqrt(dn) / sqrt(pn) < 1.1920928955078125e-07;
    if (++st.iters >= 20 || small) return LM_DONE;
    st.prevErr2 = err2;   // accepted: the pass just made is the next CALC_J
    st.cur = buf;
    return LM_SOLVE_NEWBASE;
}

// One point's contribution to v[0..20] (upper triangle of JtJ), v[21..26] (JtErr), v[27] (|err|^2) at the pose
// (R, param[3..5]) with dR/dr = J (cv::projectPoints' Jacobians dp/drvec, dp/dtvec for zero distortion).
DSAC_HD void lm_point_contrib(const double* R, const double* J, const double* param, double X, double Y, double Z, double pix_u,
                              double pix_v, double f, double cx, double cy, double* v) {
    double x = R[0] * X + R[1] * Y + R[2] * Z + param[3];
    double y = R[3] * X + R[4] * Y + R[5] * Z + param[4];
    double z = R[6] * X + R[7] * Y + R[8] * Z + param[5];
    z = z ? 1. / z : 1;
    x *= z;
    y *= z;
    const double eu = (x * f + cx) - pix_u;
    const double ev = (y * f + cy) - pix_v;
    v[27] += eu * eu + ev * ev;
    double ju[6], jv[6];
#pragma unroll
    for (int j = 0; j < 3; j++) {
        const double dx0 = X * J[j * 9 + 0] + Y * J[j * 9 + 1] + Z * J[j * 9 + 2];
        const double dy0 = X * J[j * 9 + 3] + Y * J[j * 9 + 4] + Z * J[j * 9 + 5];
        const double dz0 = X * J[j * 9 + 6] + Y * J[j * 9 + 7] + Z * J[j * 9 + 8];
        ju[j] = f * (z * (dx0 - x * dz0));
        jv[j] = f * (z * (dy0 - y * dz0));
    }
    ju[3] = f * z; ju[4] = 0; ju[5] = f * (-x * z);
    jv[3] = 0; jv[4] = f * z; jv[5] = f * (-y * z);
    int k = 0;
#pragma unroll
    for (int a = 0; a < 6; a++)
#pragma unroll
        for (int b = a; b < 6; b++) {
            v[k] += ju[a] * ju[b] + jv[a] * jv[b];
            k++;
        }
#pragma unroll
    for (int a = 0; a < 6; a++) v[21 + a] += ju[a] * eu + jv[a] * ev;
}

// The same for a camera of a multi-camera rig: (R, param) is the rig pose, and the point's rig-frame position goes through
// the camera's fixed extrinsic (Rc row-major, tc) before the projection; the Jacobian is the camera Jacobian chained
// through Rc.  With Rc = I and tc = 0 every product with Rc and every sum with tc is exact, so the contribution equals
// lm_point_contrib's bit for bit (up to the sign of zero terms).
DSAC_HD void lm_point_contrib_ext(const double* R, const double* J, const double* param, const double* Rc, const double* tc, double X,
                                  double Y, double Z, double pix_u, double pix_v, double f, double cx, double cy, double* v) {
    const double xr = R[0] * X + R[1] * Y + R[2] * Z + param[3];
    const double yr = R[3] * X + R[4] * Y + R[5] * Z + param[4];
    const double zr = R[6] * X + R[7] * Y + R[8] * Z + param[5];
    double x = Rc[0] * xr + Rc[1] * yr + Rc[2] * zr + tc[0];
    double y = Rc[3] * xr + Rc[4] * yr + Rc[5] * zr + tc[1];
    double z = Rc[6] * xr + Rc[7] * yr + Rc[8] * zr + tc[2];
    z = z ? 1. / z : 1;
    x *= z;
    y *= z;
    const double eu = (x * f + cx) - pix_u;
    const double ev = (y * f + cy) - pix_v;
    v[27] += eu * eu + ev * ev;
    double ju[6], jv[6];
#pragma unroll
    for (int j = 0; j < 3; j++) {
        const double ax = X * J[j * 9 + 0] + Y * J[j * 9 + 1] + Z * J[j * 9 + 2];
        const double ay = X * J[j * 9 + 3] + Y * J[j * 9 + 4] + Z * J[j * 9 + 5];
        const double az = X * J[j * 9 + 6] + Y * J[j * 9 + 7] + Z * J[j * 9 + 8];
        const double dx0 = Rc[0] * ax + Rc[1] * ay + Rc[2] * az;
        const double dy0 = Rc[3] * ax + Rc[4] * ay + Rc[5] * az;
        const double dz0 = Rc[6] * ax + Rc[7] * ay + Rc[8] * az;
        ju[j] = f * (z * (dx0 - x * dz0));
        jv[j] = f * (z * (dy0 - y * dz0));
    }
#pragma unroll
    for (int k = 0; k < 3; k++) {   // d(camera point)/dt = column k of Rc
        ju[3 + k] = f * (z * (Rc[k] - x * Rc[6 + k]));
        jv[3 + k] = f * (z * (Rc[3 + k] - y * Rc[6 + k]));
    }
    int k = 0;
#pragma unroll
    for (int a = 0; a < 6; a++)
#pragma unroll
        for (int b = a; b < 6; b++) {
            v[k] += ju[a] * ju[b] + jv[a] * jv[b];
            k++;
        }
#pragma unroll
    for (int a = 0; a < 6; a++) v[21 + a] += ju[a] * eu + jv[a] * ev;
}

}  // namespace dsac
