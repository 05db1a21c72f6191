// ift.cuh -- implicit-function derivatives of a fitted pose with respect to its scene coordinates
// (dsac_set_coord_derivatives(DSAC_DERIV_IMPLICIT)): the per-point and 6x6 arithmetic, shared by the kernels in
// backward.cuh and the host build of the tests.
//
// A fitted pose theta* is a stationary point of E(theta) = sum_i |r_i(theta, Y_i)|^2 over the cells the fit used:
//   RGB    r_i = pi(R Y_i + t) - p_i     (pi: pinhole projection with the frame's camera, p_i the cell's pixel)
//   RGB-D  r_i = R Y_i + t - e_i         (e_i the cell's eye point)
// so d theta* / d Y_i = -H^-1 B_i with the full Hessian H = d2E / d theta2 (Gauss-Newton terms plus the residual
// curvature) and B_i = d2E / d theta dY_i (the common factor 2 cancels).  Both are evaluated in the chart
// R = exp([w]x) R*, t = t* + tau at the solution (xi = (w, tau) = 0), where
//   d/dw_a exp([w]x) q = e_a x q,   d2/dw_a dw_b exp([w]x) q = (e_a q_b + e_b q_a) / 2 - delta_ab q.
// The derivative is reported in the jp 6-vector of jp6_from_cv_dev (rodrigues(D R), D t, D = diag(1, -1, -1)):
// D exp([w]x) R* = exp([D w]x) D R*, so d jp6 / d xi = blockdiag(Jl^-1(r_jp) D, D) with Jl^-1 the inverse left Jacobian of
// SO(3) -- the matrix->vector Rodrigues Jacobian contracted with the left perturbation, in a form that stays accurate
// at the jp rotation of an ordinary pose, whose angle is near pi.
// The same fit also gives the pose covariance of dsac_pose_uncertainty_device (ift_fit_covariance; uncertainty.cuh): the
// Gauss-Newton information sum_i J_i^T J_i in the same chart, inverted and scaled by the residual variance.
#pragma once
#include "pose_math.cuh"
#include "rigid.cuh"

namespace dsac {

// Residual geometry of one point at the solution: q = R Y, X = q + t, the residual r, the gradients g_m = dr_m/dX of its
// components, Gs = sum_m r_m d2r_m/dX2 and gs = sum_m r_m g_m.
struct IftPoint {
    double q[3], r[3], g[3][3], Gs[6], gs[3];   // Gs: 00 01 02 11 12 22; RGB: r[2] = 0, g[2] = 0
};

// e: the pixel (u, v) for RGB, the eye point for RGB-D
DSAC_HD void ift_point_setup(const double R[9], const double t[3], const double Y[3], const double e[3], double f, double cx,
                             double cy, bool rgbd, IftPoint& P) {
    double X[3];
    for (int k = 0; k < 3; k++) {
        P.q[k] = R[k * 3] * Y[0] + R[k * 3 + 1] * Y[1] + R[k * 3 + 2] * Y[2];
        X[k] = P.q[k] + t[k];
    }
    if (rgbd) {
        for (int m = 0; m < 3; m++) {
            for (int k = 0; k < 3; k++) P.g[m][k] = m == k ? 1.0 : 0.0;
            P.gs[m] = X[m] - e[m];
            P.r[m] = P.gs[m];
        }
        for (int k = 0; k < 6; k++) P.Gs[k] = 0;
    } else {
        const double iz = 1.0 / X[2];
        const double r0 = f * X[0] * iz + cx - e[0], r1 = f * X[1] * iz + cy - e[1];
        P.r[0] = r0; P.r[1] = r1; P.r[2] = 0;
        P.g[0][0] = f * iz; P.g[0][1] = 0; P.g[0][2] = -f * X[0] * iz * iz;
        P.g[1][0] = 0; P.g[1][1] = f * iz; P.g[1][2] = -f * X[1] * iz * iz;
        for (int k = 0; k < 3; k++) { P.g[2][k] = 0; P.gs[k] = r0 * P.g[0][k] + r1 * P.g[1][k]; }
        P.Gs[0] = 0; P.Gs[1] = 0; P.Gs[2] = -r0 * f * iz * iz;
        P.Gs[3] = 0; P.Gs[4] = -r1 * f * iz * iz;
        P.Gs[5] = 2 * f * iz * iz * iz * (r0 * X[0] + r1 * X[1]);
    }
}

// dX / dxi_a: e_a x q (rotation), e_a (translation)
DSAC_HD void ift_dX(const double q[3], int a, double d[3]) {
    d[0] = d[1] = d[2] = 0;
    if (a >= 3) { d[a - 3] = 1; return; }
    const int b = (a + 1) % 3, c = (a + 2) % 3;
    d[c] = q[b];
    d[b] = -q[c];
}

DSAC_HD double ift_quad(const double Gs[6], const double u[3], const double v[3]) {
    const double w0 = Gs[0] * v[0] + Gs[1] * v[1] + Gs[2] * v[2];
    const double w1 = Gs[1] * v[0] + Gs[3] * v[1] + Gs[4] * v[2];
    const double w2 = Gs[2] * v[0] + Gs[4] * v[1] + Gs[5] * v[2];
    return u[0] * w0 + u[1] * w1 + u[2] * w2;
}

// this point's term of the Hessian, added to H21 (upper triangle row by row: 00 01 .. 05 11 .. 55)
DSAC_HD void ift_point_hess(const IftPoint& P, double H21[21]) {
    double dX[6][3], J[3][6];
    for (int a = 0; a < 6; a++) ift_dX(P.q, a, dX[a]);
    for (int m = 0; m < 3; m++)
        for (int a = 0; a < 6; a++) J[m][a] = P.g[m][0] * dX[a][0] + P.g[m][1] * dX[a][1] + P.g[m][2] * dX[a][2];
    const double gq = P.gs[0] * P.q[0] + P.gs[1] * P.q[1] + P.gs[2] * P.q[2];
    int k = 0;
    for (int a = 0; a < 6; a++)
        for (int b = a; b < 6; b++, k++) {
            double h = 0;
            for (int m = 0; m < 3; m++) h += J[m][a] * J[m][b];   // (RGB: row 2 of g is zero)
            h += ift_quad(P.Gs, dX[a], dX[b]);
            if (b < 3) h += 0.5 * (P.gs[a] * P.q[b] + P.gs[b] * P.q[a]) - (a == b ? gq : 0.0);
            H21[k] += h;
        }
}

// this point's Gauss-Newton term J^T J alone (J = dr / dxi), added to acc[0..20] in ift_point_hess' order, and |r|^2 to
// acc[21]: the information of a least-squares fit, whose residual-curvature terms vanish in expectation
DSAC_HD void ift_point_gn(const IftPoint& P, double acc[22]) {
    double dX[6][3], J[3][6];
    for (int a = 0; a < 6; a++) ift_dX(P.q, a, dX[a]);
    for (int m = 0; m < 3; m++)
        for (int a = 0; a < 6; a++) J[m][a] = P.g[m][0] * dX[a][0] + P.g[m][1] * dX[a][1] + P.g[m][2] * dX[a][2];
    int k = 0;
    for (int a = 0; a < 6; a++)
        for (int b = a; b < 6; b++, k++) acc[k] += J[0][a] * J[0][b] + J[1][a] * J[1][b] + J[2][a] * J[2][b];
    acc[21] += P.r[0] * P.r[0] + P.r[1] * P.r[1] + P.r[2] * P.r[2];
}

// B = d2E / dxi dY of this point (6 x 3, row-major)
DSAC_HD void ift_point_cross(const IftPoint& P, const double R[9], double B[18]) {
    double dX[6][3], J[3][6];
    for (int a = 0; a < 6; a++) ift_dX(P.q, a, dX[a]);
    for (int m = 0; m < 3; m++)
        for (int a = 0; a < 6; a++) J[m][a] = P.g[m][0] * dX[a][0] + P.g[m][1] * dX[a][1] + P.g[m][2] * dX[a][2];
    for (int j = 0; j < 3; j++) {
        const double c[3] = {R[j], R[3 + j], R[6 + j]};   // dX / dY_j
        double JY[3];
        for (int m = 0; m < 3; m++) JY[m] = P.g[m][0] * c[0] + P.g[m][1] * c[1] + P.g[m][2] * c[2];
        const double cg[3] = {c[1] * P.gs[2] - c[2] * P.gs[1], c[2] * P.gs[0] - c[0] * P.gs[2], c[0] * P.gs[1] - c[1] * P.gs[0]};
        for (int a = 0; a < 6; a++) {
            double s = 0;
            for (int m = 0; m < 3; m++) s += J[m][a] * JY[m];
            s += ift_quad(P.Gs, dX[a], c);
            if (a < 3) s += cg[a];   // gs . (e_a x c)
            B[a * 3 + j] = s;
        }
    }
}

// In-place Cholesky of the packed upper triangle H21 (H = U^T U, U stored in place).  False when H is not positive
// definite: a pivot below 1e-12 of its diagonal entry, or not finite.
DSAC_HD bool ift_chol6(double U[21]) {
    auto at = [](int i, int j) { return i * 6 - i * (i - 1) / 2 + (j - i); };
    for (int i = 0; i < 6; i++) {
        const double hii = U[at(i, i)];
        double d = hii;
        for (int k = 0; k < i; k++) d -= U[at(k, i)] * U[at(k, i)];
        if (!(d > 1e-12 * hii) || !(d < 1e300)) return false;
        d = sqrt(d);
        U[at(i, i)] = d;
        for (int j = i + 1; j < 6; j++) {
            double s = U[at(i, j)];
            for (int k = 0; k < i; k++) s -= U[at(k, i)] * U[at(k, j)];
            U[at(i, j)] = s / d;
        }
    }
    return true;
}

// x = H^-1 b with H = U^T U from ift_chol6
DSAC_HD void ift_chol6_solve(const double U[21], const double b[6], double x[6]) {
    auto at = [](int i, int j) { return i * 6 - i * (i - 1) / 2 + (j - i); };
    double y[6];
    for (int i = 0; i < 6; i++) {
        double s = b[i];
        for (int k = 0; k < i; k++) s -= U[at(k, i)] * y[k];
        y[i] = s / U[at(i, i)];
    }
    for (int i = 5; i >= 0; i--) {
        double s = y[i];
        for (int k = i + 1; k < 6; k++) s -= U[at(i, k)] * x[k];
        x[i] = s / U[at(i, i)];
    }
}

// Inverse left Jacobian of SO(3) at rotation vector r: I - [r]x / 2 + c [r]x^2, c = 1/th^2 - cot(th/2) / (2 th)
DSAC_HD void so3_jl_inv(const double r[3], double Ji[9]) {
    const double th2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2], th = sqrt(th2);
    const double c = th < 1e-4 ? 1.0 / 12 + th2 / 720 : 1.0 / th2 - cos(th / 2) / sin(th / 2) / (2 * th);
    const double K[9] = {0, -r[2], r[1], r[2], 0, -r[0], -r[1], r[0], 0};
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double k2 = 0;
            for (int k = 0; k < 3; k++) k2 += K[i * 3 + k] * K[k * 3 + j];
            Ji[i * 3 + j] = (i == j ? 1.0 : 0.0) - 0.5 * K[i * 3 + j] + c * k2;
        }
}

// Left Jacobian of SO(3) at rotation vector r: I + a [r]x + b [r]x^2, a = (1 - cos th) / th^2, b = (th - sin th) / th^3
DSAC_HD void so3_jl(const double r[3], double J[9]) {
    const double th2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2], th = sqrt(th2);
    const double a = th < 1e-4 ? 0.5 - th2 / 24 : (1 - cos(th)) / th2;
    const double b = th < 1e-4 ? 1.0 / 6 - th2 / 120 : (th - sin(th)) / (th2 * th);
    const double K[9] = {0, -r[2], r[1], r[2], 0, -r[0], -r[1], r[0], 0};
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double k2 = 0;
            for (int k = 0; k < 3; k++) k2 += K[i * 3 + k] * K[k * 3 + j];
            J[i * 3 + j] = (i == j ? 1.0 : 0.0) + a * K[i * 3 + j] + b * k2;
        }
}

// d r_out / d r of r_out = log(A exp([r]x)) for a fixed rotation A: exp([Jl(r) dr]x) exp([r]x) = exp([r + dr]x) to first
// order, and A exp([v]x) = exp([A v]x) A, so Jl(r_out) dr_out = A Jl(r) dr.  K = Jl(r_out)^-1 A Jl(r) (3 x 3).
DSAC_HD void so3_left_mul_jac(const double A[9], const double r[3], const double r_out[3], double K[9]) {
    double Jl[9], Ji[9], T[9];
    so3_jl(r, Jl);
    so3_jl_inv(r_out, Ji);
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) T[i * 3 + j] = A[i * 3] * Jl[j] + A[i * 3 + 1] * Jl[3 + j] + A[i * 3 + 2] * Jl[6 + j];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) K[i * 3 + j] = Ji[i * 3] * T[j] + Ji[i * 3 + 1] * T[3 + j] + Ji[i * 3 + 2] * T[6 + j];
}

// ---- multi-camera rigs (the rig backward, rig.cuh).  A camera's extrinsic (Rc, tc) maps rig coordinates to its own,
// X_cam = Rc X_rig + tc (pose_math.cuh's rig_compose / rig_lift).

// The rig pool's lift as a function of the camera hypothesis, L = d lift(T, E) / d T (6 x 6, row-major) in the cv 6-vector
// (rvec, tvec) in which the rig's soft-argmax averages its pool: lift (R, t) = (Rc^T R, Rc^T (t - tc)) has the rotation
// block so3_left_mul_jac(Rc^T) and the translation block Rc^T.  r: the hypothesis' rvec.  An extrinsic rotation that is
// exactly I (a zero rvec) gives L = I exactly, as the lift then keeps the hypothesis' rvec.
DSAC_HD void rig_lift_jac(const double Rc[9], const double r[3], double L[36]) {
    for (int k = 0; k < 36; k++) L[k] = 0;
    bool ident = true;
    for (int k = 0; k < 9; k++) ident = ident && Rc[k] == (k % 4 == 0 ? 1.0 : 0.0);
    if (ident) {
        for (int k = 0; k < 6; k++) L[k * 7] = 1;
        return;
    }
    double Rt[9], Rh[9], Rr[9], rr[3], K[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) Rt[i * 3 + j] = Rc[j * 3 + i];
    rodrigues_v2m(r, Rh);
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) Rr[i * 3 + j] = Rt[i * 3] * Rh[j] + Rt[i * 3 + 1] * Rh[3 + j] + Rt[i * 3 + 2] * Rh[6 + j];
    rodrigues_m2v(Rr, rr);
    so3_left_mul_jac(Rt, r, rr, K);
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            L[i * 6 + j] = K[i * 3 + j];
            L[(3 + i) * 6 + 3 + j] = Rt[i * 3 + j];
        }
}

// Camera c's pose of the pool slot that camera c2's hypothesis T = (Rh, th) (cv) lifts to, as a function of T, both in the
// jp 6-vector (rodrigues(D R), D t; D = diag(1, -1, -1)): T_c o lift(T, E_c2) = (A Rh, A th + b) with A = Rc Rc2^T, so
// K = d jp(T_c o lift(T, E_c2)) / d jp(T) (6 x 6) has the rotation block so3_left_mul_jac(D A D) at the jp rotation
// vectors and the translation block D A D.  same: c == c2, where the composition is T itself and K = I exactly.
DSAC_HD void rig_cross_jac(const double Rc[9], const double Rc2[9], const double Rh[9], bool same, double K[36]) {
    for (int k = 0; k < 36; k++) K[k] = 0;
    if (same) {
        for (int k = 0; k < 6; k++) K[k * 7] = 1;
        return;
    }
    double A[9], Aj[9], Rj[9], Ro[9], r[3], ro[3], Kr[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) A[i * 3 + j] = Rc[i * 3] * Rc2[j * 3] + Rc[i * 3 + 1] * Rc2[j * 3 + 1] + Rc[i * 3 + 2] * Rc2[j * 3 + 2];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            Aj[i * 3 + j] = ((i == 0) == (j == 0) ? 1.0 : -1.0) * A[i * 3 + j];   // D A D
            Rj[i * 3 + j] = (i == 0 ? 1.0 : -1.0) * Rh[i * 3 + j];                // D Rh
        }
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) Ro[i * 3 + j] = Aj[i * 3] * Rj[j] + Aj[i * 3 + 1] * Rj[3 + j] + Aj[i * 3 + 2] * Rj[6 + j];
    rodrigues_m2v(Rj, r);
    rodrigues_m2v(Ro, ro);
    so3_left_mul_jac(Aj, r, ro, Kr);
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            K[i * 6 + j] = Kr[i * 3 + j];
            K[(3 + i) * 6 + 3 + j] = Aj[i * 3 + j];
        }
}

// A rig's fit (k_refine_rig) over cells of several cameras: the residual of a cell of camera c is its camera-frame
// residual at X_cam = Rc X + tc, X = R Y + t in the rig frame.  The map is linear, so a point set up in its camera frame
// (ift_point_setup at the composed pose (Rc R, Rc t + tc)) becomes the rig frame's exactly: q = R Y = Rc^T q_cam,
// g_m -> Rc^T g_m, gs -> Rc^T gs, Gs -> Rc^T Gs Rc.  ift_point_hess and ift_point_cross (with the rig's R) then
// differentiate the rig pose.  An identity Rc changes no bit.
DSAC_HD void ift_point_to_rig(const double Rc[9], IftPoint& P) {
    double q[3];
    for (int k = 0; k < 3; k++) q[k] = P.q[0] * Rc[k] + P.q[1] * Rc[3 + k] + P.q[2] * Rc[6 + k];
    for (int k = 0; k < 3; k++) P.q[k] = q[k];
    for (int m = 0; m < 3; m++) {
        double g[3];
        for (int k = 0; k < 3; k++) g[k] = P.g[m][0] * Rc[k] + P.g[m][1] * Rc[3 + k] + P.g[m][2] * Rc[6 + k];
        for (int k = 0; k < 3; k++) P.g[m][k] = g[k];
    }
    double gs[3];
    for (int k = 0; k < 3; k++) gs[k] = P.gs[0] * Rc[k] + P.gs[1] * Rc[3 + k] + P.gs[2] * Rc[6 + k];
    const double G[9] = {P.Gs[0], P.Gs[1], P.Gs[2], P.Gs[1], P.Gs[3], P.Gs[4], P.Gs[2], P.Gs[4], P.Gs[5]};
    double T[9];   // G Rc
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) T[i * 3 + j] = G[i * 3] * Rc[j] + G[i * 3 + 1] * Rc[3 + j] + G[i * 3 + 2] * Rc[6 + j];
    auto at = [&](int i, int j) { return Rc[i] * T[j] + Rc[3 + i] * T[3 + j] + Rc[6 + i] * T[6 + j]; };   // (Rc^T G Rc)_ij
    P.Gs[0] = at(0, 0); P.Gs[1] = at(0, 1); P.Gs[2] = at(0, 2); P.Gs[3] = at(1, 1); P.Gs[4] = at(1, 2); P.Gs[5] = at(2, 2);
    for (int k = 0; k < 3; k++) P.gs[k] = gs[k];
}

// M = d jp6 / d xi (6 x 6, row-major) at the cv pose (rvec, tvec); R gets the cv rotation
DSAC_HD void ift_jp_jacobian(const double pose[6], double R[9], double M[36]) {
    rodrigues_v2m(pose, R);
    double Rj[9], rj[3], Ji[9];
    for (int k = 0; k < 9; k++) Rj[k] = k < 3 ? R[k] : -R[k];   // D R
    rodrigues_m2v(Rj, rj);
    so3_jl_inv(rj, Ji);
    for (int k = 0; k < 36; k++) M[k] = 0;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) M[i * 6 + j] = Ji[i * 3 + j] * (j == 0 ? 1.0 : -1.0);
    M[3 * 6 + 3] = 1; M[4 * 6 + 4] = -1; M[5 * 6 + 5] = -1;
}

// W = H^-1 M^T (6 x 6, row-major: W[a * 6 + k]) from the Cholesky factor of H
DSAC_HD void ift_weights(const double U[21], const double M[36], double W[36]) {
    for (int k = 0; k < 6; k++) {
        double b[6], x[6];
        for (int a = 0; a < 6; a++) b[a] = M[k * 6 + a];
        ift_chol6_solve(U, b, x);
        for (int a = 0; a < 6; a++) W[a * 6 + k] = x[a];
    }
}

// d jp6 / dY of one point, D[k * 3 + j] = -(W^T B)[k][j]
DSAC_HD void ift_point_deriv(const double W[36], const double B[18], double D[18]) {
    for (int k = 0; k < 6; k++)
        for (int j = 0; j < 3; j++) {
            double s = 0;
            for (int a = 0; a < 6; a++) s += W[a * 6 + k] * B[a * 3 + j];
            D[k * 3 + j] = -s;
        }
}

// The refinement's IFT over m cells (host form of k_refine_ift): Y [m][3], e [m][3] (pixels (u, v, -) or eye points),
// pose the cv pose.  D [m][6][3] = d jp6 / dY_i; false (D zero) when H is not positive definite or the result is not finite.
DSAC_HD bool ift_fit_deriv(int m, const double* Y, const double* e, const double pose[6], double f, double cx, double cy, bool rgbd,
                           double* D) {
    double R[9], M[36], H[21] = {0}, W[36];
    ift_jp_jacobian(pose, R, M);
    IftPoint P;
    for (int i = 0; i < m; i++) {
        ift_point_setup(R, pose + 3, Y + i * 3, e + i * 3, f, cx, cy, rgbd, P);
        ift_point_hess(P, H);
    }
    bool ok = m > 0 && ift_chol6(H);
    if (ok) ift_weights(H, M, W);
    for (int i = 0; i < m && ok; i++) {
        double B[18];
        ift_point_setup(R, pose + 3, Y + i * 3, e + i * 3, f, cx, cy, rgbd, P);
        ift_point_cross(P, R, B);
        ift_point_deriv(W, B, D + i * 18);
        for (int k = 0; k < 18; k++) ok = ok && D[i * 18 + k] - D[i * 18 + k] == 0.0;
    }
    if (!ok)
        for (int k = 0; k < m * 18; k++) D[k] = 0;
    return ok;
}

// Pose covariance of a least-squares fit over m cells from its Gauss-Newton information (the packed upper triangle
// `info`, factored in place) and its residual sum of squares rss: sigma2 = rss / dof, dof = 2m - 6 (RGB) or 3m - 6 (RGB-D),
// cov_xi = sigma2 info^-1 in the chart xi = (w, tau) of R = exp([w]x) R*, t = t* + tau, and cov_jp6 = M cov_xi M^T in the
// jp 6-vector (M = ift_jp_jacobian at the cv pose).  Both outputs are exactly symmetric.  False, with every output zero,
// when dof <= 0, ift_chol6 rejects the information or an output is not finite.
DSAC_HD bool ift_cov_from_info(double info[21], double rss, int m, bool rgbd, const double pose[6], double cov_xi[36],
                               double cov_jp6[36], double* sigma2) {
    const int dof = (rgbd ? 3 : 2) * m - 6;
    const double s2 = dof > 0 ? rss / dof : 0.0;
    bool ok = dof > 0 && ift_chol6(info);
    if (ok) {
        for (int k = 0; k < 6; k++) {   // column k of info^-1
            double b[6] = {0, 0, 0, 0, 0, 0}, x[6];
            b[k] = 1;
            ift_chol6_solve(info, b, x);
            for (int a = 0; a < 6; a++) cov_xi[a * 6 + k] = s2 * x[a];
        }
        for (int a = 0; a < 6; a++)
            for (int b = a + 1; b < 6; b++) cov_xi[a * 6 + b] = cov_xi[b * 6 + a] = 0.5 * (cov_xi[a * 6 + b] + cov_xi[b * 6 + a]);
        double R[9], M[36], T[36];
        ift_jp_jacobian(pose, R, M);
        for (int i = 0; i < 6; i++)
            for (int b = 0; b < 6; b++) {
                double s = 0;
                for (int a = 0; a < 6; a++) s += M[i * 6 + a] * cov_xi[a * 6 + b];
                T[i * 6 + b] = s;
            }
        for (int i = 0; i < 6; i++)
            for (int j = i; j < 6; j++) {
                double s = 0;
                for (int b = 0; b < 6; b++) s += T[i * 6 + b] * M[j * 6 + b];
                cov_jp6[i * 6 + j] = cov_jp6[j * 6 + i] = s;
            }
        ok = s2 - s2 == 0.0;
        for (int k = 0; k < 36; k++) ok = ok && cov_xi[k] - cov_xi[k] == 0.0 && cov_jp6[k] - cov_jp6[k] == 0.0;
    }
    if (!ok)
        for (int k = 0; k < 36; k++) cov_xi[k] = cov_jp6[k] = 0;
    *sigma2 = ok ? s2 : 0.0;
    return ok;
}

// The covariance of the refined pose over the m cells its last accepted step fitted (host form of k_pose_uncertainty):
// Y [m][3], e [m][3] (pixels (u, v, -) or eye points), pose the cv pose; outputs and false as ift_cov_from_info.
DSAC_HD bool ift_fit_covariance(int m, const double* Y, const double* e, const double pose[6], double f, double cx, double cy,
                                bool rgbd, double cov_xi[36], double cov_jp6[36], double* sigma2) {
    double R[9], acc[22] = {0};
    rodrigues_v2m(pose, R);
    IftPoint P;
    for (int i = 0; i < m; i++) {
        ift_point_setup(R, pose + 3, Y + i * 3, e + i * 3, f, cx, cy, rgbd, P);
        ift_point_gn(P, acc);
    }
    return ift_cov_from_info(acc, acc[21], m, rgbd, pose, cov_xi, cov_jp6, sigma2);
}

// Gaussian elimination with partial pivoting of A x = b for `nb` right-hand sides (A 6 x 6, b 6 x nb, both row-major,
// overwritten; x in b).  False when a pivot is below 1e-13 of the largest entry of A or not finite.
DSAC_HD bool ift_lu6_solve(double A[36], double* b, int nb) {
    double amax = 0;
    for (int k = 0; k < 36; k++) amax = fmax(amax, fabs(A[k]));
    for (int c = 0; c < 6; c++) {
        int piv = c;
        for (int r = c + 1; r < 6; r++)
            if (fabs(A[r * 6 + c]) > fabs(A[piv * 6 + c])) piv = r;
        if (!(fabs(A[piv * 6 + c]) > 1e-13 * amax) || !(amax < 1e300)) return false;
        if (piv != c) {
            for (int k = 0; k < 6; k++) { const double x = A[c * 6 + k]; A[c * 6 + k] = A[piv * 6 + k]; A[piv * 6 + k] = x; }
            for (int k = 0; k < nb; k++) { const double x = b[c * nb + k]; b[c * nb + k] = b[piv * nb + k]; b[piv * nb + k] = x; }
        }
        for (int r = c + 1; r < 6; r++) {
            const double l = A[r * 6 + c] / A[c * 6 + c];
            for (int k = c; k < 6; k++) A[r * 6 + k] -= l * A[c * 6 + k];
            for (int k = 0; k < nb; k++) b[r * nb + k] -= l * b[c * nb + k];
        }
    }
    for (int c = 5; c >= 0; c--)
        for (int k = 0; k < nb; k++) {
            double s = b[c * nb + k];
            for (int j = c + 1; j < 6; j++) s -= A[c * 6 + j] * b[j * nb + k];
            b[c * nb + k] = s / A[c * 6 + c];
        }
    return true;
}

// dPNP of a P3P hypothesis by the IFT: the pose (cv) satisfies pi(R X_k + t) = p_k for k = 0..2, six equations in six
// unknowns, so d xi / dX = -J_xi^-1 J_X.  X [3][3] scene points, uv [3][2] pixels.  out [6][12] = d jp6 / d(point, channel),
// the 4th point's columns zero; false (out zero) for a singular system or a non-finite result.
// col in 0..8: only that column is solved for and written (the others stay zero); -1: all nine.
DSAC_HD bool ift_dpnp_p3p(const double pose[6], const double X[9], const double uv[6], double f, double cx, double cy, double out[72],
                          int col = -1) {
    double R[9], M[36], A[36], b[6 * 9];
    ift_jp_jacobian(pose, R, M);
    for (int k = 0; k < 6 * 9; k++) b[k] = 0;
    for (int p = 0; p < 3; p++) {
        const double e[3] = {uv[p * 2], uv[p * 2 + 1], 0};
        IftPoint P;
        ift_point_setup(R, pose + 3, X + p * 3, e, f, cx, cy, false, P);
        for (int m = 0; m < 2; m++) {
            double dX[3];
            for (int a = 0; a < 6; a++) {
                ift_dX(P.q, a, dX);
                A[(p * 2 + m) * 6 + a] = P.g[m][0] * dX[0] + P.g[m][1] * dX[1] + P.g[m][2] * dX[2];
            }
            for (int j = 0; j < 3; j++)   // -dr / dY_j on the right-hand side
                if (col < 0) b[(p * 2 + m) * 9 + p * 3 + j] = -(P.g[m][0] * R[j] + P.g[m][1] * R[3 + j] + P.g[m][2] * R[6 + j]);
                else if (p * 3 + j == col) b[p * 2 + m] = -(P.g[m][0] * R[j] + P.g[m][1] * R[3 + j] + P.g[m][2] * R[6 + j]);
        }
    }
    const int nb = col < 0 ? 9 : 1;
    bool ok = ift_lu6_solve(A, b, nb);
    for (int k = 0; k < 72; k++) out[k] = 0;
    for (int i = 0; i < 6 && ok; i++)
        for (int c = 0; c < nb; c++) {
            double s = 0;
            for (int a = 0; a < 6; a++) s += M[i * 6 + a] * b[a * nb + c];
            out[i * 12 + (col < 0 ? c : col)] = s;
            ok = ok && s - s == 0.0;
        }
    if (!ok)
        for (int k = 0; k < 72; k++) out[k] = 0;
    return ok;
}

// dPNP of an RGB-D hypothesis by the IFT of the 3-point Kabsch fit, scene a [3][3] to eye b [3][3] (the fit at which it is
// evaluated is recomputed here); out [6][12] as ift_dpnp_p3p.
DSAC_HD bool ift_dpnp_kabsch(const double a[9], const double b[9], double out[72]) {
    double R[9], pose[6], D[3 * 18];
    kabsch_fit(3, a, b, R, pose + 3);
    rodrigues_m2v(R, pose);
    const bool ok = ift_fit_deriv(3, a, b, pose, 0, 0, 0, true, D);
    for (int i = 0; i < 6; i++) {
        for (int p = 0; p < 3; p++)
            for (int j = 0; j < 3; j++) out[i * 12 + p * 3 + j] = D[p * 18 + i * 3 + j];
        for (int j = 9; j < 12; j++) out[i * 12 + j] = 0;
    }
    return ok;
}

}  // namespace dsac
