// rigid.cuh -- the rigid-body fit (Kabsch) and the RGB-D acceptance test of a minimal set.
//
//   kabsch_fit   b ~ R a + t over m point pairs (Hypothesis::calcRigidBodyTransform, Hypothesis.cpp:145-200); k_kabsch,
//                the RGB-D sampler and the RGB-D refinement all call it
//   rgbd_accept  the acceptance test of an RGB-D minimal set (dsac_set_cell_depth_device): depth, non-degenerate triangles,
//                Kabsch on points 0..2, all four points in front of the camera, then the reference's reprojection check
#pragma once
#ifdef __CUDACC__
#include <cuda_runtime.h>
#endif

#include "pose_math.cuh"

namespace dsac {

constexpr uint32_t ST_NO_DEPTH = 64u;   // DSAC_ST_NO_DEPTH

// Jacobi eigen-decomposition of a symmetric 3x3 matrix: S = V diag(w) V^T.
DSAC_HDN void sym_eig3(const double S[9], double w[3], double V[9]) {
    double A[9];
    for (int i = 0; i < 9; i++) { A[i] = S[i]; V[i] = (i % 4 == 0) ? 1.0 : 0.0; }
    for (int sweep = 0; sweep < 40; sweep++) {
        double off = fabs(A[1]) + fabs(A[2]) + fabs(A[5]);
        if (off == 0.0) break;
        for (int pq = 0; pq < 3; pq++) {
            const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
            double apq = A[p * 3 + q];
            if (apq == 0.0) continue;
            double theta = (A[q * 3 + q] - A[p * 3 + p]) / (2.0 * apq);
            double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
            double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
            for (int k = 0; k < 3; k++) {
                double akp = A[k * 3 + p], akq = A[k * 3 + q];
                A[k * 3 + p] = c * akp - s * akq;
                A[k * 3 + q] = s * akp + c * akq;
            }
            for (int k = 0; k < 3; k++) {
                double apk = A[p * 3 + k], aqk = A[q * 3 + k];
                A[p * 3 + k] = c * apk - s * aqk;
                A[q * 3 + k] = s * apk + c * aqk;
            }
            A[p * 3 + q] = A[q * 3 + p] = 0.0;
            for (int k = 0; k < 3; k++) {
                double vkp = V[k * 3 + p], vkq = V[k * 3 + q];
                V[k * 3 + p] = c * vkp - s * vkq;
                V[k * 3 + q] = s * vkp + c * vkq;
            }
        }
    }
    w[0] = A[0]; w[1] = A[4]; w[2] = A[8];
}

// b ~ R a + t with R = V diag(1,1,sign) U^T from the SVD of sum (a-ca)(b-cb)^T; a, b: m points of 3 doubles.  A proper
// rotation also for m = 3 (rank-2 covariance): the third left vector then completes the right-handed frame.
DSAC_HD void kabsch_fit(int m, const double* pa, const double* pb, double Ro[9], double to[3]) {
    double cA[3] = {0, 0, 0}, cB[3] = {0, 0, 0};
    for (int k = 0; k < m; k++)
        for (int d = 0; d < 3; d++) { cA[d] += pa[k * 3 + d]; cB[d] += pb[k * 3 + d]; }
    for (int d = 0; d < 3; d++) { cA[d] *= 1.0 / (double)m; cB[d] *= 1.0 / (double)m; }
    double C[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};   // pointsA * pointsB^T
    for (int k = 0; k < m; k++)
        for (int r = 0; r < 3; r++)
            for (int c = 0; c < 3; c++) C[r * 3 + c] += (pa[k * 3 + r] - cA[r]) * (pb[k * 3 + c] - cB[c]);
    // SVD C = U diag(s) V^T through the eigen-decomposition of C^T C (V) and U = C V / s
    double S[9], w[3], V[9];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) S[r * 3 + c] = C[0 * 3 + r] * C[0 * 3 + c] + C[1 * 3 + r] * C[1 * 3 + c] + C[2 * 3 + r] * C[2 * 3 + c];
    sym_eig3(S, w, V);
    // order eigenvalues descending
    int o[3] = {0, 1, 2};
    if (w[o[0]] < w[o[1]]) { int x = o[0]; o[0] = o[1]; o[1] = x; }
    if (w[o[1]] < w[o[2]]) { int x = o[1]; o[1] = o[2]; o[2] = x; }
    if (w[o[0]] < w[o[1]]) { int x = o[0]; o[0] = o[1]; o[1] = x; }
    double Vs[9], U[9];
    for (int j = 0; j < 3; j++)
        for (int k = 0; k < 3; k++) Vs[k * 3 + j] = V[k * 3 + o[j]];
    for (int j = 0; j < 2; j++) {
        double u[3], nn = 0;
        for (int k = 0; k < 3; k++) { u[k] = C[k * 3] * Vs[0 * 3 + j] + C[k * 3 + 1] * Vs[1 * 3 + j] + C[k * 3 + 2] * Vs[2 * 3 + j]; nn += u[k] * u[k]; }
        nn = nn > 0 ? 1.0 / sqrt(nn) : 0.0;
        for (int k = 0; k < 3; k++) U[k * 3 + j] = u[k] * nn;
    }
    // third left vector: C v3 / s3 when s3 is well above rounding, else completes the right-handed frame
    {
        double u[3], nn = 0;
        for (int k = 0; k < 3; k++) { u[k] = C[k * 3] * Vs[0 * 3 + 2] + C[k * 3 + 1] * Vs[1 * 3 + 2] + C[k * 3 + 2] * Vs[2 * 3 + 2]; nn += u[k] * u[k]; }
        double cr[3] = {U[3] * U[7] - U[6] * U[4], U[6] * U[1] - U[0] * U[7], U[0] * U[4] - U[3] * U[1]};
        if (nn > 1e-24 * (w[o[0]] > 0 ? w[o[0]] : 1.0)) {
            nn = 1.0 / sqrt(nn);
            for (int k = 0; k < 3; k++) U[k * 3 + 2] = u[k] * nn;
        } else {
            for (int k = 0; k < 3; k++) U[k * 3 + 2] = cr[k];
        }
    }
    // sign = det(V U^T) < 0 ? -1 : 1 ; R = V diag(1,1,sign) U^T
    double VUt[9];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) VUt[r * 3 + c] = Vs[r * 3] * U[c * 3] + Vs[r * 3 + 1] * U[c * 3 + 1] + Vs[r * 3 + 2] * U[c * 3 + 2];
    double det = VUt[0] * (VUt[4] * VUt[8] - VUt[5] * VUt[7]) - VUt[1] * (VUt[3] * VUt[8] - VUt[5] * VUt[6]) + VUt[2] * (VUt[3] * VUt[7] - VUt[4] * VUt[6]);
    double sign = det < 0 ? -1.0 : 1.0;
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) Ro[r * 3 + c] = Vs[r * 3] * U[c * 3] + Vs[r * 3 + 1] * U[c * 3 + 1] + sign * Vs[r * 3 + 2] * U[c * 3 + 2];
    for (int r = 0; r < 3; r++) to[r] = -(Ro[r * 3] * cA[0] + Ro[r * 3 + 1] * cA[1] + Ro[r * 3 + 2] * cA[2]) + cB[r];
}

// |(P1 - P0) x (P2 - P0)|^2 >= 1 mm^4: the triangle spans at least 1 mm^2 of (doubled) area
DSAC_HD bool triangle_ok(const double* P) {
    const double a0 = P[3] - P[0], a1 = P[4] - P[1], a2 = P[5] - P[2];
    const double b0 = P[6] - P[0], b1 = P[7] - P[1], b2 = P[8] - P[2];
    const double c0 = a1 * b2 - a2 * b1, c1 = a2 * b0 - a0 * b2, c2 = a0 * b1 - a1 * b0;
    return c0 * c0 + c1 * c1 + c2 * c2 >= 1.0;
}

// The RGB-D acceptance test of one minimal set.  scene / eye: the four points (mm, eye coordinates NaN where the cell has
// no depth); obj / img: the float correspondences of the reprojection check.  R, t: the least-squares rigid transform
// eye ~ R scene + t of points 0..2; the hypothesis is (rodrigues(R), t) as minimal_set_accept leaves it, which also sets
// *fragile.
DSAC_HDN bool rgbd_accept(const double scene[12], const double eye[12], const float obj[12], const float img[8], double f,
                          double cx, double cy, int thr, double rvec[3], double tvec[3], bool* fragile) {
    *fragile = false;
    for (int j = 0; j < 4; j++)
        if (!(eye[j * 3 + 2] > 0.0)) return false;   // (NaN: no depth)
    if (!triangle_ok(scene) || !triangle_ok(eye)) return false;
    double R[9], t[3];
    kabsch_fit(3, scene, eye, R, t);
    for (int j = 0; j < 4; j++) {
        const double z = R[6] * scene[j * 3] + R[7] * scene[j * 3 + 1] + R[8] * scene[j * 3 + 2] + t[2];
        if (!(z > 0.0)) return false;
    }
    return minimal_set_accept(obj, img, f, cx, cy, thr, R, t, 0.0, rvec, tvec, fragile);
}

// The inputs of rgbd_accept for cells[4] of one frame: coords [N][3] int16, eye [N][3] fp64, pix [N][2].
DSAC_HDN bool rgbd_accept_cells(const int16_t* coords, const double* eye, const int32_t* pix, const int cells[4], double f, double cx,
                                double cy, int thr, double rvec[3], double tvec[3], bool* fragile) {
    double scene[12], ex[12];
    float obj[12], img[8];
    for (int j = 0; j < 4; j++) {
        const int c = cells[j];
        for (int k = 0; k < 3; k++) {
            scene[j * 3 + k] = (double)coords[c * 3 + k];
            ex[j * 3 + k] = eye[c * 3 + k];
            obj[j * 3 + k] = (float)scene[j * 3 + k];
        }
        img[j * 2] = (float)pix[c * 2];
        img[j * 2 + 1] = (float)pix[c * 2 + 1];
    }
    return rgbd_accept(scene, ex, obj, img, f, cx, cy, thr, rvec, tvec, fragile);
}

}  // namespace dsac
