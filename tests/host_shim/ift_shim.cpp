// Host build of the implicit-function derivatives (dsac_b200/csrc/ift.cuh compiled with DSAC_HOST_ONLY) and of the
// product's P3P and Kabsch solvers in double, for tests/test_ift_host.py.  Test infrastructure only.
#define DSAC_HOST_ONLY 1
#include "../../dsac_b200/csrc/ift.cuh"

extern "C" {
int shim_ift_fit_deriv(int m, const double* Y, const double* e, const double* pose, double f, double cx, double cy, int rgbd,
                       double* D) {
    return dsac::ift_fit_deriv(m, Y, e, pose, f, cx, cy, rgbd != 0, D) ? 1 : 0;
}
int shim_ift_dpnp_p3p(const double* pose, const double* X, const double* uv, double f, double cx, double cy, double* out) {
    return dsac::ift_dpnp_p3p(pose, X, uv, f, cx, cy, out) ? 1 : 0;
}
int shim_ift_dpnp_kabsch(const double* a, const double* b, double* out) { return dsac::ift_dpnp_kabsch(a, b, out) ? 1 : 0; }
void shim_ift_jp_jacobian(const double* pose, double* R, double* M) { dsac::ift_jp_jacobian(pose, R, M); }
// the product's P3P (points 0..2, the 4th picks the solution) on double-valued points and pixels
int shim_p3p_double(const double* X, const double* uv, double f, double cx, double cy, double* R, double* t) {
    dsac::P3PProblem pr;
    for (int i = 0; i < 4; i++) {
        pr.mu[i] = uv[i * 2];
        pr.mv[i] = uv[i * 2 + 1];
        for (int k = 0; k < 3; k++) pr.X[i][k] = X[i * 3 + k];
    }
    double e2;
    return dsac::p3p_best(pr, f, cx, cy, R, t, &e2);
}
void shim_kabsch(int m, const double* a, const double* b, double* R, double* t) { dsac::kabsch_fit(m, a, b, R, t); }
}
