// Host build of the rig backward's fp64 arithmetic (dsac_b200/csrc/ift.cuh with DSAC_HOST_ONLY): the lift's and the
// composition's Jacobians, and the implicit-function derivative of a rig fit over cells of several cameras as
// k_refine_ift_rig forms it, for tests/test_rig_grad_host.py.  Test infrastructure only.
#define DSAC_HOST_ONLY 1
#include "../../dsac_b200/csrc/ift.cuh"

extern "C" {
void shim_rig_lift_jac(const double* Rc, const double* r, double* L) { dsac::rig_lift_jac(Rc, r, L); }
void shim_rig_cross_jac(const double* Rc, const double* Rc2, const double* Rh, int same, double* K) {
    dsac::rig_cross_jac(Rc, Rc2, Rh, same != 0, K);
}
// m cells: cam [m] camera index, Y [m][3], uv [m][2]; ext [C][12] (Rc row-major, tc), fcc [C][3] (f, cx, cy); pose the
// rig's cv pose.  D [m][6][3] = d jp6 / dY_i; 0 (D zero) when the Hessian is not positive definite or D is not finite.
int shim_rig_ift_deriv(int m, const int* cam, const double* Y, const double* uv, const double* ext, const double* fcc,
                       const double* pose, double* D) {
    double R[9], M[36], H[21] = {0}, W[36];
    dsac::ift_jp_jacobian(pose, R, M);
    auto point = [&](int i, dsac::IftPoint& P) {
        const double* E = ext + cam[i] * 12;
        const double* c = fcc + cam[i] * 3;
        const double e[3] = {uv[i * 2], uv[i * 2 + 1], 0};
        double Rk[9], tk[3];
        dsac::rig_compose(E, E + 9, R, pose + 3, Rk, tk);
        dsac::ift_point_setup(Rk, tk, Y + i * 3, e, c[0], c[1], c[2], false, P);
        dsac::ift_point_to_rig(E, P);
    };
    dsac::IftPoint P;
    for (int i = 0; i < m; i++) {
        point(i, P);
        dsac::ift_point_hess(P, H);
    }
    bool ok = m > 0 && dsac::ift_chol6(H);
    if (ok) dsac::ift_weights(H, M, W);
    for (int i = 0; i < m && ok; i++) {
        double B[18];
        point(i, P);
        dsac::ift_point_cross(P, R, B);
        dsac::ift_point_deriv(W, B, D + i * 18);
        for (int k = 0; k < 18; k++) ok = ok && D[i * 18 + k] - D[i * 18 + k] == 0.0;
    }
    if (!ok)
        for (int k = 0; k < m * 18; k++) D[k] = 0;
    return ok ? 1 : 0;
}
}
