// Host build of the RGB-D rig arithmetic (dsac_b200/csrc/pose_math.cuh, rigid.cuh and ift.cuh with DSAC_HOST_ONLY): the
// rig-frame eye point, the rig Kabsch fit as k_refine_rig_rgbd forms it, and the implicit-function derivative and the
// covariance of that fit as k_refine_ift_rig_rgbd and k_pose_uncertainty_rig_rgbd form them, for
// tests/test_rig_rgbd_host.py and tests/test_gpu_rig_rgbd.py.  Test infrastructure only.
#define DSAC_HOST_ONLY 1
#include <vector>

#include "../../dsac_b200/csrc/ift.cuh"

namespace {
// cell i of camera cam[i] (Y [m][3], eye point e [m][3]) set up in its camera frame at the composed pose, mapped to the rig's
void rig_rgbd_point(const double* ext, const int* cam, const double* Y, const double* e, const double R[9], const double t[3],
                    int i, dsac::IftPoint& P) {
    const double* E = ext + cam[i] * 12;
    double Rk[9], tk[3];
    dsac::rig_compose(E, E + 9, R, t, Rk, tk);
    dsac::ift_point_setup(Rk, tk, Y + i * 3, e + i * 3, 0, 0, 0, true, P);
    dsac::ift_point_to_rig(E, P);
}
}  // namespace

extern "C" {
void shim_rig_point(const double* Rc, const double* tc, const double* e, double* o) { dsac::rig_point(Rc, tc, e, o); }

// The rig Kabsch fit over m cells in order: cam [m], Y [m][3] scene, e [m][3] camera-frame eye points, ext [C][12] (Rc
// row-major, tc); pose [6] the cv rig pose (rodrigues of the fitted rotation, translation).
void shim_rig_kabsch(int m, const int* cam, const double* Y, const double* e, const double* ext, double* pose) {
    std::vector<double> b((size_t)m * 3);
    for (int i = 0; i < m; i++) {
        const double* E = ext + cam[i] * 12;
        dsac::rig_point(E, E + 9, e + i * 3, &b[(size_t)i * 3]);
    }
    double R[9];
    dsac::kabsch_fit(m, Y, b.data(), R, pose + 3);
    dsac::rodrigues_m2v(R, pose);
}

// D [m][6][3] = d jp6 / dY_i of the rig Kabsch fit at the cv rig pose; 0 (D zero) as ift_fit_deriv.
int shim_rig_rgbd_ift_deriv(int m, const int* cam, const double* Y, const double* e, const double* ext, const double* pose, double* D) {
    double R[9], M[36], H[21] = {0}, W[36];
    dsac::ift_jp_jacobian(pose, R, M);
    dsac::IftPoint P;
    for (int i = 0; i < m; i++) {
        rig_rgbd_point(ext, cam, Y, e, R, pose + 3, i, P);
        dsac::ift_point_hess(P, H);
    }
    bool ok = m > 0 && dsac::ift_chol6(H);
    if (ok) dsac::ift_weights(H, M, W);
    for (int i = 0; i < m && ok; i++) {
        double B[18];
        rig_rgbd_point(ext, cam, Y, e, R, pose + 3, i, P);
        dsac::ift_point_cross(P, R, B);
        dsac::ift_point_deriv(W, B, D + i * 18);
        for (int k = 0; k < 18; k++) ok = ok && D[i * 18 + k] - D[i * 18 + k] == 0.0;
    }
    if (!ok)
        for (int k = 0; k < m * 18; k++) D[k] = 0;
    return ok ? 1 : 0;
}

// The covariance of the rig Kabsch fit over m cells; outputs and return value as ift_cov_from_info (RGB-D: 3m - 6).
int shim_rig_rgbd_fit_covariance(int m, const int* cam, const double* Y, const double* e, const double* ext, const double* pose,
                                 double* cov_xi, double* cov_jp6, double* sigma2) {
    double R[9], acc[22] = {0};
    dsac::rodrigues_v2m(pose, R);
    dsac::IftPoint P;
    for (int i = 0; i < m; i++) {
        rig_rgbd_point(ext, cam, Y, e, R, pose + 3, i, P);
        dsac::ift_point_gn(P, acc);
    }
    return dsac::ift_cov_from_info(acc, acc[21], m, true, pose, cov_xi, cov_jp6, sigma2) ? 1 : 0;
}

// ift_fit_covariance (RGB-D) over m cells of one camera
int shim_fit_covariance_rgbd(int m, const double* Y, const double* e, const double* pose, double* cov_xi, double* cov_jp6,
                             double* sigma2) {
    return dsac::ift_fit_covariance(m, Y, e, pose, 0, 0, 0, true, cov_xi, cov_jp6, sigma2) ? 1 : 0;
}
}
