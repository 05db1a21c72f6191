// Host build of the rig tracking arithmetic (dsac_b200/csrc/prior.cuh and ift.cuh with DSAC_HOST_ONLY): the composition of
// a rig prior with an extrinsic, the prior gate's distance, and the covariance of a rig fit over cells of several cameras as
// k_pose_uncertainty_rig forms it, for tests/test_rig_tracking_host.py and tests/test_gpu_rig_tracking.py.  Test
// infrastructure only.
#define DSAC_HOST_ONLY 1
#include "../../dsac_b200/csrc/ift.cuh"
#include "../../dsac_b200/csrc/prior.cuh"

extern "C" {
// ext [6], pose [6], info [36] or null; out_pose [6], out_info [36] (written with info).  1: the extrinsic is finite.
int shim_rig_prior_compose(const double* ext, const double* pose, const double* info, double* out_pose, double* out_info) {
    return dsac::rig_prior_compose(ext, pose, info, out_pose, out_info) ? 1 : 0;
}
// d^2 of the cv pose hyp [6] against the prior (pose [6], info [36]); -1 when prior_entry refuses the prior.
double shim_prior_d2(const double* hyp, const double* pose, const double* info) {
    dsac::PriorGate g;
    if (!dsac::prior_entry(pose, info, g)) return -1.0;
    double R[9];
    dsac::rodrigues_v2m(hyp, R);
    return dsac::prior_d2(R, hyp + 3, g);
}
// The rig fit's covariance over m cells: cam [m], Y [m][3], uv [m][2], ext [C][12] (Rc row-major, tc), fcc [C][3]
// (f, cx, cy), pose the rig's cv pose; outputs and the return value as ift_cov_from_info.
int shim_rig_fit_covariance(int m, const int* cam, const double* Y, const double* uv, const double* ext, const double* fcc,
                            const double* pose, double* cov_xi, double* cov_jp6, double* sigma2) {
    double R[9], acc[22] = {0};
    dsac::rodrigues_v2m(pose, R);
    for (int i = 0; i < m; i++) {
        const double* E = ext + cam[i] * 12;
        const double* c = fcc + cam[i] * 3;
        const double e[3] = {uv[i * 2], uv[i * 2 + 1], 0};
        double Rk[9], tk[3];
        dsac::rig_compose(E, E + 9, R, pose + 3, Rk, tk);
        dsac::IftPoint P;
        dsac::ift_point_setup(Rk, tk, Y + i * 3, e, c[0], c[1], c[2], false, P);
        dsac::ift_point_to_rig(E, P);
        dsac::ift_point_gn(P, acc);
    }
    return dsac::ift_cov_from_info(acc, acc[21], m, false, pose, cov_xi, cov_jp6, sigma2) ? 1 : 0;
}
// ift_fit_covariance (RGB) over m cells of one camera
int shim_fit_covariance(int m, const double* Y, const double* uv, const double* fcc, const double* pose, double* cov_xi,
                        double* cov_jp6, double* sigma2) {
    double* e = new double[(size_t)m * 3 + 1];
    for (int i = 0; i < m; i++) { e[i * 3] = uv[i * 2]; e[i * 3 + 1] = uv[i * 2 + 1]; e[i * 3 + 2] = 0; }
    const bool ok = dsac::ift_fit_covariance(m, Y, e, pose, fcc[0], fcc[1], fcc[2], false, cov_xi, cov_jp6, sigma2);
    delete[] e;
    return ok ? 1 : 0;
}
}
